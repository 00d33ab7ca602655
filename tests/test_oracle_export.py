"""CPU-only properties of the oracle of include/cvb200_export.h (oracle/ref_export.c): the restatement of cv-sfm's
triangulate_landmark_robust, export_reconstruction and normalize_reconstruction that the device is held to bit for bit.

No scene here reaches CVB_EXPORT_AT_INFINITY: a robust landmark has two world-frame bearings at an angle, and then none of the three
triangulators returns a point whose w is exactly zero (LinearEigen's null vector has w = 0 only for parallel bearings, MeanMean's w is zero
only when an observation's cross product with the mean bearing underflows, which makes the sum NaN first).  The state is kept because the
reference distinguishes it."""
import io
import os
import tempfile

import numpy as np
import pytest

from oracle import pyoracle_export as X
from oracle.pyoracle_reconstruction import CONSTRAINT_DTYPE
from oracle.pyoracle_tri import LINEAR_EIGEN, SINE_L1, triangulator
from tests.export_scenes import args, colors_for, exact_scene, first_view_without_robust_landmark, negate_landmark, with_empty_view
from tests.reconstruction_scenes import inv, mul, recon_scene

POINT, NOT_ROBUST, TRI_FAILED, AT_INFINITY = 0, 1, 2, 3


@pytest.mark.parametrize("method", [LINEAR_EIGEN, SINE_L1])
def test_noise_free_scene_gives_the_true_points(method):
    """(MeanMean is an approximation even on exact bearings, so it is left out.)"""
    s, world = exact_scene(8)
    r = X.robust_landmarks(*args(s), tri=triangulator(method))
    pts = r["points"][r["state"] == POINT]
    assert len(pts) > 50
    assert np.all(np.isnan(world[r["state"] == NOT_ROBUST][:, 0]) | (np.diff(s["landmark_offsets"])[r["state"] == NOT_ROBUST] < 3))
    got = pts[:, :3] / pts[:, 3:]
    assert np.abs(got - world[r["state"] == POINT]).max() < 1e-9


def test_states_not_robust_and_triangulation_failed_are_reached():
    s, _ = exact_scene(6)
    lo = s["landmark_offsets"]
    l = next(i for i in range(len(lo) - 1) if lo[i + 1] - lo[i] >= 3)
    r = X.robust_landmarks(*args(negate_landmark(s, l)))
    assert r["state"][l] == TRI_FAILED and not r["points"][l].any()
    assert set(np.unique(r["state"])) == {POINT, NOT_ROBUST, TRI_FAILED}
    single = np.diff(lo) == 1
    assert np.all(r["state"][single] == NOT_ROBUST)


def _distances(s, pts, state, v):
    P = s["poses"][v]
    R, t = P[:9].reshape(3, 3), P[9:]
    vo, vl = s["view_offsets"], s["view_landmarks"]
    out = []
    for l in vl[vo[v]:vo[v + 1]]:
        if state[l] in (POINT, AT_INFINITY):
            h = pts[l]
            x = R @ h[:3] + t * h[3]
            out.append(np.linalg.norm(x / h[3]))
    return out


def test_running_mean_equals_numpy_mean():
    s, _, _ = recon_scene(16, points=300)
    r = X.robust_landmarks(*args(s))
    e = X.export_reconstruction(*args(s), colors_for(s))
    for v in range(16):
        d = _distances(s, r["points"], r["state"], v)
        assert len(d) > 10
        assert abs(e["mean_distance"][v] - np.mean(d)) <= 1e-12 * np.mean(d)
        assert e["cameras"][v]["focal_length"] == e["mean_distance"][v] * 0.01


def test_empty_view_gives_nan():
    s, _ = exact_scene(5)
    s = with_empty_view(s)
    e = X.export_reconstruction(*args(s), colors_for(s))
    assert np.isnan(e["mean_distance"][-1]) and np.isnan(e["cameras"][-1]["focal_length"])
    assert np.isfinite(e["mean_distance"][:-1]).all()


def test_cameras_and_points_follow_the_reference_formulas():
    s, _, _ = recon_scene(8, points=200)
    col = colors_for(s, 3)
    e = X.export_reconstruction(*args(s), col)
    r = X.robust_landmarks(*args(s))
    keep = np.flatnonzero(r["state"] == POINT)
    assert e["points"].shape == (len(keep), 3)
    assert np.array_equal(e["points"], r["points"][keep, :3] / r["points"][keep, 3:])
    lo, ob, vo = s["landmark_offsets"], s["observations"], s["view_offsets"]
    first = ob[lo[keep]]
    assert np.array_equal(e["colors"], col[vo[first[:, 0]] + first[:, 1]])
    for v in range(8):
        c2w = inv(s["poses"][v])
        R = c2w[:9].reshape(3, 3)
        c = e["cameras"][v]
        assert np.allclose(c["optical_center"], c2w[9:], atol=1e-14)
        assert np.allclose(c["up_direction"], -R[:, 1], atol=1e-15) and np.allclose(c["forward_direction"], R[:, 2], atol=1e-15)


def test_normalisation_moves_the_first_view_to_the_origin_at_unit_scale():
    """Exact bearings at the true poses: otherwise LinearEigen's least squares are not invariant to the similarity, so the recomputed mean would move."""
    s, _, cons = recon_scene(12, points=300, noise=0.0, pose_rot=0.0, pose_trans=0.0)
    for first in (0, 5):
        n = X.normalize_reconstruction(*args(s), cons, first_view=first)
        assert n["result"]["normalized"] == 1 and n["result"]["robust_points"] > 10
        P = n["poses"]
        assert np.abs(P[first] - np.concatenate([np.eye(3).reshape(9), np.zeros(3)])).max() < 1e-12
        s2 = dict(s, poses=P)
        again = X.normalize_reconstruction(*args(s2), cons, first_view=first)
        assert abs(again["result"]["mean_distance"] - 1.0) < 1e-12
        k = 1.0 / n["result"]["mean_distance"]
        T = inv(s["poses"][first])
        for v in range(12):
            want = mul(s["poses"][v], T)
            assert np.abs(P[v][:9] - want[:9]).max() < 1e-12   # relative rotations kept
            assert np.abs(P[v][9:] - want[9:] * k).max() < 1e-12
        for field in ("views", "landmarks"):
            assert np.array_equal(n["constraints"][field], cons[field])
        assert np.array_equal(n["constraints"]["poses"]["r"], cons["poses"]["r"])
        assert np.array_equal(n["constraints"]["poses"]["t"], cons["poses"]["t"] * k)


def test_non_normal_mean_returns_the_inputs_bit_for_bit():
    s = first_view_without_robust_landmark()
    cons = np.zeros(1, CONSTRAINT_DTYPE)
    cons["views"] = [[1, 2, 3]]
    cons["poses"]["t"] = 0.5
    n = X.normalize_reconstruction(*args(s), cons, first_view=0)
    assert n["result"]["normalized"] == 0 and n["result"]["robust_points"] == 0 and np.isnan(n["result"]["mean_distance"])
    assert n["poses"].tobytes() == np.ascontiguousarray(s["poses"]).tobytes()
    assert n["constraints"].tobytes() == cons.tobytes()


def test_robust_minimum_observations_two_three_and_above_the_view_count():
    s, _, _ = recon_scene(6, points=300)
    counts = np.diff(s["landmark_offsets"])
    st = {m: X.robust_landmarks(*args(s), cfg=X.ExportCfg(robust_minimum_observations=m))["state"] for m in (2, 3, 6, 7, 100)}
    assert np.all(st[2][counts == 1] == NOT_ROBUST) and np.any((st[2] == POINT) & (counts == 2))
    assert np.all(st[3][counts < 3] == NOT_ROBUST) and np.any(st[3] == POINT)
    assert np.all(st[6][counts < 6] == NOT_ROBUST) and np.any(st[6] == POINT)
    # min(robust_minimum_observations, V): above V the requirement is every view
    assert np.array_equal(st[7], st[6]) and np.array_equal(st[100], st[6])


def test_ply_has_five_vertices_and_four_faces_per_camera():
    from cv_b200.export import write_ply
    s, _, _ = recon_scene(8, points=200)
    e = X.export_reconstruction(*args(s), colors_for(s))
    with tempfile.TemporaryDirectory() as d:
        p = os.path.join(d, "r.ply")
        write_ply(p, e["points"], e["colors"], e["cameras"], camera_faces=True)
        text = open(p).read()
    V, n = 8, len(e["points"])
    assert f"element vertex {5 * V + n}\n" in text and f"element face {4 * V}\n" in text
    body = text.split("end_header\n")[1].splitlines()
    assert len(body) == 5 * V + n + 4 * V
    assert all(line.endswith(" 255 0 255") for line in body[:5 * V])
    buf = io.StringIO()
    from cv_b200.formats import export_ply
    export_ply(buf, list(zip(e["points"], e["colors"])), [], False)
    assert f"element vertex {n}\n" in buf.getvalue() and "element face" not in buf.getvalue()

"""GPU parity for cv-pinhole on the device (include/cvb200_pinhole.h): the pose reprojection error over all six triangulators and the
EssentialMatrix model equal the CPU oracle (oracle/ref_pinhole.c) bit for bit on seeded batches that include degenerate and failing
rows.  Both sides use only +, -, x, / and sqrt in f64 without contraction.  NaN rows are compared by position: the NaN a computation
produces has a platform-dependent sign and payload."""
import ctypes as C

import numpy as np
import pytest

import cv_b200
from cv_b200 import pinhole as P
from cv_b200.geom import POSE_DTYPE
from oracle import pyoracle_pinhole as O
from oracle import pyoracle_tri as T
from tests.geom_util import rot_angle, two_view_scene, unit
from tests.pinhole_cases import DOC_POSE, essential_batch, random_rs_scene, reprojection_batch

pytestmark = pytest.mark.gpu

REL_CLASSES = [cv_b200.LinearEigenTriangulator, cv_b200.SineL1Triangulator, cv_b200.MeanMeanTriangulator, cv_b200.RelativeDltTriangulator,
               cv_b200.AngularL1Triangulator, cv_b200.AngularLInfinityTriangulator]


def _same(x, y):
    x, y = np.asarray(x, np.float64), np.asarray(y, np.float64)
    nx, ny = np.isnan(x), np.isnan(y)
    return x.shape == y.shape and np.array_equal(nx, ny) and np.array_equal(x[~nx].view(np.uint64), y[~ny].view(np.uint64))


def _oracle_cfg(tri):
    c = tri.cfg
    return T.triangulator(c.method, c.epsilon, c.max_iterations, c.optimization_rate)


def _poses(Rs, ts):
    p = np.zeros(len(Rs), POSE_DTYPE)
    p["r"] = np.asarray(Rs).reshape(-1, 9); p["t"] = ts
    return p


@pytest.fixture(scope="module")
def rep_data():
    return reprojection_batch(np.random.default_rng(7), 12000)


@pytest.mark.parametrize("cls", REL_CLASSES, ids=lambda c: c.__name__)
@pytest.mark.parametrize("shared", [False, True], ids=["npose_n", "npose_1"])
def test_reprojection_error_equals_oracle_bit_for_bit(rep_data, cls, shared):
    Rs, ts, a, b = rep_data
    poses = _poses(Rs[:1], ts[:1]) if shared else _poses(Rs, ts)
    tri = cls()
    err, avg, ok = P._reprojection(poses, a, b, tri, None)
    oe, oa, ook = O.pose_reprojection_error_batch(_oracle_cfg(tri), poses, a, b)
    assert np.array_equal(ok, ook), np.flatnonzero(ok != ook)[:10]
    assert _same(err.reshape(-1, 4), oe) and _same(avg, oa)
    assert np.isnan(err[~ok]).all() and np.isnan(avg[~ok]).all()
    assert 0 < ok.sum() < len(ok)
    assert np.isnan(avg[ok]).any() or np.isinf(avg[ok]).any()          # +0.0 z / +NaN pass the sign test and reach the error


def test_reprojection_doc_tests():
    # cv-pinhole/src/lib.rs:291-313, 344-364
    pa = np.array([0.4, -0.25, 5.0]); R, t = np.eye(3), np.array([0.1, 0.2, -0.5])
    a, b = unit(pa), unit(R @ pa + t)
    for cls in REL_CLASSES:
        avg = cv_b200.average_pose_reprojection_error((R, t), a, b, cls())
        e = cv_b200.pose_reprojection_error((R, t), a, b, cls())
        assert avg is not None and e is not None and e.shape == (2, 2)
        assert avg < (1e-2 if cls is cv_b200.MeanMeanTriangulator else 1e-6), (cls.__name__, avg)
        assert abs(np.linalg.norm(e, axis=1).sum() * 0.5 - avg) < 1e-15


def _dev_chain(a, b, found_override=None, n_max_pad=64, tri=None):
    import torch
    from cv_b200.pair import bind
    ctx = cv_b200.Context(0)
    bind(ctx.lib)
    cv_b200.geom._lib(ctx)
    dev = torch.device("cuda", 0)
    n = len(a); n_max = n + n_max_pad
    ta = torch.zeros(n_max * 3, dtype=torch.float64, device=dev); tb = torch.zeros(n_max * 3, dtype=torch.float64, device=dev)
    ta[:3 * n] = torch.from_numpy(a.reshape(-1)).to(dev); tb[:3 * n] = torch.from_numpy(b.reshape(-1)).to(dev)
    n_dev = torch.tensor([n], dtype=torch.int32, device=dev)
    model = torch.zeros(12, dtype=torch.float64, device=dev)
    inl = torch.zeros(n_max, dtype=torch.int32, device=dev); ninl = torch.zeros(1, dtype=torch.int32, device=dev)
    found = torch.zeros(1, dtype=torch.int32, device=dev)
    sentinel = -1234.5
    err = torch.full((n_max * 4,), sentinel, dtype=torch.float64, device=dev)
    avg = torch.full((n_max,), sentinel, dtype=torch.float64, device=dev)
    ok = torch.full((n_max,), 7, dtype=torch.uint8, device=dev)
    torch.cuda.synchronize()
    ars = cv_b200.Arrsac(1e-6, cv_b200.Xoshiro256PlusPlus(5), ctx)
    ctx.check(ctx.lib.cvb_arrsac_eight_point_dev(ctx.handle, C.addressof(ars.cfg), ta.data_ptr(), tb.data_ptr(), n_dev.data_ptr(), n_max,
                                                 C.addressof(ars.rng.state), model.data_ptr(), inl.data_ptr(), n_max, ninl.data_ptr(),
                                                 found.data_ptr()))
    if found_override is not None:
        ctx.sync()
        found.fill_(found_override)
        torch.cuda.synchronize()
    tri = tri or cv_b200.LinearEigenTriangulator()
    P.pose_reprojection_error_dev(model.data_ptr(), 1, ta.data_ptr(), tb.data_ptr(), n_dev.data_ptr(), n_max, found.data_ptr(),
                                  err.data_ptr(), avg.data_ptr(), ok.data_ptr(), tri, ctx)
    ctx.sync()
    out = dict(model=model.cpu().numpy(), found=int(found.item()), err=err.cpu().numpy().reshape(n_max, 4), avg=avg.cpu().numpy(),
               ok=ok.cpu().numpy(), n=n, sentinel=sentinel)
    ctx.close()
    return out


@pytest.mark.parametrize("cls", [cv_b200.LinearEigenTriangulator, cv_b200.AngularL1Triangulator], ids=lambda c: c.__name__)
def test_device_chain_equals_host_entry_point(cls):
    _, _, a, b, _ = two_view_scene(np.random.default_rng(40), 2000, outlier_frac=0.3, noise=1e-4)
    r = _dev_chain(a, b, tri=cls())
    assert r["found"] == 1
    n = r["n"]
    pose = (r["model"][:9].reshape(3, 3), r["model"][9:12])
    err, avg, ok = P._reprojection([pose], a, b, cls(), None)
    assert np.array_equal(r["ok"][:n].astype(bool), ok)
    assert _same(r["err"][:n], err.reshape(-1, 4)) and _same(r["avg"][:n], avg)
    assert (r["err"][n:] == r["sentinel"]).all() and (r["avg"][n:] == r["sentinel"]).all() and (r["ok"][n:] == 7).all()
    assert ok.sum() > n // 2


def test_device_chain_not_found_marks_every_row():
    _, _, a, b, _ = two_view_scene(np.random.default_rng(41), 500, outlier_frac=0.2, noise=1e-4)
    r = _dev_chain(a, b, found_override=0)
    n = r["n"]
    assert (r["ok"][:n] == 0).all() and np.isnan(r["err"][:n]).all() and np.isnan(r["avg"][:n]).all()
    assert (r["err"][n:] == r["sentinel"]).all() and (r["ok"][n:] == 7).all()


@pytest.mark.parametrize("eps,iters", [(1e-12, 1000), (1e-6, 50), (1e-12, 2)])
def test_eight_point_essential_equals_oracle(eps, iters):
    rng = np.random.default_rng(11)
    _, _, a, b, _ = two_view_scene(rng, 3000, outlier_frac=0.4, noise=1e-3)
    samples = rng.integers(0, len(a), (4096, 8)).astype(np.uint32)
    samples[::16] = samples[::16, :1]                                     # one match eight times: a rank-one design
    E, ok = P.eight_point_essential_batch(a, b, samples, eps, iters)
    oE, ook = O.eight_point_essential_batch(a, b, samples, eps, iters)
    assert np.array_equal(ok, ook) and _same(E, oE)
    if iters == 2:
        assert 0 < ok.sum() < len(ok)
    else:
        assert ok.all()


def test_residuals_essential_equals_oracle():
    rng = np.random.default_rng(12)
    _, _, a, b, _ = two_view_scene(rng, 5000, outlier_frac=0.3, noise=1e-4)
    a[7, 2] = 0.0; b[9] = np.nan
    Es = essential_batch(rng, 64)
    got = P.residuals_essential(Es, a, b)
    assert got.shape == (64, 5000) and _same(got, O.residuals_essential(Es, a, b))


@pytest.mark.parametrize("eps,iters", [(1e-12, 1000), (1e-6, 50), (1e-12, 0)])
def test_recondition_and_decompose_equal_oracle(eps, iters):
    Es = essential_batch(np.random.default_rng(13), 4096)
    E, ok = P.essential_recondition_batch(Es, eps, iters)
    oE, ook = O.essential_recondition_batch(Es, eps, iters)
    assert np.array_equal(ok, ook) and _same(E, oE)
    ra, rb, t, ok2 = P.essential_decompose_batch(Es, eps, iters)
    ora, orb, ot, ook2 = O.essential_decompose_batch(Es, eps, iters)
    assert np.array_equal(ok2, ook2) and _same(ra, ora) and _same(rb, orb) and _same(t, ot)
    if iters == 0:
        assert not ok.any() and not ok2.any()
    else:
        assert not ok[2::8].any() and not ok[3::8].any() and ok[0::8].all()   # rank one and zero: no SVD here (documented)
        assert np.isnan(E[~ok]).all() and np.isnan(ra[~ok2]).all()


def test_eight_point_random_rs_on_device():
    # eight-point/tests/random.rs:14-36: >= 950 of 1000 random scenes have every residual <= 1e-4
    rng = np.random.default_rng(1)
    scenes = [random_rs_scene(rng) for _ in range(1000)]
    a = np.concatenate([s[0] for s in scenes]); b = np.concatenate([s[1] for s in scenes])
    samples = (np.arange(1000)[:, None] * 16 + np.arange(8)[None]).astype(np.uint32)
    E, ok = P.eight_point_essential_batch(a, b, samples)
    assert ok.all()
    successes = sum(bool((np.abs(P.residuals_essential(E[k:k + 1], a[16 * k:16 * k + 16], b[16 * k:16 * k + 16])) <= 1e-4).all())
                    for k in range(1000))
    assert successes > 950, successes
    first = cv_b200.EightPoint().from_matches(a[:16], b[:16])
    assert np.array_equal(first.mat, E[0])


def test_decomposition_doc_tests_on_device():
    # essential.rs:93-113 (possible_rotations_unscaled_translation), 168-183 (possible_rotations), 197-216 (possible_unscaled_poses)
    R, t = DOC_POSE
    E = cv_b200.EssentialMatrix.from_pose((R, t))
    ra, rb, tt = E.possible_rotations_unscaled_translation(1e-6, 50)
    assert rot_angle(ra, R) < 1e-4 or rot_angle(rb, R) < 1e-4
    assert 1.0 - abs(unit(tt) @ unit(t)) < 1e-4
    assert any(rot_angle(r, R) < 1e-4 for r in E.possible_rotations(1e-6, 50))
    poses = E.possible_unscaled_poses(1e-6, 50)
    assert any(rot_angle(Rp, R) < 1e-4 and 1.0 - unit(tp) @ unit(t) < 1e-4 for Rp, tp in poses)
    assert len(E.possible_unscaled_poses_bearing(1e-6, 50)) == 2
    assert np.abs(E.residuals(*[unit(np.array([[0.1, 0.2, 1.0]])), unit(np.array([[0.1, 0.2, 1.0]]) @ R.T + t)])).max() < 1e-12
    Er = E.recondition(1e-12, 1000)
    s = np.linalg.svd(Er.mat, compute_uv=False)
    assert abs(s[0] - s[1]) < 1e-12 * s[0] and s[2] < 1e-12 * s[0]

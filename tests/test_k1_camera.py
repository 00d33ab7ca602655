"""CPU: the K1 camera (cv-pinhole CameraIntrinsicsK1Distortion) and cv-sfm's bicubic colour sampling, oracle and numpy.

  * the oracle meets the reference's doc-tests (cv-pinhole/src/lib.rs:169-190 and :206-223);
  * with k1 = 0 ref_calibrate_k1 is ref_calibrate bit for bit over a grid covering 1920 x 1080 and its borders;
  * cv_b200.CameraIntrinsicsK1Distortion equals the oracle bit for bit, NaN where the reference's uncalibrate yields NaN or None;
  * ref_bicubic_rgb8 (cv-sfm/src/bicubic.rs) on cases that separate it from the plausible wrong alternatives."""
import numpy as np
import pytest

import cv_b200
from cv_b200 import CameraIntrinsics, CameraIntrinsicsK1Distortion
from oracle import pyoracle as O
from oracle import pyoracle_sfm as OS

DOC = (800.0, 900.0, 500.0, 600.0, 1.7)
VSLAM = (893.39010814, 898.32648616, 951.1310043, 555.13350077, 0.0, -0.28052513)      # vslam-sandbox/src/main.rs:71-78
TUTORIAL = (9.842439e+02, 9.808141e+02, 6.900000e+02, 2.331966e+02, 0.0, -3.728755e-01)  # tutorial chapter 5 main.rs:36-42


def _cam(fx, fy, cx, cy, skew, k1):
    return CameraIntrinsicsK1Distortion(CameraIntrinsics((fx, fy), (cx, cy), skew), k1)


def _bits(a):
    return np.ascontiguousarray(a, np.float64).view(np.uint64)


def test_oracle_k1_calibrate_doc_test():
    """cv-pinhole/src/lib.rs:169-190: distance between the K1 bearing's image point and simple / (1 + k1 |simple|^2) < 0.1"""
    k1 = -0.164624
    n = OS.calibrate_k1(*DOC, k1, 471.0, 322.0)
    s = O.calibrate(*DOC, 471.0, 322.0)
    nkp, skp = n[:2] / n[2], s[:2] / s[2]
    assert np.linalg.norm(nkp - skp / (1.0 + k1 * (skp @ skp))) < 0.1


def test_oracle_k1_round_trip_doc_test():
    """cv-pinhole/src/lib.rs:206-223: calibrate -> uncalibrate returns the pixel within 1e-6"""
    b = OS.calibrate_k1(*DOC, -0.164624, 471.0, 322.0)
    p = OS.uncalibrate_k1(*DOC, -0.164624, b)
    assert p is not None and np.linalg.norm(p - np.array([471.0, 322.0])) < 1e-6


def _grid():
    xs = np.concatenate([np.linspace(-2.0, 1922.0, 97), [0.0, 0.5, 1919.0, 1919.5, 1920.0]])
    ys = np.concatenate([np.linspace(-2.0, 1082.0, 61), [0.0, 0.5, 1079.0, 1079.5, 1080.0]])
    X, Y = np.meshgrid(xs, ys)
    return np.stack([X.ravel(), Y.ravel()], 1)


@pytest.mark.parametrize("K", [DOC, VSLAM[:5], TUTORIAL[:5]])
def test_oracle_k1_zero_is_the_undistorted_camera_bit_for_bit(K):
    for x, y in _grid():
        assert _bits(OS.calibrate_k1(*K, 0.0, x, y)).tolist() == _bits(O.calibrate(*K, x, y)).tolist(), (x, y)


@pytest.mark.parametrize("K", [DOC + (-0.164624,), VSLAM, TUTORIAL, DOC + (0.0,), DOC + (0.3,)])
def test_numpy_k1_camera_equals_oracle_bit_for_bit(K):
    cam = _cam(*K)
    px = _grid()
    got = cam.calibrate(px)
    want = np.array([OS.calibrate_k1(*K, x, y) for x, y in px])
    assert np.array_equal(_bits(got), _bits(want))
    # uncalibrate, including its NaN cases: the principal point (k1 * u2 == 0), k1 = 0, 4 k1 u2 > 1 (k1 > 0 far out), z < 0 / -0.0 (None)
    rng = np.random.default_rng(5)
    b = np.concatenate([got, [[0.0, 0.0, 1.0], [0.3, 0.2, -0.9], [0.1, 0.1, -0.0], [0.9, 0.1, 0.1]], rng.normal(size=(200, 3))])
    b /= np.linalg.norm(b, axis=1, keepdims=True)
    back = cam.uncalibrate(b)
    for i, v in enumerate(b):
        w = OS.uncalibrate_k1(*K, v)
        if w is None:
            assert np.isnan(back[i]).all(), i
        else:
            assert _bits(back[i]).tolist() == _bits(w).tolist() or (np.isnan(back[i]) == np.isnan(w)).all() and np.isnan(w).any(), (i, back[i], w)
    assert np.isnan(cam.uncalibrate([[0.0, 0.0, 1.0]])).all()                     # the principal point: 0 / 0
    assert np.isnan(cam.uncalibrate([[0.3, 0.2, -0.9]])).all()                    # None
    if K[5] == 0.0:
        assert np.isnan(back).all()


def test_numpy_k1_round_trip_on_the_reference_cameras():
    for K in (VSLAM, TUTORIAL):
        cam = _cam(*K)
        px = np.random.default_rng(1).uniform([0, 0], [1920, 1080] if K is VSLAM else [1392, 512], (500, 2))
        assert np.abs(cam.uncalibrate(cam.calibrate(px)) - px).max() < 1e-6


def test_calibrate_keypoints_uses_the_f32_coordinates():
    kps = np.zeros(3, cv_b200.KP_DTYPE)
    kps["x"] = [10.25, 951.1, 1900.7]; kps["y"] = [3.5, 555.1, 1070.3]
    cam = _cam(*VSLAM)
    want = np.array([OS.calibrate_k1(*VSLAM, float(k["x"]), float(k["y"])) for k in kps])
    assert np.array_equal(_bits(cam.calibrate_keypoints(kps)), _bits(want))


# ---- cv-sfm/src/bicubic.rs ---------------------------------------------------------------------------------------------------------
def _blend(p0, p1, p2, p3, x):
    f = np.float32
    p0, p1, p2, p3, x = f(p0), f(p1), f(p2), f(p3), f(x)
    return p1 + f(0.5) * x * (p2 - p0 + x * (f(2.0) * p0 - f(5.0) * p1 + f(4.0) * p2 - p3 + x * (f(3.0) * (p1 - p2) + p3 - p0)))


def _clamp(v):
    return 255 if not v < 255 else (int(v) if v > 0 else 0)


def _bicubic_np(img, x, y, clamp_rows=True):
    """float32 restatement for the tests; clamp_rows=False is the plausible mistake of clamping only once at the end"""
    x, y = np.float32(x), np.float32(y)
    left, top = np.floor(x) - np.float32(1), np.floor(y) - np.float32(1)
    h, w = img.shape[:2]
    if left < 0 or left + 4 >= w or top < 0 or top + 4 >= h:
        return np.zeros(3, np.uint8)
    xw, yw = x - (left + np.float32(1)), y - (top + np.float32(1))
    out = np.zeros(3, np.uint8)
    for c in range(3):
        rows = []
        for r in range(4):
            p = img[int(top) + r, int(left):int(left) + 4, c]
            v = _blend(*p, xw)
            rows.append(np.float32(_clamp(v)) if clamp_rows else v)
        out[c] = _clamp(_blend(*rows, yw))
    return out


def test_bicubic_integer_coordinates_return_the_pixel():
    img = np.random.default_rng(2).integers(0, 256, (40, 50, 3), dtype=np.uint8)
    for x, y in [(1, 1), (5, 7), (45, 35), (20, 9)]:
        assert OS.bicubic_rgb8(img, float(x), float(y)).tolist() == img[y, x].tolist()


def test_bicubic_constant_image_returns_the_constant():
    img = np.zeros((30, 30, 3), np.uint8)
    img[...] = (17, 200, 255)
    for x, y in np.random.default_rng(3).uniform(1, 26, (50, 2)):
        assert OS.bicubic_rgb8(img, x, y).tolist() == [17, 200, 255]


def test_bicubic_border_rule_uses_left_plus_four():
    h, w = 30, 40
    img = np.full((h, w, 3), 99, np.uint8)
    below = float(np.nextafter(np.float32(w - 3), np.float32(0)))
    assert OS.bicubic_rgb8(img, 1.0, 10.0).tolist() == [99] * 3            # left = 0: inside
    assert OS.bicubic_rgb8(img, 0.99, 10.0).tolist() == [0] * 3            # left = -1: black
    assert OS.bicubic_rgb8(img, below, 10.0).tolist() == [99] * 3          # left = w - 5, right = w - 1: inside
    assert OS.bicubic_rgb8(img, float(w - 3), 10.0).tolist() == [0] * 3    # right = w: black, though column w - 1 would be readable
    belowy = float(np.nextafter(np.float32(h - 3), np.float32(0)))
    assert OS.bicubic_rgb8(img, 10.0, belowy).tolist() == [99] * 3
    assert OS.bicubic_rgb8(img, 10.0, float(h - 3)).tolist() == [0] * 3
    assert OS.bicubic_rgb8(img, 10.0, 0.5).tolist() == [0] * 3


def test_bicubic_rows_are_clamped_before_the_column_blend():
    img = np.zeros((12, 12, 3), np.uint8)
    img[4, 2:6] = [[0, 0, 0], [255, 255, 255], [255, 255, 255], [0, 0, 0]]     # row blend overshoots above 255
    img[5, 2:6] = [[255, 255, 255], [0, 0, 0], [0, 0, 0], [255, 255, 255]]     # and below 0
    img[6, 2:6] = 255
    x, y = 4.5, 5.5
    want, wrong = _bicubic_np(img, x, y), _bicubic_np(img, x, y, clamp_rows=False)
    assert want.tolist() != wrong.tolist()
    assert OS.bicubic_rgb8(img, x, y).tolist() == want.tolist()


def test_bicubic_equals_the_float32_restatement_on_random_points():
    rng = np.random.default_rng(4)
    img = rng.integers(0, 256, (64, 80, 3), dtype=np.uint8)
    for x, y in rng.uniform(-1, [82, 66], (400, 2)).astype(np.float32):
        assert OS.bicubic_rgb8(img, x, y).tolist() == _bicubic_np(img, x, y).tolist(), (x, y)


def test_oracle_kps_descriptors_is_the_per_keypoint_composition():
    from tests.common import kitti_frame
    img = kitti_frame("0000000000")[:200, :400].copy()
    rgb = np.random.default_rng(6).integers(0, 256, img.shape + (3,), dtype=np.uint8)
    kps, desc, bear, resp, col = OS.kps_descriptors(O.Akaze(detector_threshold=0.001), img, rgb, TUTORIAL)
    assert len(kps) > 20 and len(desc) == len(kps)
    assert np.all(np.diff(resp) <= 0)
    for i in range(len(kps)):
        assert _bits(bear[i]).tolist() == _bits(OS.calibrate_k1(*TUTORIAL, float(kps[i]["x"]), float(kps[i]["y"]))).tolist()
        assert col[i].tolist() == _bicubic_np(rgb, kps[i]["x"], kps[i]["y"]).tolist()

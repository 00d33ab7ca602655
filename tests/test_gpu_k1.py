"""GPU: the K1 camera on the device and cv-sfm's frame ingestion (cvb_frame_features_batch).

  * cvb_pair_bearings_k1_dev equals the oracle bit for bit on random keypoints over 1920 x 1080 with the vslam-sandbox and tutorial
    cameras; with k1 = 0 it equals cvb_pair_bearings_dev bit for bit;
  * tutorial chapter 5 (tutorial-code/chapter5-geometric-verification/src/main.rs) on the committed KITTI frames through
    two_view_frames equals the oracle's pipeline: matches, inlier set and generator state equal, pose within 1e-9;
  * frame_features on two seeded 1080p frames equals Akaze.extract_batch and the oracle's kps_descriptors."""
import ctypes as C

import numpy as np
import pytest

import cv_b200
from cv_b200 import CameraIntrinsics, CameraIntrinsicsK1Distortion
from cv_b200.checkpoint import features_to_bytes
from oracle import pyoracle as O
from oracle import pyoracle_sfm as OS
from tests.common import kitti_frame
from tests.synth import synth_frame, warp_frame

pytestmark = pytest.mark.gpu

VSLAM = (893.39010814, 898.32648616, 951.1310043, 555.13350077, 0.0, -0.28052513)      # vslam-sandbox/src/main.rs:71-78
TUTORIAL = (9.842439e+02, 9.808141e+02, 6.900000e+02, 2.331966e+02, 0.0, -3.728755e-01)  # tutorial chapter 5 main.rs:36-42


def _cam(fx, fy, cx, cy, skew, k1):
    return CameraIntrinsicsK1Distortion(CameraIntrinsics((fx, fy), (cx, cy), skew), k1)


def _bits(a):
    return np.ascontiguousarray(a, np.float64).view(np.uint64)


def _device_bearings(kpa, kpb, K, k1_entry=True):
    import torch
    from cv_b200._lib import KP_DTYPE
    from cv_b200.pair import Intrinsics, IntrinsicsK1, bind
    ctx = cv_b200.Context(0)
    bind(ctx.lib)
    dev = torch.device("cuda", 0)
    n = len(kpa)
    ka = torch.from_numpy(kpa.view(np.uint8).copy()).to(dev)
    kb = torch.from_numpy(kpb.view(np.uint8).copy()).to(dev)
    pairs = torch.from_numpy(np.repeat(np.arange(n, dtype=np.int32), 2)).to(dev)      # match i = (i, i)
    npairs = torch.tensor([n], dtype=torch.int32, device=dev)
    a = torch.zeros(n * 3, dtype=torch.float64, device=dev); b = torch.zeros(n * 3, dtype=torch.float64, device=dev)
    torch.cuda.synchronize()
    if k1_entry:
        k = IntrinsicsK1(*K)
        ctx.check(ctx.lib.cvb_pair_bearings_k1_dev(ctx.handle, ka.data_ptr(), kb.data_ptr(), pairs.data_ptr(), npairs.data_ptr(), n, C.byref(k),
                                                   a.data_ptr(), b.data_ptr()))
    else:
        k = Intrinsics(*K[:5])
        ctx.check(ctx.lib.cvb_pair_bearings_dev(ctx.handle, ka.data_ptr(), kb.data_ptr(), pairs.data_ptr(), npairs.data_ptr(), n, C.byref(k),
                                                a.data_ptr(), b.data_ptr()))
    ctx.sync()
    out = a.cpu().numpy().reshape(n, 3), b.cpu().numpy().reshape(n, 3)
    ctx.close()
    assert KP_DTYPE.itemsize == 28
    return out


def _random_keypoints(seed, n):
    from cv_b200._lib import KP_DTYPE
    rng = np.random.default_rng(seed)
    kp = np.zeros(n, KP_DTYPE)
    kp["x"] = rng.uniform(0, 1920, n).astype(np.float32); kp["y"] = rng.uniform(0, 1080, n).astype(np.float32)
    kp["x"][:4] = [0.0, 1919.0, 951.1310043, 0.5]; kp["y"][:4] = [0.0, 1079.0, 555.13350077, 1079.5]
    return kp


@pytest.mark.parametrize("K", [VSLAM, TUTORIAL], ids=["vslam_sandbox", "tutorial_ch5"])
def test_pair_bearings_k1_equals_oracle_bit_for_bit(K):
    kpa, kpb = _random_keypoints(1, 4099), _random_keypoints(2, 4099)
    a, b = _device_bearings(kpa, kpb, K)
    wa = np.array([OS.calibrate_k1(*K, float(k["x"]), float(k["y"])) for k in kpa])
    wb = np.array([OS.calibrate_k1(*K, float(k["x"]), float(k["y"])) for k in kpb])
    assert np.array_equal(_bits(a), _bits(wa)) and np.array_equal(_bits(b), _bits(wb))
    assert np.array_equal(_bits(a), _bits(_cam(*K).calibrate_keypoints(kpa)))


def test_pair_bearings_k1_zero_equals_the_undistorted_entry_bit_for_bit():
    kpa, kpb = _random_keypoints(3, 3000), _random_keypoints(4, 3000)
    K = VSLAM[:5] + (0.0,)
    a1, b1 = _device_bearings(kpa, kpb, K, k1_entry=True)
    a0, b0 = _device_bearings(kpa, kpb, K, k1_entry=False)
    assert np.array_equal(_bits(a1), _bits(a0)) and np.array_equal(_bits(b1), _bits(b0))
    wa = np.array([O.calibrate(*K[:5], float(k["x"]), float(k["y"])) for k in kpa])
    assert np.array_equal(_bits(a0), _bits(wa))


def _oracle_symmetric(d0, d1, better_by):
    oi, od = O.hamming_knn(d0, d1, 2)
    ri, rd = O.hamming_knn(d1, d0, 2)
    fwd = np.where(od[:, 0].astype(np.int64) + better_by <= od[:, 1], oi[:, 0].astype(np.int64), -1)
    rev = np.where(rd[:, 0].astype(np.int64) + better_by <= rd[:, 1], ri[:, 0].astype(np.int64), -1)
    return np.array([(i, j) for i, j in enumerate(fwd) if j >= 0 and rev[j] == i], np.int64).reshape(-1, 2)


def test_tutorial_chapter5_on_kitti_equals_the_oracle_pipeline():
    """Akaze::default(), symmetric matching with the tutorial's strict d0 + 24 < d1 (better_by = 25), the chapter-5 K1 camera,
    Arrsac::new(1e-7, Xoshiro256PlusPlus::seed_from_u64(0)) + EightPoint."""
    frames = np.stack([kitti_frame("0000000000"), kitti_frame("0000000014")])
    cam = _cam(*TUTORIAL)
    ars = cv_b200.Arrsac(1e-7, cv_b200.Xoshiro256PlusPlus(0))
    out = cv_b200.two_view_frames(cv_b200.Akaze(), frames, cam, ars, better_by=25)
    ok = [O.Akaze().extract(frames[f]) for f in range(2)]
    for f in range(2):
        assert out["keypoints"][f].tobytes() == ok[f][0].tobytes() and np.array_equal(out["descriptors"][f], ok[f][1])
    pairs = _oracle_symmetric(ok[0][1], ok[1][1], 25)
    assert np.array_equal(out["matches"], pairs) and len(pairs) > 8
    a = np.array([OS.calibrate_k1(*TUTORIAL, float(ok[0][0][i]["x"]), float(ok[0][0][i]["y"])) for i in pairs[:, 0]])
    b = np.array([OS.calibrate_k1(*TUTORIAL, float(ok[1][0][j]["x"]), float(ok[1][0][j]["y"])) for j in pairs[:, 1]])
    orng = O.rng_xoshiro(0)
    want = O.arrsac(O.arrsac_cfg(1e-7), 0, a, b, orng)
    assert (out["pose"] is None) == (want is None)
    assert [int(x) for x in ars.rng.state.s] == [int(x) for x in orng.s]
    if want is not None:
        assert np.array_equal(out["inliers"], want[2])
        assert np.allclose(out["pose"][0], want[0], rtol=0, atol=1e-9) and np.allclose(out["pose"][1], want[1], rtol=0, atol=1e-9)
        print(f"\ntutorial chapter 5 on KITTI: {len(pairs)} matches, {len(want[2])} inliers, "
              f"camera moved forward: {-out['pose'][1][2]!r}, right: {-out['pose'][1][0]!r}, down: {-out['pose'][1][1]!r}")
    # the same frames with the undistorted camera still take the k1 = 0 entry and give the bearings of CameraIntrinsics
    ars0 = cv_b200.Arrsac(1e-7, cv_b200.Xoshiro256PlusPlus(0))
    out0 = cv_b200.two_view_frames(cv_b200.Akaze(), frames, cam.simple_intrinsics, ars0, better_by=25)
    a0, b0 = cam.simple_intrinsics.calibrate_keypoints(ok[0][0][pairs[:, 0]]), cam.simple_intrinsics.calibrate_keypoints(ok[1][0][pairs[:, 1]])
    want0 = O.arrsac(O.arrsac_cfg(1e-7), 0, a0, b0, O.rng_xoshiro(0))
    assert (out0["pose"] is None) == (want0 is None)
    if want0 is not None:
        assert np.array_equal(out0["inliers"], want0[2])


def _rgb_frames(gray, seed):
    """seeded RGB8 frames whose channels differ: the luma texture, a seeded noise channel and the inverted texture"""
    rng = np.random.default_rng(seed)
    r = np.round(gray * 255).astype(np.uint8)
    g = rng.integers(0, 256, gray.shape, dtype=np.uint8)
    return np.ascontiguousarray(np.stack([r, g, 255 - r], -1))


def test_frame_features_equals_extract_batch_and_oracle():
    a = synth_frame(11)
    gray = np.stack([a, warp_frame(a, 1011)])
    rgb = _rgb_frames(gray, 12)
    cam = _cam(*VSLAM)
    ak = cv_b200.Akaze(maximum_features=5000)
    got = cv_b200.frame_features(ak, gray, rgb, cam)
    kps, descs = ak.extract_batch(gray)
    for f in range(2):
        g = got[f]
        assert len(g["keypoints"]) > 1000
        assert g["keypoints"].tobytes() == kps[f].tobytes() and np.array_equal(g["descriptors"], descs[f])
        assert np.all(np.diff(g["responses"]) <= 0)
        okp, odesc, obear, oresp, ocol = OS.kps_descriptors(O.Akaze(maximum_features=5000), gray[f], rgb[f], VSLAM)
        assert okp.tobytes() == g["keypoints"].tobytes() and np.array_equal(odesc, g["descriptors"])
        assert np.array_equal(_bits(g["bearings"]), _bits(obear))
        assert np.array_equal(g["colors"], ocol)
        assert len(np.unique(ocol[:, 0].astype(np.int32) - ocol[:, 1])) > 10
        assert features_to_bytes(g["bearings"], g["responses"], g["colors"]) == features_to_bytes(obear, oresp, ocol)


def test_frame_features_grayscale_rgb_is_replicated():
    a = synth_frame(13, h=270, w=480, nblobs=600)
    gray = a[None]
    luma8 = np.round(a * 255).astype(np.uint8)[None]
    ak = cv_b200.Akaze()
    got = cv_b200.frame_features(ak, gray, luma8, _cam(*TUTORIAL))[0]
    want = cv_b200.frame_features(ak, gray, np.repeat(luma8[..., None], 3, -1), _cam(*TUTORIAL))[0]
    assert len(got["colors"]) > 20 and np.array_equal(got["colors"], want["colors"])
    assert (got["colors"][:, 0] == got["colors"][:, 1]).all() and (got["colors"][:, 1] == got["colors"][:, 2]).all()

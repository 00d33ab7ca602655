"""GPU: AKAZE's staged surface (include/cvb200_stages.h) against the CPU oracle and against the one-call extractor.

- find_image_keypoints equals the oracle's refined stage byte for byte (two KITTI frames, a synthetic 1080p frame, a batch of 3);
- find, sorted by the extractor's rule (descending response, ties in index order) and truncated to maximum_features, then
  described, is byte-identical to extract, at batch 1 and 3;
- describe at caller keypoints equals the describe oracle (oracle/ref_stages.c) bit for bit: angles in [0, 2pi), [-pi, pi), degrees,
  1e6, 1e30, +-inf, NaN; NaN / inf coordinates; size 0, negative, NaN; an octave that disagrees with class_id; border keypoints;
  duplicates; an empty list; other descriptor configs on the same scale space;
- errors: invalid keypoints (CVB_EINVAL / flag 4), stale tickets, an image too small for one octave;
- the _dev entry points on torch tensors equal the host entry points."""
import ctypes as C

import numpy as np
import pytest

import cv_b200
from cv_b200._lib import CVB_EINVAL, KP_DTYPE, load_stages_library
from oracle import pyoracle as O
from oracle import pyoracle_stages as OS
from tests.common import kitti_frame
from tests.synth import synth_frame

pytestmark = pytest.mark.gpu

THR = 0.01


def _sorted_truncated(kps, max_features):
    order = np.lexsort((np.arange(len(kps)), -kps["response"].astype(np.float64)))
    out = kps[order]
    return out if max_features < 0 else out[:max_features]


@pytest.fixture(scope="module")
def frames():
    return {"k0": kitti_frame("0000000000"), "k14": kitti_frame("0000000014")}


@pytest.fixture(scope="module")
def oracles(frames):
    out = {}
    for name, img in frames.items():
        A = O.Akaze(detector_threshold=THR)
        A.extract(img)
        out[name] = A
    return out


@pytest.mark.parametrize("name", ["k0", "k14"])
def test_find_equals_oracle_refined_kitti(frames, oracles, name):
    ak = cv_b200.Akaze(THR)
    ss = ak.create_scale_space(frames[name])
    (got,) = ak.find_image_keypoints(ss)
    want = oracles[name].stage("refined")
    assert len(got) == len(want) > 100 and got.tobytes() == want.tobytes()
    ev = ss.evolutions
    assert len(ev) == oracles[name].num_evolutions()
    for i, e in enumerate(ev):
        info = oracles[name].evolution_info(i)
        assert (e["width"], e["height"], e["octave"], e["esigma"], e["n_fed_steps"]) == (info["w"], info["h"], info["octave"],
                                                                                      info["esigma"], len(info["tau"]))
    # EvolutionStep::new (evolution.rs:46-58): etime = 0.5 * esigma^2, sigma_size = esigma.round() (half away from zero),
    # sublevel counts up from 0 inside each octave
    sub = [0]
    for i in range(1, len(ev)):
        sub.append(sub[-1] + 1 if ev["octave"][i] == ev["octave"][i - 1] else 0)
    assert list(ev["sublevel"]) == sub
    assert np.array_equal(ev["etime"], 0.5 * (ev["esigma"] * ev["esigma"]))
    assert np.array_equal(ev["sigma_size"], np.floor(ev["esigma"] + 0.5).astype(np.uint32))
    assert list(ev["sigma_size"][:4]) == [2, 2, 2, 3]   # Akaze::default(): esigma 1.6, 1.90, 2.26, 2.69
    (again,) = ak.find_image_keypoints(ss)   # detection runs again on the same planes: the same keypoints
    assert again.tobytes() == got.tobytes()


def test_find_rejects_another_detector_config(frames):
    ss = cv_b200.Akaze(THR).create_scale_space(frames["k0"])
    with pytest.raises(ValueError, match="detector config"):
        cv_b200.Akaze(0.001).find_image_keypoints(ss)
    with pytest.raises(ValueError, match="detector config"):
        cv_b200.Akaze(THR, derivative_factor=2.0).find_image_keypoints(ss)
    (a,) = cv_b200.Akaze(THR, maximum_features=5, descriptor_channels=1).find_image_keypoints(ss)
    (b,) = cv_b200.Akaze(THR).find_image_keypoints(ss)
    assert len(a) > 5 and a.tobytes() == b.tobytes()


def test_find_equals_oracle_refined_synthetic_1080p():
    img = synth_frame(5)
    ak = cv_b200.Akaze(0.001)
    (got,) = ak.find_image_keypoints(ak.create_scale_space(img))
    A = O.Akaze(detector_threshold=0.001)
    A.extract(img)
    want = A.stage("refined")
    assert len(got) == len(want) > 1000 and got.tobytes() == want.tobytes()


def test_find_batch_of_three_equals_single_frames(frames, oracles):
    imgs = np.stack([frames["k0"], frames["k14"], frames["k0"][::-1].copy()])
    ak = cv_b200.Akaze(THR)
    got = ak.find_image_keypoints(ak.create_scale_space(imgs))
    A = O.Akaze(detector_threshold=THR)
    A.extract(imgs[2])
    for g, w in zip(got, [oracles["k0"].stage("refined"), oracles["k14"].stage("refined"), A.stage("refined")]):
        assert g.tobytes() == w.tobytes()


@pytest.mark.parametrize("max_features", [-1, 150])
@pytest.mark.parametrize("batch", [1, 3])
def test_find_sort_describe_equals_extract(frames, batch, max_features):
    imgs = np.stack([frames["k0"], frames["k14"], synth_frame(2, *frames["k0"].shape)][:batch])
    ak = cv_b200.Akaze(THR, maximum_features=max_features)
    ss = ak.create_scale_space(imgs)
    found = ak.find_image_keypoints(ss)
    sel = [_sorted_truncated(k, max_features) for k in found]
    kps, descs = ak.extract_descriptors(ss, sel)
    ekps, edescs = ak.extract_batch(imgs)
    for b in range(batch):
        assert kps[b].tobytes() == ekps[b].tobytes() and np.array_equal(descs[b], edescs[b]), b
        assert len(kps[b]) > (50 if b < 2 else 0)   # the KITTI frames; the synthetic one has few keypoints at 0.01


def _caller_keypoints(kps, E, rng, W, H):
    base = kps[np.argsort(-kps["size"], kind="stable")[:40]]
    out = [base]
    for lo, hi in ((0, 2 * np.pi), (-np.pi, np.pi), (0, 360)):
        k = base.copy()
        k["angle"] = rng.uniform(lo, hi, len(k)).astype(np.float32)
        out.append(k)
    for a in (1e6, -1e6, 1e30, np.inf, -np.inf, np.nan, 120.0, 119.99999):
        k = base[:6].copy()
        k["angle"] = a
        out.append(k)
    for field, v in (("x", np.nan), ("y", np.nan), ("x", np.inf), ("y", -np.inf), ("x", -1e30), ("size", 0.0), ("size", -20.0),
                     ("size", np.nan)):
        k = base[:4].copy()
        k[field] = v
        out.append(k)
    k = base[:8].copy()   # octave disagreeing with class_id (still valid)
    k["octave"] = (k["octave"] + 1) % 4
    out.append(k)
    k = base[:8].copy()
    k["class_id"] = (k["class_id"] + 3) % E
    out.append(k)
    border = np.zeros(12, KP_DTYPE)
    border["x"] = [0, W - 1, 0, W - 1, 60, 60, W - 61, 5.5, 30, 30, 29.4, 29.6]
    border["y"] = [0, 0, H - 1, H - 1, 30, 29, 30, 200, H - 31, H - 30, 100, 100]
    border["size"] = 4.8
    border["angle"] = 0.0
    out.append(border)
    ties = np.zeros(6, KP_DTYPE)   # angle 0 and integer scales: sample positions at exact .5 ties (rounded away from zero)
    ties["x"] = [100.5, 101.5, 200.5, 300.0, 64.5, 65.5]
    ties["y"] = [80.5, 81.5, 120.0, 150.5, 90.5, 91.5]
    ties["size"] = [5.0, 5.0, 7.0, 6.0, 4.0, 9.0]   # 0.5 * size: 2.5 and 3.5 are ties of the scale itself
    out.append(ties)
    out.append(base[:5])   # duplicates of the first keypoints
    out.append(base[:5])
    return np.concatenate(out)


def test_caller_keypoints_equal_the_oracle(frames, oracles):
    rng = np.random.default_rng(11)
    ak = cv_b200.Akaze(THR)
    ss = ak.create_scale_space(frames["k0"])
    kps = _caller_keypoints(oracles["k0"].stage("refined"), len(ss.evolutions), rng, ss.width, ss.height)
    (gk,), (gd,) = ak.extract_descriptors(ss, kps)
    ok, od = OS.describe(oracles["k0"], kps)
    assert len(gk) == len(ok) and gk.tobytes() == ok.tobytes() and np.array_equal(gd, od)
    assert 0 < len(ok) < len(kps)   # some dropped, some kept
    assert np.isnan(gk["x"]).any() and np.isnan(gk["angle"]).any()
    (ek,), (ed,) = ak.extract_descriptors(ss, kps[:0])
    assert len(ek) == 0 and ed.shape == (0, 64)


@pytest.mark.parametrize("channels,pattern", [(1, 10), (2, 10), (3, 6), (2, 7)])
def test_other_descriptor_configs_on_the_same_scale_space(frames, oracles, channels, pattern):
    ak = cv_b200.Akaze(THR)
    ss = ak.create_scale_space(frames["k14"])
    (found,) = ak.find_image_keypoints(ss)
    other = cv_b200.Akaze(THR, descriptor_channels=channels, descriptor_pattern_size=pattern)
    (gk,), (gd,) = other.extract_descriptors(ss, found)
    ok, od = OS.describe(oracles["k14"], found, channels, pattern)
    assert len(gk) > 50 and gk.tobytes() == ok.tobytes() and np.array_equal(gd, od)
    (gk2,), (gd2,) = ak.extract_descriptors(ss, found)   # the ticket is still valid and the default tables untouched
    ok2, od2 = OS.describe(oracles["k14"], found)
    assert gk2.tobytes() == ok2.tobytes() and np.array_equal(gd2, od2)


def test_invalid_keypoints_are_rejected(frames):
    ak = cv_b200.Akaze(THR)
    ss = ak.create_scale_space(frames["k0"])
    (found,) = ak.find_image_keypoints(ss)
    E = len(ss.evolutions)
    for field, v, idx in (("class_id", E, 3), ("octave", 32, 5)):
        bad = found[:10].copy()
        bad[field][idx] = v
        with pytest.raises(cv_b200.CvbError) as e:
            ak.extract_descriptors(ss, bad)
        assert e.value.code == CVB_EINVAL and f"keypoint {idx}" in str(e.value)
    ak.extract_descriptors(ss, found[:10])   # the ticket survives a rejected call


def test_stale_ticket_is_rejected(frames):
    ak = cv_b200.Akaze(THR)
    ss = ak.create_scale_space(frames["k0"])
    (found,) = ak.find_image_keypoints(ss)
    ak.extract(frames["k14"])
    for call in (lambda: ak.find_image_keypoints(ss), lambda: ak.extract_descriptors(ss, found)):
        with pytest.raises(cv_b200.CvbError) as e:
            call()
        assert e.value.code == CVB_EINVAL and "scale space replaced" in str(e.value)
    ss2 = ak.create_scale_space(frames["k14"])
    with pytest.raises(cv_b200.CvbError):
        ak.find_image_keypoints(ss)
    ak.find_image_keypoints(ss2)
    ak.create_scale_space(frames["k14"][:200, :300].copy())   # another size rebuilds the workspace
    with pytest.raises(cv_b200.CvbError):
        ak.find_image_keypoints(ss2)


def test_image_too_small_for_one_octave():
    ak = cv_b200.Akaze(THR)
    ss = ak.create_scale_space(np.random.default_rng(0).random((30, 50), dtype=np.float32))
    assert len(ss.evolutions) == 0
    (found,) = ak.find_image_keypoints(ss)
    assert len(found) == 0
    kp = np.zeros(1, KP_DTYPE)
    kp["x"], kp["y"] = 10, 10
    with pytest.raises(cv_b200.CvbError) as e:
        ak.extract_descriptors(ss, kp)
    assert e.value.code == CVB_EINVAL
    (k,), (d,) = ak.extract_descriptors(ss, kp[:0])
    assert len(k) == 0


def _tensor(a, dev):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a).view(np.uint8).reshape(-1).copy()).to(dev)


def test_dev_entry_points_equal_host_entry_points(frames):
    import torch
    dev = torch.device("cuda", 0)
    ctx = cv_b200.Context(0)
    L = load_stages_library()
    ak = cv_b200.Akaze(THR, ctx=ctx)
    imgs = np.stack([frames["k0"], frames["k14"]])
    cfg = ak.config.to_c()
    ss = ak.create_scale_space(imgs)
    host_found = ak.find_image_keypoints(ss)
    t = C.c_uint64()
    timg = torch.from_numpy(imgs).to(dev)
    ctx.check(L.cvb_akaze_scale_space_dev(ctx.handle, C.byref(cfg), timg.data_ptr(), 2, imgs.shape[2], imgs.shape[1], C.byref(t)))
    assert t.value != ss.ticket
    cap = 4096
    kp = torch.zeros(2 * cap * KP_DTYPE.itemsize, dtype=torch.uint8, device=dev)
    n = torch.zeros(2, dtype=torch.int32, device=dev)
    ctx.check(L.cvb_akaze_find_image_keypoints_dev(ctx.handle, t.value, kp.data_ptr(), cap, n.data_ptr()))
    ctx.sync()
    kp_h = kp.cpu().numpy().view(KP_DTYPE).reshape(2, cap)
    n_h = n.cpu().numpy()
    for b in range(2):
        assert kp_h[b, :n_h[b]].tobytes() == host_found[b].tobytes()
    # describe: caller keypoints with two invalid ones -> dropped, flag 4; the rest equal the host call
    rng = np.random.default_rng(3)
    per = [_caller_keypoints(host_found[0], len(ss.evolutions), rng, ss.width, ss.height), host_found[1][:300].copy()]
    per[1]["angle"][::7] = 1e30
    ss_host = ak.create_scale_space(imgs)
    hk, hd = ak.extract_descriptors(ss_host, per)
    ctx.check(L.cvb_akaze_scale_space_dev(ctx.handle, C.byref(cfg), timg.data_ptr(), 2, imgs.shape[2], imgs.shape[1], C.byref(t)))
    flag = C.c_uint32()
    ctx.check(ctx.lib.cvb_akaze_dev_overflow(ctx.handle, C.byref(flag)))
    bad = per[1].copy()
    bad["class_id"][4] = 99
    bad["octave"][9] = 40
    allk = np.concatenate([per[0], bad])
    offs = np.array([0, len(per[0]), len(allk)], np.uint32)
    total = len(allk) + 17
    kin = _tensor(allk, dev)
    toffs = torch.from_numpy(offs.view(np.int32)).to(dev)
    kout = torch.zeros(total * KP_DTYPE.itemsize, dtype=torch.uint8, device=dev)
    dout = torch.zeros(total * 64, dtype=torch.uint8, device=dev)
    nout = torch.zeros(2, dtype=torch.int32, device=dev)
    ctx.check(L.cvb_akaze_extract_descriptors_dev(ctx.handle, C.byref(cfg), t.value, kin.data_ptr(), toffs.data_ptr(), total,
                                                  kout.data_ptr(), dout.data_ptr(), nout.data_ptr()))
    ctx.check(ctx.lib.cvb_akaze_dev_overflow(ctx.handle, C.byref(flag)))
    assert flag.value == 4
    ko = kout.cpu().numpy().view(KP_DTYPE)
    do = dout.cpu().numpy().reshape(-1, 64)
    no = nout.cpu().numpy()
    assert no[0] == len(hk[0]) and ko[:no[0]].tobytes() == hk[0].tobytes() and np.array_equal(do[:no[0]], hd[0])
    keep = np.ones(len(per[1]), bool)
    keep[[4, 9]] = False
    wk, wd = ak.extract_descriptors(ak.create_scale_space(imgs), [per[0], per[1][keep]])
    o1 = offs[1]
    assert no[1] == len(wk[1]) and ko[o1:o1 + no[1]].tobytes() == wk[1].tobytes() and np.array_equal(do[o1:o1 + no[1]], wd[1])

"""CPU-only: the oracle of include/cvb200_try_init.h (oracle/ref_try_init.c) against a short numpy restatement of add_reconstruction,
and cvb_try_init_check's refusals of every malformed list, with the init oracle's own outputs accepted."""
import numpy as np
import pytest

from cv_b200._lib import CVB_EINVAL
from cv_b200.try_init import check_try_init
from oracle import pyoracle_init as OI
from oracle import pyoracle_try_init as OT
from tests.init_scenes import init_scene
from tests.try_init_scenes import frame_store, random_lists


def _numpy_add_reconstruction(n, comb, fm, sm):
    """view_landmarks, landmark_offsets, observations by the definition in the header"""
    nc, n1, n2 = n
    maps = [{int(f): int(c) for c, f in fm} | {int(c[1]): int(c[0]) for c in comb},
            {int(s): int(c) for c, s in sm} | {int(c[2]): int(c[0]) for c in comb}]
    obs = [[(0, c)] for c in range(nc)]
    vl = list(range(nc))
    for v, nv in ((1, n1), (2, n2)):
        for j in range(nv):
            c = maps[v - 1].get(j)
            if c is None:
                obs.append([(v, j)])
                vl.append(len(obs) - 1)
            else:
                obs[c].append((v, j))
                vl.append(c)
    lo = np.cumsum([0] + [len(o) for o in obs]).astype(np.uint32)
    return np.array(vl, np.uint32), lo, np.array([x for o in obs for x in o], np.uint32).reshape(-1, 2)


@pytest.mark.parametrize("case", ["random", "empty_lists", "zero_first", "zero_second", "all_common"])
@pytest.mark.parametrize("seed", [0, 1])
def test_oracle_equals_the_numpy_restatement(case, seed):
    rng = np.random.default_rng(seed)
    cap = 512
    n = {"random": (301, 457, 233), "empty_lists": (200, 150, 99), "zero_first": (300, 0, 177), "zero_second": (250, 211, 0),
         "all_common": (100, 100, 100)}[case]
    k, k1, k2 = {"random": (80, 60, 50), "empty_lists": (0, 0, 0), "zero_first": (0, 0, 90), "zero_second": (0, 70, 0),
                 "all_common": (100, 0, 0)}[case]
    comb, fm, sm = random_lists(rng, *n, k, k1, k2)
    st = frame_store(rng, [n[1], 7, n[0], n[2]], cap)
    fp, sp = rng.normal(size=12), rng.normal(size=12)
    s = OT.add_reconstruction(st["descriptors"], st["counts"], st["bearings"], st["colors"], 2, 0, 3, fp, sp, comb, fm, sm)
    vl, lo, obs = _numpy_add_reconstruction(n, comb, fm, sm)
    assert np.array_equal(s["view_landmarks"], vl) and np.array_equal(s["landmark_offsets"], lo) and np.array_equal(s["observations"], obs)
    assert list(s["view_offsets"]) == [0, n[0], n[0] + n[1], sum(n)]
    assert len(lo) - 1 == sum(n) - len(comb) * 2 - len(fm) - len(sm) and len(obs) == sum(n)
    assert np.array_equal(s["bearings"], np.concatenate([st["bearings"][2, :n[0]], st["bearings"][0, :n[1]], st["bearings"][3, :n[2]]]))
    assert np.array_equal(s["descriptors"][n[0]:n[0] + n[1]], st["descriptors"][0, :n[1]])
    assert np.array_equal(s["colors"][n[0] + n[1]:], st["colors"][3, :n[2]])
    assert s["poses"][1].tobytes() == fp.tobytes() and s["poses"][0].tobytes() == np.concatenate([np.eye(3).ravel(), np.zeros(3)]).tobytes()
    c = s["constraints"][0]
    assert list(c["views"]) == [0, 1, 2] and c["landmarks"] == 0 and c["poses"][1]["t"].tobytes() == sp[9:].tobytes()
    assert check_try_init(*n, comb, fm, sm) == 0


def test_check_refuses_every_malformed_list():
    rng = np.random.default_rng(3)
    n = (50, 40, 30)
    comb, fm, sm = random_lists(rng, *n, 10, 8, 6)
    assert check_try_init(*n, comb, fm, sm) == 0
    bad = []
    for lst, col, lim in ((comb, 0, n[0]), (comb, 1, n[1]), (comb, 2, n[2]), (fm, 0, n[0]), (fm, 1, n[1]), (sm, 0, n[0]), (sm, 1, n[2])):
        b = lst.copy()
        b[0, col] = lim                                            # out of range of its frame's count
        bad.append((b, lst))
    for b, lst in bad:
        args = [b if x is lst else x for x in (comb, fm, sm)]
        assert check_try_init(*n, *args) == CVB_EINVAL
    f2 = fm.copy(); f2[1, 1] = fm[0, 1]                            # a first feature twice in first_matches
    assert check_try_init(*n, comb, f2, sm) == CVB_EINVAL
    f3 = fm.copy(); f3[0, 1] = comb[0, 1]                          # ... across first_matches and combined
    assert check_try_init(*n, comb, f3, sm) == CVB_EINVAL
    f4 = fm.copy(); f4[0, 0] = comb[0, 0]                          # a common center mapped twice into the first view
    assert check_try_init(*n, comb, f4, sm) == CVB_EINVAL
    f5 = fm.copy(); f5[1, 0] = fm[0, 0]                            # a center twice within first_matches
    assert check_try_init(*n, comb, f5, sm) == CVB_EINVAL
    s2 = sm.copy(); s2[1, 1] = sm[0, 1]                            # the same for the second view
    assert check_try_init(*n, comb, fm, s2) == CVB_EINVAL
    s3 = sm.copy(); s3[0, 1] = comb[0, 2]
    assert check_try_init(*n, comb, fm, s3) == CVB_EINVAL
    s4 = sm.copy(); s4[0, 0] = comb[0, 0]
    assert check_try_init(*n, comb, fm, s4) == CVB_EINVAL
    c2 = comb.copy(); c2[1, 0] = comb[0, 0]                        # a center twice within combined
    assert check_try_init(*n, c2, fm, sm) == CVB_EINVAL
    for frames in ((0, 0, 1), (0, 1, 1), (1, 0, 1)):               # two equal frames
        assert check_try_init(*n, comb, fm, sm, frames=frames) == CVB_EINVAL
    with pytest.raises(ValueError):
        OT.add_reconstruction(np.zeros((3, 64, 64), np.uint8), np.array(n), np.zeros((3, 64, 3)), None, 0, 1, 2, np.zeros(12), np.zeros(12),
                              comb, bad[3][0], sm)


@pytest.mark.parametrize("seed", [0, 1])
def test_check_accepts_the_init_oracles_lists(seed):
    sc = init_scene(np.random.default_rng(100 + seed), 4, noise=1e-4, outliers=0.1)
    F, cap = len(sc["options"]), sc["bearings"].shape[1]
    arrs = OI.options_from_matches(F, cap, sc["matches"], sc["poses"])
    w = OI.init_reconstruction(sc["bearings"], 0, sc["options"], *arrs, OI.InitCfg(three_view_patience=0))
    r = w["result"]
    assert r["status"] == OI.ACCEPTED
    n = len(sc["points"])
    assert check_try_init(n, n, n, w["combined"], w["first_matches"], w["second_matches"],
                          frames=(0, sc["options"][r["first"]], sc["options"][r["second"]])) == 0

"""ccm_search_and_fuse_host — the searches of LoopFinder / MapMerger::SearchAndFuse for every corrected keyframe in one call — against
the flat oracle (oracle/pysf.py), the golden fixture and, where it is built, the reference's own ORBmatcher::Fuse(Scw).  No device
needed."""
import copy
import ctypes as C
import os

import numpy as np
import pytest

from ccm_slam_b200 import api
from ccm_slam_b200 import synth_match as sm
from oracle import pyoracle, pysf

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "search_and_fuse.npz")


def _check(sc):
    best, settled = api.search_and_fuse(sc, host=True)
    assert np.array_equal(best, pysf.oracle(sc))
    return best, settled


def _golden(name):
    z = np.load(GOLDEN)
    sub = {k[len(name) + 1:]: z[k] for k in z.files if k.startswith(name + "_")}
    return sm.search_and_fuse_scene_from_arrays(_Npz(sub)), z[name + "_best"]


class _Npz(dict):
    @property
    def files(self):
        return list(self.keys())


@pytest.mark.parametrize("kind,seed", [("loop", 0), ("loop", 1), ("merge", 2), ("merge", 3)])
def test_host_equals_oracle(kind, seed):
    sc = sm.make_search_and_fuse_scene(kind, n_kf=5, n=400, seed=seed)
    best, settled = _check(sc)
    assert (best >= 0).sum() > 300
    assert settled > 0                                        # PredictScale boundary pairs were reached and settled with logf
    skip = sc["points"]["skip"].astype(bool)
    assert skip.any() and (best[:, skip] == -1).all()         # isBad() on entry is never searched
    dnr = sc["points"]["dnr"].astype(bool)
    assert (best[:, dnr] >= 0).any()                          # mbDoNotReplace is searched (the reference comments the test out)


def test_merge_scale_is_not_one():
    sc = sm.make_search_and_fuse_scene("merge", n_kf=3, n=200, seed=4)
    s = [np.sqrt((np.asarray(k["Scw"], np.float64)[0, :3] ** 2).sum()) for k in sc["kfs"]]
    assert all(abs(x - 1) > 0.05 for x in s)


def test_two_loop_points_claim_one_keypoint():
    sc = sm.make_search_and_fuse_scene("loop", n_kf=4, n=400, seed=5)
    best, _ = _check(sc)
    w = sc["points"]["world"]
    hit = False
    for k in range(best.shape[0]):
        got = best[k] >= 0
        _, cnt = np.unique(np.stack([w[got], best[k][got]]), axis=1, return_counts=True)
        hit |= (cnt > 1).any()
    assert hit


@pytest.mark.parametrize("name", ["loop", "merge"])
def test_golden_fixture(name):
    sc, want = _golden(name)
    best, _ = _check(sc)
    assert np.array_equal(best, want)


@pytest.mark.parametrize("variant", ["th3", "chi2", "skip_dnr", "pose_camera"])
def test_wrong_variants_fail_the_fixture(variant):
    """each plausible misreading of Fuse(Scw) changes at least one result of the fixture"""
    for name in ("loop", "merge"):
        sc, want = _golden(name)
        if variant == "th3":
            got = pysf.oracle(sc, th=3.0)
        elif variant == "chi2":
            got = pysf.oracle(sc, chi2=True)
        elif variant == "skip_dnr":
            sc["points"]["skip_dnr"] = sc["points"]["skip"] | sc["points"]["dnr"]
            got = pysf.oracle(sc, skip="skip_dnr")
        else:
            got = pysf.oracle(sc, camera="pose")
        if not np.array_equal(got, want):
            return
    pytest.fail("variant %s reproduces the fixture" % variant)


@pytest.mark.parametrize("kind,seed", [("loop", 6), ("merge", 7)])
def test_oracle_equals_reference_fuse_scw(kind, seed):
    """the flat oracle against the reference's own ORBmatcher::Fuse(pKF, Scw, vpPoints, 4, vpReplacePoint), keyframe by keyframe; the
    reference splits the f32 Scw itself"""
    if pyoracle.ref_match() is None:
        pytest.skip("the reference's ORBmatcher is not built here (oracle/_ref)")
    from tests.golden.make_search_and_fuse_golden import reference
    sc = sm.make_search_and_fuse_scene(kind, n_kf=4, n=300, seed=seed, boundary=60)
    ref = reference(sc)
    assert (ref >= 0).sum() > 200 and np.array_equal(pysf.oracle(sc), ref)


def test_split_differs_from_the_pose():
    """the split of Scw and the keyframe's [R t/s] pose differ in rounding somewhere, so the choice of camera is observable"""
    sc = sm.make_search_and_fuse_scene("merge", n_kf=6, n=100, seed=8)
    assert any(not np.array_equal(k["Tcw"], k["Tcw_pose"]) or not np.array_equal(k["Ow"], k["Ow_pose"]) for k in sc["kfs"])


def test_empty():
    sc = sm.make_search_and_fuse_scene("loop", n_kf=2, n=200, seed=9)
    e = dict(sc, kfs=[])
    best, settled = _check(e)
    assert best.shape == (0, len(sc["points"]["skip"])) and settled == 0
    e = copy.deepcopy(sc)
    e["points"] = {k: v[:0] for k, v in sc["points"].items()}
    best, settled = _check(e)
    assert best.shape == (2, 0) and settled == 0
    e = copy.deepcopy(sc)
    e["points"]["skip"][:] = 1
    best, _ = _check(e)
    assert (best == -1).all()


def _refused(sc, mutate, msg):
    keep = []
    kfs, K, pts = api.search_and_fuse_structs(sc, keep)
    best = np.full((max(K, 1), max(pts.n, 1)), -3, np.int32)
    settled = C.c_int32(-7)
    args = dict(kfs=kfs, K=K, pts=C.byref(pts), best=api._p(best))
    mutate(args, kfs, pts)
    L = api.lib()
    for fn in (L.ccm_search_and_fuse_host, L.ccm_search_and_fuse):
        assert fn(args["kfs"], args["K"], args["pts"], args["best"], C.byref(settled)) == -1
        assert msg in L.ccm_last_error().decode()
        assert (best == -3).all() and settled.value == -7           # nothing written


def test_refusals_write_nothing():
    sc = sm.make_search_and_fuse_scene("merge", n_kf=3, n=200, seed=10, boundary=0)

    def null_kfs(a, kfs, pts): a["kfs"] = None
    def null_best(a, kfs, pts): a["best"] = None
    def null_desc(a, kfs, pts): pts.desc = None
    def null_sf(a, kfs, pts): kfs[1].scale_factors = None
    def big_grid(a, kfs, pts): kfs[2].grid.grid_cols = 20000; kfs[2].grid.grid_rows = 1
    def too_many(a, kfs, pts): pts.n = 1 << 29
    _refused(sc, null_kfs, "null keyframe array")
    _refused(sc, null_best, "null output array")
    _refused(sc, null_desc, "null point array")
    _refused(sc, null_sf, "keyframe 1: null or empty scale pyramid")
    _refused(sc, big_grid, "keyframe 2: too many keypoints for the 20-bit visiting position")
    _refused(sc, too_many, "pairs (each keyframe's points padded to a multiple of 32)")


def test_inv_level_sigma2_is_not_read():
    sc = sm.make_search_and_fuse_scene("loop", n_kf=2, n=200, seed=11)
    keep = []
    kfs, K, pts = api.search_and_fuse_structs(sc, keep)
    for k in range(K):
        kfs[k].inv_level_sigma2 = None
    best = np.full((K, pts.n), -3, np.int32)
    assert api.lib().ccm_search_and_fuse_host(kfs, K, C.byref(pts), api._p(best), None) == 0
    assert np.array_equal(best, pysf.oracle(sc))

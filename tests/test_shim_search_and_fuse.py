"""shim/SearchAndFuse_shim.cpp (cslam::ccm_b200_search_and_fuse) against a literal restatement of LoopFinder::SearchAndFuse and
MapMerger::SearchAndFuse, Fuse(Scw), Replace and ReplaceAndLock (oracle/ref_search_and_fuse_wrap.cpp), member for member on stand-in
keyframes and points, at both sites.  The device entry point is answered by the host entry point here (oracle/ccm_search_and_fuse_double.cpp)."""
import numpy as np
import pytest

from ccm_slam_b200 import synth_match as sm
from oracle import pysf


def scene(kind, seed):
    return sm.make_search_and_fuse_scene(kind, n_kf=6, n=300, n_loop=900, seed=seed, held_frac=0.5, occupied_frac=0.3, dup=120)


def run_both(sc, merge, gpu=False, empty_kf=()):
    a = pysf.StandIn(sc, gpu=gpu, empty_kf=empty_kf)
    b = pysf.StandIn(sc, gpu=gpu, empty_kf=empty_kf)
    try:
        a.run(0, merge)
        s0 = b.stats()
        b.run(1, merge)
        return a.members(), b.members(), b.stats() - s0
    finally:
        a.close(); b.close()


def same_members(ref, shim):
    for k in ref:
        assert np.array_equal(ref[k], shim[k]), k


@pytest.mark.parametrize("kind,merge,seed", [("loop", False, 0), ("loop", False, 1), ("merge", True, 2), ("merge", True, 3)])
def test_shim_equals_restatement(kind, merge, seed):
    sc = scene(kind, seed)
    ref, shim, stats = run_both(sc, merge)
    same_members(ref, shim)
    assert stats[0] == 1                                      # one library call for the whole member
    assert stats[1] > 0                                       # points whose descriptor an earlier replacement changed were searched again
    log = bytes(ref["log"]).decode()
    assert ("L" if merge else "R") in log or "l" in log       # replacements happened, with the site's lock flag
    assert ("l" in log) == merge and ("R" in log) != merge
    P0 = len(sc["points"]["skip"])
    held = {int(r) for sl in sc["kf_slot"] for r in sl if r >= 0}
    turned_bad = [r for r in held if ref["bad"][r] and not sc["points"]["skip"][r]]
    assert turned_bad                                         # a loop point some keyframe held was replaced mid-walk
    assert (ref["bad"][P0:] == 1).any()                       # occupants merged into loop points


def test_empty_keyframe_is_skipped_by_replace_and_lock():
    sc = scene("merge", 4)
    ref, shim, _ = run_both(sc, True, empty_kf=(1, 3))
    same_members(ref, shim)


def test_no_keyframes():
    sc = scene("loop", 5)
    ref, shim, stats = run_both(dict(sc, kfs=[], kf_slot=[]), False)
    same_members(ref, shim)
    assert stats[0] == 1 and stats[1] == 0 and not ref["bad"][sc["points"]["skip"] == 0].any()

"""shim/FuseNeighbours_shim.cpp (LocalMapping::SearchInNeighbors over one ccm_fuse_neighbours call) against a literal restatement of
the member, of ORBmatcher::Fuse and of MapPoint::Replace (oracle/ref_fuse_neighbours_wrap.cpp), member for member on stand-in objects:
every keyframe's mvpMapPoints, each point's observations in map order, bad flag, mpReplaced, descriptor, fuse-candidate mark and the
order of the members called on it, each keyframe's fuse-target mark and UpdateConnections calls.  The device entry point is answered
by the host entry point here; tests/test_gpu_fuse_neighbours.py runs the same over the real library."""
import numpy as np
import pytest

from ccm_slam_b200 import synth_match as sm
from oracle import pyfn


def run_both(sc, gpu=False):
    out, stats = [], None
    for mode in (0, 1):
        s = pyfn.StandIn(sc, gpu=gpu)
        before = s.stats()
        s.run(mode)
        out.append(s.members())
        if mode == 1:
            stats = s.stats() - before
        s.close()
    return out[0], out[1], stats


def same_members(a, b):
    for k in ("mvp", "bad", "replaced", "desc", "cand_mark", "obs_ptr", "obs", "log_ptr", "log", "target_mark", "conn_updates"):
        assert a[k].tobytes() == b[k].tobytes(), k


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_shim_equals_restatement(seed):
    sc = sm.make_fuse_scene(n_first=6, n_second=3, n=400, seed=seed)
    ref, shim, stats = run_both(sc)
    same_members(ref, shim)
    log = bytes(ref["log"]).decode()
    assert stats[0] == 1                    # one library call
    assert stats[1] >= 1                    # at least one pair searched again because Replace changed its point's descriptor
    assert "i" in log                       # Replace's id-mismatch branch, through the third keyframe
    assert log.count("r") > 20 and (ref["replaced"] >= 0).sum() > 20
    assert (ref["conn_updates"][0] == 1)

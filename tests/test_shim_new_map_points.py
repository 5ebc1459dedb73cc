"""shim/NewMapPoints_shim.cpp (LocalMapping::CreateNewMapPoints over one ccm_new_map_points call) against a literal restatement of
the reference body (oracle/ref_new_points_wrap.cpp), member for member on stand-in objects: mvpMapPoints of every keyframe, each new
point's position, reference keyframe, observations and the order of the members called on it, the map's point list and the
recent-points list — with neighbours skipped for their baseline, and with CheckNewKeyFrames() ending the member early at every poll.
The device entry point is doubled by the oracle here; tests/test_gpu_new_map_points.py runs the same over the real library."""
import numpy as np
import pytest

from ccm_slam_b200 import synth_match as sm
from oracle import pynp

N_NB = 7


def scene():
    return sm.make_new_points_scene(n_nb=N_NB, n=400, seed=71, zero_baseline_nb=4)


def run_both(force_at_poll, median_depth, gpu=False, sc=None):
    sc = sc or scene()
    out = []
    for mode in (0, 1):
        s = pynp.StandIn(sc["cur"], sc["neighbours"], median_depth, gpu=gpu)
        s.run(mode, force_at_poll)
        out.append(s.members())
        s.close()
    return out


def same_members(a, b):
    assert a["polls"] == b["polls"]
    for k in ("mvp", "pos", "ref", "obs", "log", "recent"):
        assert a[k].tobytes() == b[k].tobytes(), k


def skip_two():
    md = np.ones(N_NB + 1, np.float32)
    md[[2, 6]] = 1e4          # ratioBaselineDepth < 0.01: neighbours 1 and 5 (keyframes 2 and 6) are not searched
    return md


def check(lit, shim, expect_polls):
    same_members(lit, shim)
    P = len(lit["pos"])
    assert lit["polls"] == expect_polls
    assert (lit["log"][:, :5] == np.frombuffer(b"oodnm", np.uint8)).all() and (lit["log"][:, 5:] == 0).all()
    assert np.array_equal(lit["recent"], np.arange(P)) and (lit["ref"] == 0).all() and (lit["obs"][:, 0] == 0).all()
    return P


def test_the_whole_member(gpu=False):
    lit, shim = run_both(-1, None, gpu)
    assert check(lit, shim, N_NB - 1) > 100
    assert (lit["obs"][:, 2] >= 1).all() and (np.diff(lit["obs"][:, 2]) >= 0).all()      # neighbour by neighbour


def test_neighbours_skipped_for_their_baseline(gpu=False):
    lit, shim = run_both(-1, skip_two(), gpu)
    P = check(lit, shim, N_NB - 1)
    assert P > 50 and not np.isin(lit["obs"][:, 2], [2, 6]).any() and np.isin(3, lit["obs"][:, 2])
    full = run_both(-1, None, gpu)[0]
    assert P != len(full["pos"])                                                           # the skip changes the result


@pytest.mark.parametrize("poll", range(1, N_NB))
def test_an_early_return_keeps_the_reference_prefix(poll, gpu=False):
    # the poll before neighbour `poll` answers true: neighbours 0 .. poll-1 were applied, skipped ones included in the count of polls
    lit, shim = run_both(poll, skip_two(), gpu)
    P = check(lit, shim, poll)
    full = run_both(-1, skip_two(), gpu)[0]
    keep = full["obs"][:, 2] <= poll
    assert P == keep.sum() and lit["pos"].tobytes() == full["pos"][keep].tobytes()
    assert (lit["obs"][:, 2] <= poll).all()


def test_the_shim_makes_one_call_and_counts_what_it_drops():
    sc = scene()
    s = pynp.StandIn(sc["cur"], sc["neighbours"])
    c0, st0 = s.device_calls(), s.stats()
    s.run(1, 3)
    m = s.members()
    st = s.stats() - st0
    assert s.device_calls() - c0 == 1 and st[0] == 1 and st[1] == len(m["pos"]) and st[2] > 0
    s.close()

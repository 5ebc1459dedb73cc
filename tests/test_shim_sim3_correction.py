"""CPU suite: shim/Sim3Correction_shim.cpp (ccm_b200_correct_sim3, the drop-in for the Sim3 pass of LoopFinder::CorrectLoop and
MapMerger::MergeMaps) against a literal restatement of both loop bodies, on stand-in KeyFrame / MapPoint objects held by real
shared_ptr in a real KeyFrameAndPose (oracle/ref_sim3_correction_wrap.cpp).  Both leave every keyframe's Tcw / Twc / Ow, connections
and mCorrected_MM and every point's position, normal, depth limits, tags and mCorrectedReference_* identical, the same sChangedKFs and
the same UpdateConnections order; the shim takes one device call (here the oracle's CPU double), moves each point with the call's
values and parks every normal.  The GPU suite runs the same over the real library (tests/test_gpu_sim3_correction.py)."""
import numpy as np
import pytest

from ccm_slam_b200 import synth
from oracle import pysc

EDGES = dict(K=24, P=700, window=6, null_frac=0.1, dup_frac=0.1, bad_mp_frac=0.05, tagged_frac=0.05, bad_kf_frac=0.3, all_bad_frac=0.08,
             off_ref_frac=0.3, empty_frac=0.15, null_entry_frac=0.15, unlisted_frac=0.05)
SCENES = {"loop": dict(kind="loop", seed=101, K=80, P=2000, n_loop=30, unlisted_frac=0.05),
          "merge": dict(kind="merge", seed=102, K=50, P=1500, unlisted_frac=0.05),
          "loop_edges": dict(kind="loop", seed=103, n_loop=9, **EDGES), "merge_edges": dict(kind="merge", seed=104, **EDGES)}


def compare(sc, gpu=False):
    merge = sc["kind"] == "merge"
    a = pysc.StandIn(sc, gpu=gpu)
    b = pysc.StandIn(sc, gpu=gpu)
    assert np.array_equal(a.map_order(), sc["entry_kf"])               # std::less<kfptr> is the scene's rank order
    a.literal(merge)
    s0 = b.stats()
    b.shim(merge)
    s1 = b.stats()
    ra, rb = a.read(), b.read()
    a.close(); b.close()
    for k in ra:
        assert np.array_equal(ra[k], rb[k], equal_nan=True), k
    moved_mask = (rb["tag_mm" if merge else "tag_lc"][:, 1] == 3) & ~sc["mp_tagged"]
    moved = int(moved_mask.sum())
    observed = np.diff(sc["obs_ptr"]) > 0
    d = s1 - s0
    assert d[0] == 1 and d[1] == moved and d[2] == 0                    # one call, one device value per moved point, no fallback
    assert d[3] == int((moved_mask & observed).sum()) and d[4] == 0 and d[5] == 0   # every normal from the call, none on the host
    assert d[6] == len(sc["entry_kf"])                                  # the entries' connections prepared in one batch
    assert moved > 100 and np.array_equal(ra["log"], sc["entry_kf"])   # UpdateConnections once per entry, in map order
    return ra


@pytest.mark.parametrize("name", list(SCENES))
def test_shim_leaves_the_members_the_reference_loop_leaves(name):
    sc = synth.make_sim3_correction(**SCENES[name])
    sc["kind"] = SCENES[name]["kind"]
    r = compare(sc)
    merge = sc["kind"] == "merge"
    assert (r["changed"].sum() == 0) if merge else (r["changed"].sum() == len(sc["entry_kf"]))
    assert (r["corrected_mm"][sc["entry_kf"], 1] == 3).all() if merge else (r["corrected_mm"][:, 1] != 3).all()

"""CPU suite: shim/KeyFrameConnections_shim.cpp over the CPU double of the device entry point (oracle/covis.mk).

 * a MergeMaps-shaped loop (per keyframe SetPose + UpdateConnections) leaves every keyframe's mConnectedKeyFrameWeights, ordered
   list and weights, parent and children exactly as the literal restatement does, through the parked path (one device call, one hit
   per keyframe) and through the host path;
 * the scenes include keyframes whose lists gain sub-threshold neighbours through later AddConnection calls, so the call order of
   the loop is what is checked, not only each keyframe's own counter;
 * a changed mvpMapPoints, observation count or point flag makes the member count on the host, with the reference's result;
 * Map::LoadMap's keyframe loop split into "every AddMapPoint, one prepare, every UpdateConnections" leaves the same members.
The same over the real library: tests/test_gpu_covisibility.py."""
import numpy as np
import pytest

from ccm_slam_b200 import synth
from oracle import pycv

MEMBER_KEYS = ("w_ptr", "w_kf", "w_w", "o_ptr", "o_kf", "o_w", "c_ptr", "c_kf", "parent", "first")


def scene(seed, **kw):
    base = dict(K=70, P=3500, max_deg=10, window=14, n_maps=2, same_id_frac=0.05, null_frac=0.1, dup_frac=0.02)
    base.update(kw)
    return synth.make_covisibility(seed=seed, **base)


def members_equal(a, b):
    for k in MEMBER_KEYS:
        assert np.array_equal(a[k], b[k]), k


def run(sc, mode, first_connection=None):
    s = pycv.StandIn(sc, first_connection=first_connection)
    c0, d0 = s.stats(), s.device_calls()
    s.merge(mode)
    out = s.members(), tuple(s.stats() - c0), s.device_calls() - d0
    s.close()
    return out


@pytest.mark.parametrize("first", ["all", "none", "mixed"])
def test_merge_loop_parked_and_host_paths_equal_the_literal(first):
    sc = scene(51)
    K, B = len(sc["kf_id"]), len(sc["batch"])
    fc = dict(all=np.ones(K, np.uint8), none=np.zeros(K, np.uint8),
              mixed=(np.random.default_rng(5).random(K) < 0.5).astype(np.uint8))[first]
    lit, _, _ = run(sc, 0, fc)
    host, hs, hd = run(sc, 1, fc)
    parked, ps, pd = run(sc, 2, fc)
    assert hs == (0, 0, B) and hd == 0
    assert ps == (B, 0, 0) and pd == 1
    members_equal(host, lit)
    members_equal(parked, lit)
    if first != "none":
        assert (lit["parent"] >= 0).sum() > K // 3 and lit["c_ptr"][-1] > K // 3
    # call order: some keyframe holds a neighbour below 15 next to ones at or above it, added to its list by a later keyframe's
    # AddConnection (UpdateBestCovisibles sorts the whole weight map)
    low_mixed = [k for k in range(K) if lit["o_ptr"][k + 1] > lit["o_ptr"][k]
                 and lit["o_w"][lit["o_ptr"][k]:lit["o_ptr"][k + 1]].min() < 15 <= lit["o_w"][lit["o_ptr"][k]:lit["o_ptr"][k + 1]].max()]
    assert len(low_mixed) > 5


def test_batch_in_address_order_and_a_partial_batch():
    sc = scene(52, batch_frac=0.5)
    sc["batch"] = sc["batch"][np.argsort(sc["kf_rank"][sc["batch"]])]      # CorrectedSim3All's std::map order
    lit, _, _ = run(sc, 0)
    parked, ps, _ = run(sc, 2)
    assert ps == (len(sc["batch"]), 0, 0)
    members_equal(parked, lit)


@pytest.mark.parametrize("kind", [1, 2, 3], ids=["map-point-index", "observation-added", "point-bad"])
def test_a_changed_keyframe_counts_on_the_host(kind):
    sc = scene(53)
    B = len(sc["batch"])
    extra = int(np.argmax(sc["kf_rank"]))
    s = pycv.StandIn(sc)
    s.merge_stale(kind, extra, literal=True)
    want = s.members()
    s.close()
    s = pycv.StandIn(sc)
    c0 = s.stats()
    s.merge_stale(kind, extra)
    hits, stale, host = s.stats() - c0
    got = s.members()
    s.close()
    members_equal(got, want)
    n = np.diff(sc["mvp_ptr"])[sc["batch"]]
    changed = int((n[::3] > 0).sum())
    assert host == stale and hits + stale == B
    if kind == 1:                                         # that keyframe alone
        assert stale == changed
    else:                                                 # every keyframe that lists the changed point
        assert changed <= stale < B


def test_an_observer_replaced_at_equal_count_is_not_seen():
    # the snapshot's blind spot (DESIGN §5): same mvpMapPoints, flags and counts; the parked counter is used
    sc = scene(54)
    extra = int(np.argmax(sc["kf_rank"]))
    s = pycv.StandIn(sc)
    c0 = s.stats()
    s.merge_stale(4, extra)
    assert tuple(s.stats() - c0)[1:] == (0, 0)
    s.close()


def test_load_map_split_equals_the_reference_loop():
    sc = scene(55, n_maps=3)
    outs = []
    for split in (0, 1):
        s = pycv.StandIn(sc, fill_mvp=False)
        c0 = s.stats()
        s.load_map(split)
        outs.append((s.members(), tuple(s.stats() - c0)))
        s.close()
    (ref, _), (got, st) = outs
    assert st == (len(sc["batch"]), 0, 0)
    members_equal(got, ref)
    assert (ref["parent"] >= 0).sum() > len(sc["kf_id"]) // 2

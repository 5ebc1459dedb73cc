"""CPU suite: shim/MapPointDescriptor_shim.cpp over the CPU doubles of the device entry points (oracle/distinctive.mk).

 * on fresh scenes the parked path (ccm_b200_prepare_descriptors + the member) and the host path leave identical mDescriptor members:
   bytes, type and shape; one parked choice is taken per written point; the store variant of the preparation gives the same;
 * an observation replaced (same count), an observation added, a point turned bad: stale or untouched, exactly as the reference;
 * the update loop of LocalMapping::SearchInNeighbors and the split loop of KeyFrame::EstablishInitialConnectionsServer leave the
   members the reference body leaves.
The same over the real library: tests/test_gpu_distinctive_descriptors.py."""
import numpy as np
import pytest

from ccm_slam_b200 import synth
from oracle import pydd


def scene(seed, **kw):
    base = dict(K=60, P=3000, max_deg=10, bad_kf_frac=0.1, all_bad_frac=0.01, empty_frac=0.01, bad_mp_frac=0.02, map_order=True)
    base.update(kw)
    return synth.make_distinctive(seed=seed, **base)


def members_equal(got, lit):
    w = lit["best"] >= 0
    assert np.array_equal(got["written"], w.astype(np.uint8))          # 1 = a continuous 1 x 32 CV_8U matrix; 0 = untouched
    assert np.array_equal(got["desc"], lit["desc"])


@pytest.mark.parametrize("store", [False, True], ids=["rows-with-the-call", "store"])
def test_parked_and_host_paths_leave_identical_members(store):
    sc = scene(91)
    s = pydd.StandIn(sc)
    lit = s.literal()
    if store:
        for k in range(len(sc["kf_bad"])):
            s.store_put(sc["kf_uid"][k], sc["kf_desc"][sc["kf_desc_ptr"][k]:sc["kf_desc_ptr"][k + 1]])
        s.register_store(1)
    calls, c0 = s.device_calls(), s.stats()
    try:
        parked = s.shim(prepare=1)
    finally:
        s.register_store(None)
    d = np.subtract(s.device_calls(), calls)
    assert tuple(d) == ((0, 1) if store else (1, 0))
    n_live = int(((np.diff(sc["obs_ptr"]) > 0) & ~sc["mp_bad"]).sum())   # every point the member gets past its first return on
    assert tuple(s.stats() - c0) == (n_live, 0, 0)                      # one hit each, the all-bad ones included (untouched)
    s.close()
    s = pydd.StandIn(sc)
    c0 = s.stats()
    host = s.shim(prepare=0)
    assert tuple(s.stats() - c0) == (0, 0, n_live)
    s.close()
    assert (lit["best"] >= 0).sum() > 2500 and (lit["best"] == -1).sum() > 50
    members_equal(parked, lit)
    members_equal(host, lit)


@pytest.mark.parametrize("kind", [1, 2, 3], ids=["observation-replaced", "observation-added", "point-bad"])
def test_stale_snapshot_falls_back_or_returns_untouched(kind):
    sc = scene(92, P=1500)
    s = pydd.StandIn(sc)
    before = s.literal()
    rng = np.random.default_rng(7)
    extra = s.add_keyframe(uid=99999, desc=rng.integers(0, 256, (16, 32), dtype=np.uint8))
    c0 = s.stats()
    r = s.stale(kind, extra)
    hits, stale, host = s.stats() - c0
    changed = np.zeros(s.P, bool); changed[::2] = True
    prepared = (np.diff(sc["obs_ptr"]) > 0) & ~sc["mp_bad"]
    after = s.literal()                                   # the scene as the members found it
    members_equal(r, after)
    if kind == 3:                                         # the member returns before it looks at the parked choice
        assert stale == 0 and hits == int((prepared & ~changed).sum()) and (r["written"][changed] == 0).all()
    else:
        assert stale == int((prepared & changed).sum()) and hits == int((prepared & ~changed).sum())
        assert not np.array_equal(before["desc"][prepared & changed], after["desc"][prepared & changed])
        newly = changed & ~prepared & ~sc["mp_bad"] if kind == 2 else np.zeros(s.P, bool)   # an empty point given an observer
        assert host == stale + int(newly.sum())
    s.close()


def test_search_in_neighbors_loop():
    sc = scene(93, P=2000)
    s = pydd.StandIn(sc)
    lit = s.literal()
    rng = np.random.default_rng(8)
    pts = rng.choice(s.P, 900, replace=False)
    pts = np.concatenate([pts, pts[:20]])                 # a point matched twice
    c0, n0 = s.stats(), s.normal_stats()
    got = s.search_in_neighbors(pts)
    touched = np.zeros(s.P, bool); touched[pts] = True
    w = touched & (lit["best"] >= 0)
    live = touched & (np.diff(sc["obs_ptr"]) > 0) & ~sc["mp_bad"]
    assert np.array_equal(got["desc"][touched], lit["desc"][touched]) and np.array_equal(got["written"][touched], w[touched].astype(np.uint8))
    assert (got["written"][~touched] == 0).all()
    hits, stale, host = s.stats() - c0
    assert hits == int(live.sum()) and stale == 0 and host == int(live[pts[:20]].sum())   # a repeat finds its entry taken: host
    assert (s.normal_stats() - n0)[0] > 0.9 * hits       # UpdateNormalAndDepth ran on the parked normals too
    s.close()


def test_establish_initial_connections_split_equals_the_reference_loop():
    sc = scene(94, P=1500, bad_kf_frac=0.05)
    rng = np.random.default_rng(9)
    M = 1200
    new_desc = rng.integers(0, 256, (M, 32), dtype=np.uint8)
    mp_of_idx = np.full(M, -1, np.int32)
    idx = rng.choice(M, 900, replace=False)
    mp_of_idx[idx] = rng.choice(s_P := 1500, 900, replace=False)
    dup = rng.choice(np.flatnonzero(mp_of_idx < 0), 30, replace=False)
    mp_of_idx[dup] = mp_of_idx[idx[:30]]                  # a point at two indices of the keyframe
    # a new observation near the point's own descriptors, so that it sometimes wins
    for i in np.flatnonzero(mp_of_idx >= 0):
        p = mp_of_idx[i]
        if sc["obs_ptr"][p + 1] > sc["obs_ptr"][p] and rng.random() < 0.5:
            new_desc[i] = sc["obs_desc"][sc["obs_ptr"][p]]
    outs = []
    for split in (0, 1):
        s = pydd.StandIn(sc)
        k = s.add_keyframe(uid=77777, desc=new_desc)
        outs.append(s.establish(k, mp_of_idx, split))
        s.close()
    ref, got = outs
    t = ref["written"] == 1
    assert t.sum() > 800 and np.array_equal(got["written"], ref["written"])
    assert np.array_equal(got["desc"][t], ref["desc"][t])
    assert s_P == len(sc["obs_ptr"]) - 1

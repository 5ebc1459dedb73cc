"""GPU suite: ccm_distinctive_descriptors and ccm_kfstore_distinctive_descriptors (MapPoint::ComputeDistinctiveDescriptors for a batch,
ccm_slam_b200/csrc/distinctive.cu) against the host entry point and the oracle, exactly, on the fixture, on the observer structure of
the BA shapes and on N distributions that cross every kernel-path edge; the store variant's bus traffic and argument checks; and
shim/MapPointDescriptor_shim.cpp over the real library."""
import numpy as np
import pytest

from ccm_slam_b200 import api, synth
from ccm_slam_b200.frontend import KeyFrameStore
from oracle import pydd
from tests import test_distinctive_descriptors as TD

pytestmark = pytest.mark.gpu

SHAPES = {
    "tiny": lambda: synth.make_config("tiny"),
    "small": lambda: synth.make_config("small"),
    "cfg2": lambda: synth.make_config("cfg2"),
    "cfg4": lambda: synth.make_config("cfg4"),
    "cfg5_tenth": lambda: synth.make_config("cfg5", K=1000, P=100000),
    "awkward": lambda: synth.make_awkward_ba(),
}
KEYS = ("best", "best_median", "desc")
# N around 32 (warp / CTA) and 1024 (staged / in place), with bad observers that move N across an edge only after the skip
EDGES = (1, 2, 3, 4, 30, 31, 32, 33, 34, 63, 64, 65, 255, 256, 257, 1023, 1024, 1025, 1026, 2048, 4000)


def same(a, b):
    for k in KEYS:
        assert np.array_equal(a[k], b[k]), k


@pytest.fixture(scope="module", autouse=True)
def device():
    if api.device_count() == 0:
        pytest.skip("no CUDA device")
    api.init(0)


def test_device_reproduces_the_fixture():
    for name, sc, want in TD.fixture_cases():
        same(api.distinctive_descriptors(sc), want)


@pytest.mark.parametrize("name", list(SHAPES))
def test_device_equals_host_and_oracle(name):
    sc = synth.make_distinctive(SHAPES[name](), seed=101, bad_kf_frac=0.05, all_bad_frac=0.002, empty_frac=0.002, bad_mp_frac=0.01)
    l0 = api.kernel_launches()
    r = api.distinctive_descriptors(sc)
    assert api.kernel_launches() == l0 + 3
    same(r, api.distinctive_descriptors(sc, host=True))
    if name not in ("cfg4", "cfg5_tenth"):
        same(r, pydd.oracle(sc))
    assert (r["best"] >= 0).sum() > 0.9 * len(r["best"])


@pytest.mark.parametrize("seed", [102, 103])
def test_every_kernel_path_edge(seed):
    rng = np.random.default_rng(seed)
    forced = tuple(int(n) for n in rng.permutation(np.repeat(EDGES, 2)))
    sc = synth.make_distinctive(seed=seed, K=5000, P=3000, max_deg=40, bad_kf_frac=0.1, all_bad_frac=0.01, empty_frac=0.01, forced_n=forced)
    # points whose survivors cross 32 and 1024 only after the skip: many bad keyframes among their observers
    n = np.add.reduceat(np.append(~sc["kf_bad"].astype(bool)[sc["obs_kf"]], False).astype(np.int64), sc["obs_ptr"][:-1])
    for e in EDGES:
        assert (n == e).sum() >= 2, e
    r = api.distinctive_descriptors(sc)
    same(r, api.distinctive_descriptors(sc, host=True))
    same(r, pydd.oracle(sc))
    skewed = synth.make_distinctive(seed=seed + 10, K=3000, P=0, bad_kf_frac=0.0, forced_n=(50, 50, 50, 1500, 2000))
    skewed["kf_bad"] = (rng.random(3000) < 0.5).astype(np.uint8)
    nn = np.add.reduceat(np.append(~skewed["kf_bad"].astype(bool)[skewed["obs_kf"]], False).astype(np.int64), skewed["obs_ptr"][:-1])
    deg = np.diff(skewed["obs_ptr"])
    assert ((deg > 32) & (nn <= 32)).any() and ((deg > 1024) & (nn <= 1024)).any()
    same(api.distinctive_descriptors(skewed), pydd.oracle(skewed))


def _store_of(sc):
    st = KeyFrameStore()
    for k in range(len(sc["kf_bad"])):
        d = sc["kf_desc"][sc["kf_desc_ptr"][k]:sc["kf_desc_ptr"][k + 1]]
        kps = np.zeros(len(d), st_kp_dtype())
        st.put(int(sc["kf_uid"][k]), kps, d)
    return st


def st_kp_dtype():
    from ccm_slam_b200.frontend import KP_DTYPE
    return KP_DTYPE


def test_store_variant_equals_the_host_buffer_variant():
    sc = synth.make_distinctive(synth.make_config("cfg2"), seed=104, bad_kf_frac=0.0, empty_frac=0.01, forced_n=(33, 1025, 2000))
    sc["kf_bad"] = sc["kf_bad"].copy(); sc["kf_bad"][3::11] = 1          # bad observers everywhere, forced points included
    st = _store_of(sc)
    b0 = st.h2d_bytes()
    r = st.distinctive_descriptors(sc["kf_uid"], sc["kf_bad"], sc["obs_ptr"], sc["obs_kf"], sc["obs_feat"])
    assert st.h2d_bytes() == b0
    same(r, api.distinctive_descriptors(sc))
    same(r, pydd.oracle(sc))
    # a bad observer's row is not read: its uid may be gone from the store
    bad_rows = np.flatnonzero(sc["kf_bad"])
    assert len(bad_rows)
    st.erase(int(sc["kf_uid"][bad_rows[0]]))
    same(st.distinctive_descriptors(sc["kf_uid"], sc["kf_bad"], sc["obs_ptr"], sc["obs_kf"], sc["obs_feat"]), r)
    # an unknown uid or a feature index out of range of an observer that is not bad: the call fails, names the point, writes nothing
    good = np.flatnonzero(~sc["kf_bad"].astype(bool)[sc["obs_kf"]])
    j = int(good[len(good) // 2]); p = int(np.searchsorted(sc["obs_ptr"], j, side="right") - 1)
    uid = sc["kf_uid"].copy(); uid[sc["obs_kf"][j]] = np.uint64(123456789)
    feat = sc["obs_feat"].copy(); feat[j] = sc["kf_nfeat"][sc["obs_kf"][j]]
    neg = sc["obs_feat"].copy(); neg[j] = -1
    import ctypes as C
    L = api.lib()
    live = ~sc["kf_bad"].astype(bool)[sc["obs_kf"]]
    first = int(np.flatnonzero(live & (sc["obs_kf"] == sc["obs_kf"][j]))[0])   # the unknown uid fails every point observing that row
    p_uid = int(np.searchsorted(sc["obs_ptr"], first, side="right") - 1)
    for u, f, pp in ((uid, sc["obs_feat"], p_uid), (sc["kf_uid"], feat, p), (sc["kf_uid"], neg, p)):
        P = len(sc["obs_ptr"]) - 1
        best = np.full(P, 7, np.int32); med = np.full(P, 7, np.int32); desc = np.full((P, 32), 7, np.uint8)
        a = [np.ascontiguousarray(x) for x in (u, sc["kf_bad"], sc["obs_ptr"], sc["obs_kf"], f)]
        rc = L.ccm_kfstore_distinctive_descriptors(st._h, len(u), *[x.ctypes.data_as(C.c_void_p) for x in a[:2]], P,
                                                   *[x.ctypes.data_as(C.c_void_p) for x in a[2:]], best.ctypes.data_as(C.c_void_p),
                                                   med.ctypes.data_as(C.c_void_p), desc.ctypes.data_as(C.c_void_p))
        assert rc == -1
        msg = L.ccm_last_error
        msg.restype = C.c_char_p
        assert ("point %d," % pp) in msg().decode()
        assert (best == 7).all() and (med == 7).all() and (desc == 7).all()
    assert st.h2d_bytes() == b0
    st.close()


def test_host_buffer_variant_rejects_rows_out_of_range():
    sc = synth.make_distinctive(seed=105, K=10, P=500)
    bad = dict(sc); bad["obs_kf"] = sc["obs_kf"].copy(); bad["obs_kf"][-1] = 10
    with pytest.raises(api.CCMError, match="point 499"):
        api.distinctive_descriptors(bad)
    assert len(api.distinctive_descriptors(synth.make_distinctive(seed=106, K=3, P=0))["best"]) == 0


def test_shim_over_the_real_library():
    sc = synth.make_distinctive(seed=107, K=80, P=4000, max_deg=12, bad_kf_frac=0.1, all_bad_frac=0.01, empty_frac=0.01,
                                bad_mp_frac=0.02, map_order=True)
    outs = {}
    for gpu in (False, True):
        s = pydd.StandIn(sc, gpu=gpu)
        c0 = s.stats()
        outs[gpu] = s.shim(prepare=2)
        live = int(((np.diff(sc["obs_ptr"]) > 0) & ~sc["mp_bad"]).sum())
        assert tuple(s.stats() - c0) == (live, 0, 0)
        lit = s.literal()
        s.close()
    for k in ("desc", "written"):
        assert np.array_equal(outs[True][k], outs[False][k])
    assert np.array_equal(outs[True]["desc"], lit["desc"])
    # the store variant through the shim
    st = _store_of(sc)
    s = pydd.StandIn(sc, gpu=True)
    s.register_store(st._h)
    try:
        c0 = s.stats()
        got = s.shim(prepare=1)
        assert (s.stats() - c0)[0] == live
    finally:
        s.register_store(None)
    s.close(); st.close()
    assert np.array_equal(got["desc"], lit["desc"])

"""CPU suite: map-point descriptors (MapPoint::ComputeDistinctiveDescriptors, cslam/src/MapPoint.cpp:929-994).

 * the pin: tests/golden/distinctive_descriptors.npz (a numpy witness, checked by its generator against a pure-Python restatement);
   the oracle, the library's host entry point ccm_distinctive_descriptors_host and the literal restatement on stand-in objects all
   reproduce it exactly: chosen position, median and bytes;
 * the same three agree on fresh scenes;
 * the fixture and the random scenes each catch every plausible slip of the rule;
 * ccm_distinctive_descriptors and ccm_kfstore_distinctive_descriptors need a device.
The device kernels are tests/test_gpu_distinctive_descriptors.py; the shim tests/test_shim_distinctive.py."""
import importlib.util
import os
import subprocess

import numpy as np
import pytest

from ccm_slam_b200 import api, synth
from oracle import pydd

HERE = os.path.dirname(os.path.abspath(__file__))
KEYS = ("best", "best_median", "desc")


def golden():
    spec = importlib.util.spec_from_file_location("make_distinctive_golden", os.path.join(HERE, "golden", "make_distinctive_golden.py"))
    mod = importlib.util.module_from_spec(spec); spec.loader.exec_module(mod)
    return mod


def fixture_cases():
    mod = golden()
    z = np.load(os.path.join(HERE, "golden", "distinctive_descriptors.npz"))
    return [(name,) + mod.load(z, name) for name in mod.NAMES]


def same(a, b):
    for k in KEYS:
        assert np.array_equal(a[k], b[k]), k


def max_survivors(sc):
    live = ~sc["kf_bad"].astype(bool)[sc["obs_kf"]]
    return int(np.add.reduceat(np.append(live, False).astype(np.int64), sc["obs_ptr"][:-1]).max()) if len(sc["obs_ptr"]) > 1 else 0


def test_everything_reproduces_the_fixture():
    mod = golden()
    for name, sc, want in fixture_cases():
        same(mod.witness(sc), want)
        same(pydd.oracle(sc), want)
        same(api.distinctive_descriptors(sc, host=True), want)
        if max_survivors(sc) <= 1000:                       # the literal body's stack array: 4 N^2 bytes
            s = pydd.StandIn(sc)
            same(s.literal(), want)
            s.close()
        assert (want["best"] >= 0).sum() >= 30, name


def test_the_fixture_covers_its_edge_cases():
    (_, sc, w), = [c for c in fixture_cases() if c[0] == "hand"]
    ptr, bad = sc["obs_ptr"], sc["kf_bad"].astype(bool)[sc["obs_kf"]]
    deg = np.diff(ptr)
    n = np.array([(~bad[ptr[i]:ptr[i + 1]]).sum() for i in range(len(deg))])
    for want in (1, 2, 3, 4, 31, 32, 33, 64, 65, 256, 257, 1024, 1025):
        assert (n == want).any(), want
    assert n.max() > 2500 and ((deg > 0) & (n == 0)).sum() >= 2 and (deg == 0).sum() >= 1
    # a chosen observer after skipped ones: its position counts them
    first_bad = np.array([deg[i] > 0 and bad[ptr[i]] for i in range(len(deg))])
    assert (first_bad & (w["best"] >= 2)).any()
    # a minimum tied at a later position than 0
    assert ((w["best"] > 0) & (w["best_median"] == 0)).any()


@pytest.mark.parametrize("kw", [dict(seed=81, map_order=True),
                                dict(seed=82, K=12, P=800, bad_kf_frac=0.3, bad_mp_frac=0.05, all_bad_frac=0.05, empty_frac=0.05, map_order=True),
                                dict(seed=83, K=400, P=300, max_deg=40, bad_kf_frac=0.1, forced_n=(31, 32, 33, 64, 65, 200), map_order=True),
                                dict(seed=84, K=30, P=2000, max_deg=60, bad_kf_frac=0.1)],
                         ids=["random", "edges", "wide", "repeated-observers"])
def test_oracle_host_and_literal_agree(kw):
    sc = synth.make_distinctive(**kw)
    o = pydd.oracle(sc)
    same(api.distinctive_descriptors(sc, host=True), o)
    same(golden().witness(sc), o)
    if kw.get("map_order"):
        s = pydd.StandIn(sc)
        same(s.literal(), o)
        s.close()


def slipped(sc, upper=False, last=False, survivor_index=False, le=False):
    """the witness with one slip: the upper middle for even N / the last minimum / BestIdx taken as the list position / <= for <"""
    ptr, okf, bad, D = sc["obs_ptr"], sc["obs_kf"], sc["kf_bad"].astype(bool), sc["obs_desc"]
    P = len(ptr) - 1
    best = np.full(P, -1, np.int32); med = np.zeros(P, np.int32); desc = np.zeros((P, 32), np.uint8)
    for i in range(P):
        pos = np.flatnonzero(~bad[okf[ptr[i]:ptr[i + 1]]])
        if len(pos) == 0:
            continue
        B = np.unpackbits(D[ptr[i] + pos], axis=1).astype(np.int32)
        s = B.sum(1)
        dist = s[:, None] + s[None, :] - 2 * (B @ B.T)
        N = len(pos)
        m = np.sort(dist, axis=1)[:, N // 2 if upper else (N - 1) // 2]
        if last:
            a = N - 1 - int(np.argmin(m[::-1]))
        elif le:
            a, bm = 0, 2 ** 31 - 1
            for q in range(N):
                if m[q] <= bm:
                    a, bm = q, m[q]
        else:
            a = int(np.argmin(m))
        p = a if survivor_index else pos[a]
        best[i] = p; med[i] = m[a]; desc[i] = D[ptr[i] + p]
    return dict(best=best, best_median=med, desc=desc)


SLIPS = {"upper-median": dict(upper=True), "last-minimum": dict(last=True), "survivor-index": dict(survivor_index=True), "le": dict(le=True)}


@pytest.mark.parametrize("slip", list(SLIPS))
def test_fixture_and_random_scenes_catch_each_slip(slip):
    def caught(a, b):
        return any(not np.array_equal(a[k], b[k]) for k in KEYS)
    for name, sc, want in fixture_cases():
        if name == "hand":
            assert caught(slipped(sc, **SLIPS[slip]), want), name
    sc = synth.make_distinctive(seed=85, K=20, P=1500, bad_kf_frac=0.2, map_order=True)
    assert caught(slipped(sc, **SLIPS[slip]), pydd.oracle(sc))


def test_library_entry_points():
    sc = synth.make_distinctive(seed=86, K=5, P=20)
    L = api.lib()
    for f in ("ccm_distinctive_descriptors", "ccm_distinctive_descriptors_host", "ccm_kfstore_distinctive_descriptors"):
        assert hasattr(L, f)
    if api.device_count() == 0:
        with pytest.raises(api.CCMError) as e:
            api.distinctive_descriptors(sc)
        assert e.value.code == -2
        from ccm_slam_b200.frontend import KeyFrameStore
        with pytest.raises(api.CCMError) as e:
            KeyFrameStore()
        assert e.value.code == -2
        import ctypes as C
        best = np.zeros(len(sc["obs_ptr"]) - 1, np.int32)
        a = [np.ascontiguousarray(sc[k]) for k in ("kf_uid", "kf_bad", "obs_ptr", "obs_kf", "obs_feat")]
        rc = L.ccm_kfstore_distinctive_descriptors(C.c_void_p(1), len(a[0]), *[x.ctypes.data_as(C.c_void_p) for x in a[:2]], len(best),
                                                   *[x.ctypes.data_as(C.c_void_p) for x in a[2:]], best.ctypes.data_as(C.c_void_p), None, None)
        assert rc == -2
    bad = dict(sc); bad["obs_kf"] = sc["obs_kf"].copy(); bad["obs_kf"][3] = 99
    with pytest.raises(api.CCMError, match="point"):
        api.distinctive_descriptors(bad, host=True)
    empty = synth.make_distinctive(seed=87, K=3, P=0)
    assert len(api.distinctive_descriptors(empty, host=True)["best"]) == 0


def test_shim_type_check_target():
    subprocess.check_call(["make", "-C", os.path.join(HERE, "..", "oracle"), "-s", "shim-check-distinctive"])

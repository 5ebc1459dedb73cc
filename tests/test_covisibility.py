"""CPU suite: covisibility weights (KeyFrame::UpdateConnections' counter and ordered connections, cslam/src/KeyFrame.cpp:629-711).

 * the pin: tests/golden/covisibility.npz (a pure-Python witness, checked by its generator against the oracle); the oracle, the
   library's host entry point ccm_covisibility_host and the literal restatement on stand-in objects all reproduce it exactly;
 * the same three agree on fresh scenes: random, BA observation shapes, several maps, shared mIds, tie storms;
 * the fixture catches every plausible slip of the rule;
 * the capacity rule and the row checks of the host entry point; ccm_covisibility needs a device.
The device kernels are tests/test_gpu_covisibility.py; the shim tests/test_shim_covisibility.py."""
import importlib.util
import os

import numpy as np
import pytest

from ccm_slam_b200 import api, synth
from oracle import pycv

HERE = os.path.dirname(os.path.abspath(__file__))
KEYS = ("conn_ptr", "conn_kf", "conn_w", "n_sel", "sel_kf", "sel_w", "status")


def golden():
    spec = importlib.util.spec_from_file_location("make_covisibility_golden", os.path.join(HERE, "golden", "make_covisibility_golden.py"))
    mod = importlib.util.module_from_spec(spec); spec.loader.exec_module(mod)
    return mod


def fixture_cases():
    mod = golden()
    z = np.load(os.path.join(HERE, "golden", "covisibility.npz"))
    return [(name,) + mod.load(z, name) for name in mod.NAMES]


def same(a, b):
    for k in KEYS:
        assert np.array_equal(a[k], b[k]), k


def differs(a, b):
    return any(not np.array_equal(a[k], b[k]) for k in KEYS)


def literal(sc):
    s = pycv.StandIn(sc)
    try:
        return s.literal_flat()
    finally:
        s.close()


def test_everything_reproduces_the_fixture():
    mod = golden()
    for name, sc, want in fixture_cases():
        same(mod.witness(sc), want)
        same(pycv.oracle(sc), want)
        same(api.covisibility(sc, host=True), want)
        same(literal(sc), want)
        assert want["status"].sum() >= 10, name


def test_the_fixture_covers_its_edge_cases():
    mod = golden()
    (_, sc, w), = [c for c in fixture_cases() if c[0] == "edges"]
    R = mod.EDGE_ROWS
    b_of = {int(r): b for b, r in enumerate(sc["batch"])}

    def conn(row):
        b = b_of[row]; a, e = w["conn_ptr"][b], w["conn_ptr"][b + 1]
        return dict(zip(w["conn_kf"][a:e].tolist(), w["conn_w"][a:e].tolist())), w["sel_kf"][a:a + w["n_sel"][b]].tolist()
    for r in ("no_points", "all_bad", "only_self", "same_id"):
        assert w["status"][b_of[R[r]]] == 0, r
    c, s = conn(R["below_tie"])
    top = [k for k, v in c.items() if v == max(c.values())]
    assert max(c.values()) < 15 and len(top) == 3
    assert s == [min(top, key=lambda k: sc["kf_rank"][k])]                  # the first maximum in address order
    c, s = conn(R["at_14_15"])
    assert sorted(c.values()) == [14, 15, 15, 15] and len(s) == 3
    assert [sc["kf_rank"][k] for k in s] == sorted((sc["kf_rank"][k] for k in s), reverse=True)   # equal weights: highest address first
    assert R["bad_observer"] in s and sc["kf_bad"][R["bad_observer"]]
    c, _ = conn(R["duplicate"])
    assert sorted(c.values()) == [1, 3]
    (_, st, ws), = [c for c in fixture_cases() if c[0] == "storm"]
    assert (ws["n_sel"] >= 3).sum() >= 10 and (np.diff(ws["conn_ptr"]) > 0).all()


SLIPS = ("skip_bad_observers", "strict", "ascending_ties", "last_max", "self_by_row")


@pytest.mark.parametrize("slip", SLIPS)
def test_the_fixture_catches_each_slip(slip):
    mod = golden()
    assert any(differs(mod.witness(sc, **{slip: True}), want) for _, sc, want in fixture_cases())


SCENES = {
    "random": lambda: synth.make_covisibility(seed=41, K=60, P=3000, max_deg=10, window=14, same_id_frac=0.1),
    "small": lambda: synth.make_covisibility(synth.make_config("small"), seed=42, same_id_frac=0.05),
    "cfg2": lambda: synth.make_covisibility(synth.make_config("cfg2"), seed=43, batch_frac=0.6),
    "maps": lambda: synth.make_covisibility(seed=44, K=90, P=4000, max_deg=12, window=20, n_maps=4, null_frac=0.3, dup_frac=0.05),
    "storm": lambda: golden().storm(45),
}


@pytest.mark.parametrize("name", list(SCENES))
def test_oracle_host_and_literal_agree(name):
    sc = SCENES[name]()
    o = pycv.oracle(sc)
    same(api.covisibility(sc, host=True), o)
    same(literal(sc), o)
    for th in (1, 30):
        same(api.covisibility(sc, host=True, th=th), pycv.oracle(sc, th=th))


def test_ranks_decide_every_order():
    sc = golden().storm(46)
    base = api.covisibility(sc, host=True)
    for seed in range(3):
        sc2 = dict(sc); sc2["kf_rank"] = np.random.default_rng(seed).permutation(len(sc["kf_id"])).astype(np.uint32)
        got = api.covisibility(sc2, host=True)
        same(got, pycv.oracle(sc2))
        same(got, literal(sc2))
        assert differs(got, base)                                            # the address order is an input, not noise


def _raw(sc, cap, fn="ccm_covisibility_host"):
    import ctypes as C
    b, mptr, mp = api.covisibility_batch(sc)
    a = [np.ascontiguousarray(sc[k], t) for k, t in (("kf_id", np.uint64), ("kf_rank", np.uint32), ("mp_bad", np.uint8),
                                                     ("obs_ptr", np.int64), ("obs_kf", np.int32))]
    B = len(b)
    o = dict(conn_ptr=np.full(B + 1, 7, np.int64), conn_kf=np.full(max(cap, 1), 7, np.int32), conn_w=np.full(max(cap, 1), 7, np.int32),
             n_sel=np.full(B, 7, np.int32), sel_kf=np.full(max(cap, 1), 7, np.int32), sel_w=np.full(max(cap, 1), 7, np.int32),
             status=np.full(B, 7, np.uint8))
    total = np.zeros(1, np.int64)
    p = lambda x: x.ctypes.data_as(C.c_void_p)                               # noqa: E731
    rc = getattr(api.lib(), fn)(len(a[0]), p(a[0]), p(a[1]), B, p(b), p(mptr), p(mp), len(a[2]), p(a[2]), p(a[3]), p(a[4]), 15,
                                C.c_int64(cap), *[p(o[k]) for k in KEYS], p(total))
    return rc, o, int(total[0])


def test_capacity_below_the_total_is_refused_and_nothing_written():
    sc = SCENES["random"]()
    T = int(pycv.oracle(sc)["conn_ptr"][-1])
    rc, o, total = _raw(sc, T - 1)
    assert rc == -1 and total == T
    assert all((o[k] == 7).all() for k in KEYS)
    rc, o, total = _raw(sc, T)
    assert rc == 0 and total == T and o["conn_ptr"][-1] == T


def test_rows_out_of_range_name_the_keyframe():
    sc = SCENES["random"]()
    b = 17
    row = int(sc["batch"][b])
    first = int(sc["mvp_ptr"][row])
    bad = dict(sc); bad["mvp"] = sc["mvp"].copy(); bad["mvp"][first] = len(sc["mp_bad"])
    with pytest.raises(api.CCMError, match="batch keyframe %d " % b):
        api.covisibility(bad, host=True)
    p = int(next(q for q in sc["mvp"][first:] if q >= 0 and not sc["mp_bad"][q] and sc["obs_ptr"][q + 1] > sc["obs_ptr"][q]))
    bad = dict(sc); bad["obs_kf"] = sc["obs_kf"].copy(); bad["obs_kf"][sc["obs_ptr"][p]] = len(sc["kf_id"])
    with pytest.raises(api.CCMError, match="batch keyframe"):
        api.covisibility(bad, host=True)
    K = len(sc["kf_id"])                                                     # a batch row past the table (its list empty)
    bad = dict(sc, mvp_ptr=np.append(sc["mvp_ptr"], sc["mvp_ptr"][-1]), batch=np.r_[sc["batch"][:3], K].astype(np.int32))
    with pytest.raises(api.CCMError, match="batch keyframe 3 .*out of range"):
        api.covisibility(bad, host=True)
    bad = dict(sc); bad["kf_rank"] = sc["kf_rank"].copy(); bad["kf_rank"][0] = bad["kf_rank"][1]
    with pytest.raises(api.CCMError, match="permutation"):
        api.covisibility(bad, host=True)


def test_empty_batch_and_device_without_device():
    sc = SCENES["random"]()
    r = api.covisibility(sc, host=True, batch=np.zeros(0, np.int32))
    assert r["conn_ptr"].tolist() == [0] and len(r["n_sel"]) == 0
    if api.device_count() == 0:
        with pytest.raises(api.CCMError) as e:
            api.covisibility(sc)
        assert e.value.code == -2

"""CPU suite: the redundancy test of LocalMapping::KeyFrameCullingV3 (cslam/src/Mapping.cpp:771-863), earlier culls included, behind
ccm_keyframe_culling_host.

 * the pin: tests/golden/keyframe_culling.npz, written by a witness that walks the member literally over mutable state and that its
   generator checks against the oracle; the oracle and the host entry point both reproduce it;
 * the fixture holds every edge case the contract names, and each deliberately wrong reading of the member fails it;
 * the host entry point equals the oracle on seeded server-shaped scenes, and counts again exactly the candidates a cull reached;
 * refused input: the message names the candidate or point, and nothing is written.
The device kernel is tests/test_gpu_keyframe_culling.py."""
import os

import numpy as np
import pytest

from ccm_slam_b200 import api, synth
from oracle import pykc

HERE = os.path.dirname(os.path.abspath(__file__))
OUT = ("cull", "n_mps", "n_red")


def fixture():
    z = np.load(os.path.join(HERE, "golden", "keyframe_culling.npz"))
    n = len({k.split("_")[0] for k in z.files})
    for c in range(n):
        sc = {k[len("case%d_in_" % c):]: z[k] for k in z.files if k.startswith("case%d_in_" % c)}
        yield sc, {k: z["case%d_%s" % (c, k)] for k in OUT}


def same(a, b):
    return all(np.array_equal(a[k], b[k]) for k in OUT)


def test_host_and_oracle_reproduce_the_fixture():
    cases = list(fixture())
    assert len(cases) == 4
    settled = 0
    for sc, w in cases:
        assert same(pykc.oracle(sc), w)
        h = api.keyframe_culling(sc, host=True)
        assert same(h, w)
        settled += h["n_settled"]
    assert settled > 0


def test_fixture_holds_the_edge_cases():
    cases = list(fixture())
    r = [(int(m), int(n), int(c), float(sc["red_thres"])) for sc, w in cases for m, n, c in zip(w["n_mps"], w["n_red"], w["cull"])]
    assert (50, 49, 0, 0.98) in r and (100, 98, 0, 0.98) in r                     # the ties do not cull
    assert any(m == 0 and c == 0 for m, _, c, _ in r)                             # nMPs == 0
    sc, w = cases[3]                                                              # the f64 / f32 split, culled in f64 only
    t, n, k = float(sc["red_thres"]), int(w["n_mps"][0]), int(w["n_red"][0])
    assert w["cull"][0] == 1 and k > t * n and not np.float32(k) > np.float32(t) * np.float32(n)
    for sc, w in cases[:3]:
        bad = sc["kf_bad"][sc["cand_kf"]].astype(bool)
        assert (w["cull"].astype(bool) & bad).any()                              # an already bad candidate judged redundant
        assert (w["cull"].astype(bool) & sc["cand_not_erase"].astype(bool)).any()   # ... and one with mbNotErase
        ptr, okf, ooct = sc["obs_ptr"], sc["obs_kf"], sc["obs_octave"]
        nobs = sc["mp_nobs"]
        assert (sc["slot_mp"] < 0).any() and sc["mp_bad"].any() and (sc["mp_ref"] < 0).any() and (nobs == 3).any()
        own = np.repeat(sc["cand_kf"], np.diff(sc["slot_ptr"]))
        held = sc["slot_mp"] >= 0
        assert len(np.unique(np.stack([own[held], sc["slot_mp"][held]]), axis=1)[0]) < held.sum()   # a point at two slots of one candidate
        lvl = {d: 0 for d in (1, 2)}
        for j in np.flatnonzero(held)[:20000]:
            p = sc["slot_mp"][j]
            for e in range(ptr[p], ptr[p + 1]):
                d = ooct[e] - sc["slot_octave"][j]
                if d in lvl and okf[e] != own[j] and not sc["kf_bad"][okf[e]]:
                    lvl[d] += 1
        assert lvl[1] > 0 and lvl[2] > 0                                         # observers at level + 1 and level + 2
        assert sc["kf_bad"][okf].any()                                           # bad observers


@pytest.mark.parametrize("slip", list(pykc.SLIPS))
def test_every_wrong_reading_fails_the_fixture(slip):
    assert any(not same(pykc.oracle(sc, pykc.SLIPS[slip]), w) for sc, w in fixture())


@pytest.mark.parametrize("kw", [dict(n_c=20, seed=1), dict(n_c=60, seed=2, n_redundant=5), dict(n_c=30, slots=400, seed=3, obs=(3, 9),
                                bad_kf_frac=0.25, no_ref_frac=0.05, n_redundant=6), dict(n_c=10, seed=4, edges=False)])
def test_host_equals_oracle(kw):
    sc = synth.make_keyframe_culling_scene(**kw)
    h = api.keyframe_culling(sc, host=True)
    assert same(h, pykc.oracle(sc))
    assert h["cull"].sum() >= 2 and h["n_settled"] > 0


def test_settle_counts_only_reached_candidates():
    # no effective cull: nothing is counted again, and the verdicts equal the counts over the start state
    sc = synth.make_keyframe_culling_scene(n_c=20, seed=5, n_redundant=0, edges=False)
    h = api.keyframe_culling(sc, host=True)
    assert h["cull"].sum() == 0 and h["n_settled"] == 0
    # a cascade flips a verdict: without the settle the later candidate would not cull
    sc = synth.make_keyframe_culling_scene(n_c=0, seed=6)
    h = api.keyframe_culling(sc, host=True)
    nc = pykc.oracle(sc, pykc.SLIPS["no_cascade"])
    assert h["n_settled"] > 0 and (h["cull"] != nc["cull"]).any()


def test_no_candidates():
    sc = synth.make_keyframe_culling_scene(n_c=5, seed=7, edges=False)
    sc.update(cand_kf=np.zeros(0, np.int32), cand_not_erase=np.zeros(0, np.uint8), slot_ptr=np.zeros(1, np.int64),
              slot_mp=np.zeros(0, np.int32), slot_octave=np.zeros(0, np.int32))
    h = api.keyframe_culling(sc, host=True)
    assert len(h["cull"]) == 0 and h["n_settled"] == 0


def _refused(sc, match):
    out = api.keyframe_culling_out(len(sc["cand_kf"]))
    for v in out.values():
        v.fill(7)
    with pytest.raises(api.CCMError, match=match):
        api.keyframe_culling(sc, host=True, out=out)
    for v in out.values():
        assert (v == 7).all()


def refused_cases():
    base = synth.make_keyframe_culling_scene(n_c=6, slots=200, seed=8, edges=False)
    K, P = len(base["kf_bad"]), len(base["mp_bad"])
    cases = []
    sc = dict(base, cand_kf=base["cand_kf"].copy()); sc["cand_kf"][3] = sc["cand_kf"][1]
    cases.append((sc, "candidate 3: keyframe row %d is already candidate 1" % sc["cand_kf"][1]))
    sc = dict(base, cand_kf=base["cand_kf"].copy()); sc["cand_kf"][2] = K
    cases.append((sc, "candidate 2: keyframe row %d out of range" % K))
    sc = dict(base, slot_mp=base["slot_mp"].copy()); sc["slot_mp"][base["slot_ptr"][4] + 5] = P
    cases.append((sc, "candidate 4, slot 5: point row %d out of range" % P))
    sc = dict(base, obs_kf=base["obs_kf"].copy()); sc["obs_kf"][base["obs_ptr"][9]] = -2
    cases.append((sc, "point 9: observer row -2 out of range"))
    sc = dict(base, mp_ref=base["mp_ref"].copy()); sc["mp_ref"][11] = K + 3
    cases.append((sc, "point 11: reference row %d out of range" % (K + 3)))
    return cases


@pytest.mark.parametrize("i", range(5))
def test_refused_input_writes_nothing(i):
    sc, msg = refused_cases()[i]
    _refused(sc, msg)


def test_null_array_is_refused():
    sc = synth.make_keyframe_culling_scene(n_c=4, slots=100, seed=9, edges=False)
    out = api.keyframe_culling_out(len(sc["cand_kf"]))
    argv, _keep = api.keyframe_culling_args(sc, out)
    for i, name in ((4, "null candidate array"), (13, "null observer array"), (9, "null point array")):
        a = list(argv); a[i] = None
        out["cull"].fill(7)
        assert api.lib().ccm_keyframe_culling_host(*a) == -1
        assert name in api.lib().ccm_last_error().decode() and (out["cull"] == 7).all()

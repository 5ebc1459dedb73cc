"""Keyframe database, CPU half (no device needed).

  * the oracle (oracle/kfdb_oracle.cpp) equals the reference's own Database.cpp + DBoW2 ScoringObject.cpp compiled in place
    (oracle/_ref/libkfdb_ref.so): returned vectors in order and every marker member bit for bit after every call, all three queries
    under all six scoring types, on every scene of tests/kfdb_scenes.py;
  * the oracle's scores equal an independent numpy restatement of D/ScoringObject.cpp, and its queries an independent restatement of
    S/Database.cpp's three steps;
  * ccm_kfdb_select (host code of the product) over the oracle's scored list returns the oracle's vector;
  * the golden fixture tests/golden/kfdb_queries.npz is reproduced;
  * without a device every ccm_kfdb_* device entry point returns CCM_ERR_NO_DEVICE.
"""
import math
import os

import numpy as np
import pytest

from ccm_slam_b200 import api
from ccm_slam_b200 import frontend as fe
from oracle import pykfdb

from tests.kfdb_scenes import SCORINGS, all_scenes, replay_checker

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "kfdb_queries.npz")
SCENES = all_scenes()


def np_score(scoring, w1, v1, w2, v2):
    """D/ScoringObject.cpp restated in plain Python floats (ascending common words; KL over every word of v1)"""
    d2 = dict(zip(w2.tolist(), v2.tolist()))
    s = 0.0
    if scoring == 3:
        last = int(w2[-1]) if len(w2) else -1
        eps = math.log(np.finfo(np.float64).eps)
        for w, vi in zip(w1.tolist(), v1.tolist()):
            if w in d2:
                if vi != 0 and d2[w] != 0:
                    s += vi * math.log(vi / d2[w])
            elif w < last or vi != 0:
                s += vi * (math.log(vi) - eps)
        return s
    for w, vi in zip(w1.tolist(), v1.tolist()):
        if w not in d2:
            continue
        wi = d2[w]
        if scoring == 0:
            s += abs(vi - wi) - abs(vi) - abs(wi)
        elif scoring == 2:
            if vi + wi != 0.0:
                s += vi * wi / (vi + wi)
        elif scoring == 4:
            s += math.sqrt(vi * wi)
        else:
            s += vi * wi
    if scoring == 0:
        return -s / 2.0
    if scoring == 1:
        return 1.0 if s >= 1 else 1.0 - math.sqrt(1.0 - s)
    return 2.0 * s if scoring == 2 else s


@pytest.mark.parametrize("scoring", SCORINGS)
def test_oracle_scores_equal_a_numpy_restatement(scoring):
    rng = np.random.default_rng(scoring)
    for t in range(40):
        w1 = np.unique(rng.integers(0, 300, rng.integers(0, 80))).astype(np.uint32)
        w2 = np.unique(np.concatenate([w1[rng.random(len(w1)) < 0.5], rng.integers(0, 300, rng.integers(0, 80))])).astype(np.uint32)
        v1 = rng.uniform(0.01, 1, len(w1)); v2 = rng.uniform(0.01, 1, len(w2))
        if t % 5 == 0 and len(v1):
            v1 /= v1.sum(); v2 /= max(v2.sum(), 1e-300)
        got = pykfdb.bow_score(scoring, w1, v1, w2, v2)
        ref = np_score(scoring, w1, v1, w2, v2)
        assert got == ref or (scoring == 3 and abs(got - ref) <= 1e-12 * abs(ref)), (t, got, ref)


def np_query(kfs, inv_lists, q_word, visible):
    """S/Database.cpp's first two steps restated: lKFsSharingWords order, shared-word counts, minCommonWords, the scored list"""
    order, cnt = [], {}
    for w in q_word.tolist():
        for u in inv_lists.get(w, []):
            if not visible(u):
                continue
            if u not in cnt:
                cnt[u] = 0; order.append(u)
            cnt[u] += 1
    if not order:
        return [], 0
    mx = max(cnt.values())
    mn = int(np.float32(mx) * np.float32(0.8))
    return [(u, cnt[u]) for u in order if cnt[u] > mn], mx


@pytest.mark.parametrize("name", sorted(SCENES))
def test_oracle_queries_equal_a_restatement_and_select(name):
    """scored lists against np_query; ccm_kfdb_select (host code of the product) over the oracle's scored list == the oracle"""
    scene = SCENES[name]
    rec = {k["uid"]: k for k in scene["kfs"]}
    for scoring in (0, 3):
        inv = {}
        for op, r, b in replay_checker(scene, scoring, pykfdb.Oracle):
            if op[0] == "add":
                for w in rec[op[1]]["word"].tolist():
                    inv.setdefault(w, []).append(op[1])
                continue
            if op[0] == "erase":
                for w in rec[op[1]]["word"].tolist():
                    if op[1] in inv.get(w, []):
                        inv[w].remove(op[1])
                continue
            s = b.last_scored()
            if op[0] == "loop":
                in_map, conn = set(op[4]), set(op[3])
                q = rec[op[1]]["word"]; vis = lambda u: u != op[1] and u in in_map and u not in conn
            elif op[0] == "mm":
                q = rec[op[1]]["word"]; vis = lambda u: rec[u]["client"] not in set(op[3])
            else:
                q = op[2]; vis = lambda u: True
            want, mx = np_query(rec, inv, np.asarray(q), vis)
            assert [u for u, _ in want] == s["uid"].tolist() and [c for _, c in want] == s["n_words"].tolist(), (name, op)
            assert s["max_common"] == mx
            qw, qv = (rec[op[1]]["word"], rec[op[1]]["value"]) if op[0] != "reloc" else (op[2], op[3])
            for u, sc in zip(s["uid"].tolist(), s["score_f64"].tolist()):
                assert sc == pykfdb.bow_score(scoring, qw, qv, rec[u]["word"], rec[u]["value"])
            cand = np.zeros(len(s["uid"]), fe.KFDB_CAND_DTYPE)
            cand["uid"], cand["n_words"], cand["score_f64"] = s["uid"], s["n_words"], s["score_f64"]
            cand["score"] = s["score_f64"].astype(np.float32)
            res = dict(cand=cand, n_sharing=s["n_sharing"], max_common=s["max_common"], min_common=s["min_common"])
            got = fe.KeyFrameDatabase.select(res, scene["covis"], op[0] == "reloc", op[2] if op[0] != "reloc" else 0.0)
            assert got.tolist() == r.tolist(), (name, op, got, r)


def _ref_or_skip():
    if not pykfdb.Reference.available():
        pytest.skip("oracle/_ref/libkfdb_ref.so is not built (needs the reference tree at build time)")


@pytest.mark.parametrize("scoring", SCORINGS)
@pytest.mark.parametrize("name", sorted(SCENES))
def test_oracle_equals_the_reference_database(name, scoring):
    _ref_or_skip()
    scene = SCENES[name]
    uids = sorted({k["uid"] for k in scene["kfs"]})
    mine = replay_checker(scene, scoring, pykfdb.Oracle)
    theirs = replay_checker(scene, scoring, pykfdb.Reference)
    for (op, r1, b1), (_, r2, b2) in zip(mine, theirs):
        if r1 is not None:
            assert r1.tolist() == r2.tolist(), (name, op)
        for u in uids:
            m1, m2 = b1.markers(u), b2.markers(u)
            assert np.array_equal(m1[0], m2[0]) and np.array_equal(m1[1], m2[1]), (name, op, u)
            assert m1[2].view(np.uint32).tolist() == m2[2].view(np.uint32).tolist(), (name, op, u)


def golden_results():
    """every query op of every scene under every scoring type: the returned uids and the scored list"""
    out = {}
    for name in sorted(SCENES):
        for scoring in SCORINGS:
            for i, (op, r, b) in enumerate(replay_checker(SCENES[name], scoring, pykfdb.Oracle)):
                if r is None:
                    continue
                s = b.last_scored()
                key = f"{name}/{scoring}/{i}"
                out[key + "/ret"] = r
                out[key + "/uid"] = s["uid"]; out[key + "/n_words"] = s["n_words"]; out[key + "/score"] = s["score_f64"]
    return out


def test_golden_fixture():
    g = np.load(GOLDEN)
    now = golden_results()
    assert sorted(g.files) == sorted(now)
    for k in g.files:
        if k.endswith("/score") and "/3/" in k:
            assert np.allclose(g[k], now[k], rtol=1e-12, atol=0), k
        else:
            assert np.array_equal(g[k], now[k]), k


def test_kfdb_needs_a_device():
    if api.device_count() > 0:
        pytest.skip("a device is present")
    import ctypes as C
    L = api.lib()
    h = C.c_void_p()
    assert L.ccm_kfdb_create(100, 0, C.byref(h)) == -2          # CCM_ERR_NO_DEVICE
    with pytest.raises(api.CCMError) as e:
        fe.KeyFrameDatabase(100)
    assert e.value.code == -2
    # host only: the selection runs without a device
    cand = np.zeros(2, fe.KFDB_CAND_DTYPE)
    cand["uid"] = [5, 6]; cand["score"] = [0.5, 0.4]
    got = fe.KeyFrameDatabase.select(dict(cand=cand, n_sharing=2, max_common=3, min_common=2), {5: [6], 6: [5]}, False, 0.1)
    assert got.tolist() == [5]

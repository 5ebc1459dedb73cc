"""Keyframe database on the device (ccm_kfdb_*) against the oracle, which tests/test_kfdb_cpu.py pins to the reference's own
Database.cpp: candidates (uids, order, shared words), f64 scores bit for bit (KL within 1e-12 relative), returned vectors, batched
queries, add / erase / re-add order, the golden fixture, and one end-to-end place-recognition chain."""
import os

import numpy as np
import pytest

from ccm_slam_b200 import api
from ccm_slam_b200 import frontend as fe
from ccm_slam_b200 import synth_match as sm
from oracle import pykfdb
from tests.kfdb_scenes import SCORINGS, all_scenes, replay_checker, replay_device

pytestmark = pytest.mark.gpu
SCENES = all_scenes()
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "kfdb_queries.npz")


def _same_scores(scoring, got, want):
    if scoring == 3:
        return np.allclose(got, want, rtol=1e-12, atol=0)
    return np.array_equal(got.view(np.uint64), np.asarray(want, np.float64).view(np.uint64))


@pytest.mark.parametrize("scoring", SCORINGS)
def test_device_queries_equal_the_oracle(scoring):
    api.init(0)
    for name, scene in sorted(SCENES.items()):
        db = fe.KeyFrameDatabase(scene["n_words"], scoring)
        for (op, r, b), (_, rd, raw) in zip(replay_checker(scene, scoring, pykfdb.Oracle), replay_device(scene, scoring, db)):
            if r is None:
                continue
            s = b.last_scored()
            c = raw["cand"]
            assert c["uid"].tolist() == s["uid"].tolist() and c["n_words"].tolist() == s["n_words"].tolist(), (name, op)
            assert raw["max_common"] == s["max_common"] and raw["min_common"] == s["min_common"] and raw["n_sharing"] == s["n_sharing"]
            assert _same_scores(scoring, c["score_f64"], s["score_f64"]), (name, op)
            if scoring != 3:
                assert rd.tolist() == r.tolist(), (name, op)
        db.close()


def test_batch_equals_sequential_and_score_many():
    api.init(0)
    d = sm.make_place_db(n_clients=4, kf_per_client=80, n_words=8000, local_words=90, bg_words=40, pool=200, seed=3)
    for scoring in (0, 3, 4):
        db = fe.KeyFrameDatabase(d["n_words"], scoring)
        for k in range(len(d["uid"])):
            db.add(d["uid"][k], d["client"][k], *sm.place_db_bow(d, k))
        rows = list(range(0, len(d["uid"]), 5))
        reqs = [db.request(*sm.place_db_bow(d, k), client_mask=~(1 << int(d["client"][k])) & fe.ALL_CLIENTS) for k in rows]
        reqs += [db.request(*sm.place_db_bow(d, k), exclude=[d["uid"][k], d["uid"][k - 1]]) for k in rows[1:10]]
        batch = db.query_batch(reqs)
        for rq, got in zip(reqs, batch):
            keep = rq[1]
            one = db.query(keep["w"], keep["v"], rq[0].client_mask, keep["x"])
            assert got["cand"].tobytes() == one["cand"].tobytes()
            assert (got["max_common"], got["n_sharing"]) == (one["max_common"], one["n_sharing"])
        assert sum(len(b["cand"]) for b in batch) > 50
        w, v = sm.place_db_bow(d, 7)
        uids = d["uid"][::3]
        sc = db.score_many(w, v, uids)
        idx = {int(u): k for k, u in enumerate(d["uid"])}
        want = np.array([pykfdb.bow_score(scoring, w, v, *sm.place_db_bow(d, idx[int(u)])) for u in uids])
        assert _same_scores(scoring, sc, want)
        db.close()


def test_interleaved_add_erase_readd_keeps_the_reference_order():
    """many rounds of erase / re-add on long lists (segments move and compact) -> candidate order of the reference's lists"""
    api.init(0)
    rng = np.random.default_rng(11)
    n_words, K = 300, 400
    recs = []
    for u in range(1, K + 1):
        w = np.unique(np.concatenate([rng.integers(0, 20, 8), rng.integers(0, n_words, 25)])).astype(np.uint32)
        v = rng.uniform(0.1, 1, len(w)); recs.append((u, u % 3, w, v / v.sum()))
    db = fe.KeyFrameDatabase(n_words, 0)
    orc = pykfdb.Oracle(n_words, 0)
    for u, c, w, v in recs:
        orc.keyframe(u, c, w, v)
    live = set()
    fid = 10_000
    for rnd in range(12):
        for u, c, w, v in recs:
            if u in live and rng.random() < 0.3:
                db.erase(u); orc.erase(u); live.discard(u)
            elif u not in live and rng.random() < 0.6:
                db.add(u, c, w, v); orc.add(u); live.add(u)
        for q in rng.choice(K, size=3, replace=False):
            _, _, w, v = recs[q]
            fid += 1
            got = db.query(w, v)
            orc.DetectRelocalizationCandidates(fid, w, v)          # the scored list does not read earlier markers
            s = orc.last_scored()
            assert got["cand"]["uid"].tolist() == s["uid"].tolist() and got["cand"]["n_words"].tolist() == s["n_words"].tolist()
            assert _same_scores(0, got["cand"]["score_f64"], s["score_f64"])
    assert db.size() == len(live)
    db.clear()
    assert db.size() == 0 and len(db.query(recs[0][2], recs[0][3])["cand"]) == 0


def test_golden_fixture_through_the_c_abi():
    api.init(0)
    g = np.load(GOLDEN)
    n = 0
    for name, scene in sorted(SCENES.items()):
        for scoring in SCORINGS:
            db = fe.KeyFrameDatabase(scene["n_words"], scoring)
            for i, (op, rd, raw) in enumerate(replay_device(scene, scoring, db)):
                if raw is None:
                    continue
                key = f"{name}/{scoring}/{i}"
                assert raw["cand"]["uid"].tolist() == g[key + "/uid"].tolist() and raw["cand"]["n_words"].tolist() == g[key + "/n_words"].tolist()
                assert _same_scores(scoring, raw["cand"]["score_f64"], g[key + "/score"]), key
                if scoring != 3:
                    assert rd.tolist() == g[key + "/ret"].tolist(), key
                n += 1
            db.close()
    assert n > 100


def test_end_to_end_place_recognition_chain(oracle):
    """kfstore_transform -> kfdb add -> DetectLoopCandidates -> kfstore SearchByBoW(kf, kf), against the oracle chain"""
    api.init(0)
    voc = sm.make_vocabulary(k=6, L=3, seed=31)
    V = fe.ORBVocabulary(voc); R = oracle.Vocabulary(voc)
    st = fe.KeyFrameStore()
    rng = np.random.default_rng(5)
    base = [sm.make_voc_features(voc, n=400, seed=100 + p) for p in range(6)]
    descs, clients = [], []
    for u in range(1, 25):
        d = base[(u - 1) % 6].copy()
        flip = rng.integers(0, 256, size=(len(d), 2)); d[np.arange(len(d)), flip[:, 0] % 32] ^= (1 << (flip[:, 1] % 8)).astype(np.uint8)
        descs.append(d); clients.append(u % 2)
    kps = np.zeros(400, fe.KP_DTYPE); kps["angle"] = rng.uniform(0, 360, 400).astype(np.float32)
    n_words = V.words()
    db = fe.KeyFrameDatabase(n_words, 0)
    orc = pykfdb.Oracle(n_words, 0)
    bows = {}
    for u, d in enumerate(descs, start=1):
        st.put(u, kps, d)
        t = st.transform(u, V, 1); r = R.transform(d, 1)
        assert np.array_equal(t["bow_id"], r["bow_id"]) and np.array_equal(t["bow_val"], r["bow_val"])
        bows[u] = t
        orc.keyframe(u, clients[u - 1], r["bow_id"], r["bow_val"])
    covis = {u: [v for v in range(max(1, u - 3), u + 4) if v != u and v <= 24 and clients[v - 1] == clients[u - 1]] for u in bows}
    for u, nb in covis.items():
        orc.set_covis(u, nb)
    q = 24
    for u in range(1, q):
        db.add(u, clients[u - 1], bows[u]["bow_id"], bows[u]["bow_val"]); orc.add(u)
    in_map = [u for u in range(1, 25) if clients[u - 1] == clients[q - 1] and u not in (2, 6)]   # 2, 6: in the database, not in the map
    connected = covis[q]
    got = db.DetectLoopCandidates(q, bows[q]["bow_id"], bows[q]["bow_val"], 0.01, connected, in_map, covis)
    want = orc.DetectLoopCandidates(q, 0.01, connected, in_map)
    assert got.tolist() == want.tolist() and len(got) >= 1
    has = np.ones(400, np.uint8)
    for c in got.tolist():
        fq, fc = fe.FeatureVector(bows[q]["node"]), fe.FeatureVector(bows[c]["node"])
        m, n = st.SearchByBoW_KF_KF(q, has, fq, c, has, fc, 0.75, True)
        rm, rn = oracle.match_bow_kf_kf(descs[q - 1], has, kps["angle"], oracle.FeatureVector(bows[q]["node"]), descs[c - 1], has, kps["angle"],
                                        oracle.FeatureVector(bows[c]["node"]), 0.75, True)
        assert n == rn and np.array_equal(m, rm) and n > 10
    V.close(); R.close(); st.close(); db.close()

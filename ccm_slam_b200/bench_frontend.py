"""Front-end timings for bench.py: ms per frame / per call of the ORB extractor and the two BoW-guided matchers of the north-star path,
through the C ABI with HOST buffers (copies inside the timed region — these are latency-bound per-frame calls, SURVEY.md §7), next to
the CPU oracle on the same inputs when an oracle module is passed in.

  ORBextractor::operator()        S/ORBextractor.cpp:1216-1278   752 x 480, 1000 features, 8 levels (cslam/conf/config.yaml:38-51)
  ORBmatcher::SearchByBoW         S/ORBmatcher.cpp:178-306       keyframe (≈1000 features) against frame
  ORBmatcher::SearchForTriangulation  S/ORBmatcher.cpp:700-852   keyframe pair, epipolar gate

Plumbing only: every timed call is the product's own entry point.
"""
from __future__ import annotations

import statistics
import threading
import time

import numpy as np

from . import synth
from .frontend import FeatureVector, ORBextractor, ORBmatcher
from .synth_images import make_image


def _median_ms(fn, reps, warm=2):
    for _ in range(warm):
        fn()
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter(); fn(); ts.append((time.perf_counter() - t0) * 1e3)
    return statistics.median(ts)


def run(oracle=None, reps=30, cpu_reps=3):
    out = {"unit": "ms (median)", "image": "752x480 synthetic (seeded value noise + rectangles), 1000 features, 8 levels, scale 1.2",
           "note": "host buffers, H2D/D2H inside every timed call; cpu = the oracle port, single thread"}
    imgs = [make_image(s) for s in range(4)]
    ex = ORBextractor()
    k1, d1 = ex(imgs[0])
    it = [0]

    def one():
        it[0] += 1
        ex(imgs[it[0] % 4])
    out["orb_extract_ms_per_frame"] = _median_ms(one, reps, warm=3)
    out["orb_keypoints"] = int(len(k1))
    # four agents at once: one extractor (own stream) per agent, one host thread each, as the four client front ends would call it
    exs = [ORBextractor() for _ in range(4)]
    for e, im in zip(exs, imgs):
        e(im)

    def four():
        th = [threading.Thread(target=lambda e=e, im=im: [e(im) for _ in range(5)]) for e, im in zip(exs, imgs)]
        for t in th: t.start()
        for t in th: t.join()
    out["orb_extract_4_agents_ms_per_frame"] = _median_ms(four, max(3, reps // 6), warm=1) / 20.0
    for e in exs:
        e.close()
    # matchers on two views of one scene (a shifted copy: many true matches)
    b = np.roll(imgs[0], (3, 5), axis=(0, 1))
    k2, d2 = ex(b)
    ex.close()
    rng = np.random.default_rng(1)
    node = lambda d: (d[:, 0].astype(np.int64) * 7 + d[:, 1] // 64) % 97   # ~100 vocabulary nodes like DBoW2 at levelsup = 4
    fv1, fv2 = FeatureVector(node(d1)), FeatureVector(node(d2))
    has1 = (rng.random(len(k1)) < 0.7).astype(np.uint8); has2 = (rng.random(len(k2)) < 0.7).astype(np.uint8)
    m = ORBmatcher(0.7, True)
    got_b, n_b = m.SearchByBoW_KF_Frame(d1, has1, k1["angle"], fv1, d2, k2["angle"], fv2)
    out["search_by_bow_ms_per_call"] = _median_ms(lambda: m.SearchByBoW_KF_Frame(d1, has1, k1["angle"], fv1, d2, k2["angle"], fv2), reps)
    out["search_by_bow_matches"] = int(n_b)
    fx, fy, cx, cy = [np.float32(v) for v in synth.EUROC_INTR]
    Kinv = np.linalg.inv(np.array([[fx, 0, cx], [0, fy, cy], [0, 0, 1]], np.float64))
    tx = np.array([[0, 0, 0], [0, 0, -1.0], [0, 1.0, 0]])
    F12 = (Kinv.T @ tx @ Kinv).astype(np.float32)
    sf = (1.2 ** np.arange(8)).astype(np.float32); ls2 = (sf * sf).astype(np.float32)
    v = lambda k, d, has, fv: dict(desc=d, has_mp=has, kp_xy=np.stack([k["x"], k["y"]], 1), octave=k["octave"], angle=k["angle"], fv=fv,
                                   intr=(fx, fy, cx, cy))
    mt = ORBmatcher(0.6, False)
    got_t = mt.SearchForTriangulation(v(k1, d1, has1, fv1), v(k2, d2, has2, fv2), F12, -5000.0, float(cy), ls2, sf)
    out["search_for_triangulation_ms_per_call"] = _median_ms(
        lambda: mt.SearchForTriangulation(v(k1, d1, has1, fv1), v(k2, d2, has2, fv2), F12, -5000.0, float(cy), ls2, sf), reps)
    out["search_for_triangulation_matches"] = int(len(got_t))
    if oracle is not None:
        rk, rd = oracle.orb_extract(imgs[0])
        out["cpu_orb_extract_ms_per_frame"] = _median_ms(lambda: oracle.orb_extract(imgs[1]), cpu_reps, warm=0)
        ofv1, ofv2 = oracle.FeatureVector(node(d1)), oracle.FeatureVector(node(d2))
        ref_b, rn = oracle.match_bow_kf_frame(d1, has1, k1["angle"], ofv1, d2, k2["angle"], ofv2, 0.7, True)
        out["cpu_search_by_bow_ms_per_call"] = _median_ms(
            lambda: oracle.match_bow_kf_frame(d1, has1, k1["angle"], ofv1, d2, k2["angle"], ofv2, 0.7, True), cpu_reps * 3, warm=1)
        ref_t = oracle.match_triangulation(v(k1, d1, has1, ofv1), v(k2, d2, has2, ofv2), F12, -5000.0, float(cy), ls2, sf, False)
        out["cpu_search_for_triangulation_ms_per_call"] = _median_ms(
            lambda: oracle.match_triangulation(v(k1, d1, has1, ofv1), v(k2, d2, has2, ofv2), F12, -5000.0, float(cy), ls2, sf, False),
            cpu_reps * 3, warm=1)
        out["parity"] = {"orb_bit_exact": bool(len(rk) == len(k1) and np.array_equal(rd, d1) and np.array_equal(rk["x"], k1["x"])),
                         "bow_indices_equal": bool(rn == n_b and np.array_equal(ref_b, got_b)),
                         "triangulation_indices_equal": bool(np.array_equal(ref_t, got_t))}
    kb = kfdb_block(oracle, reps)
    parity = kb.pop("parity", {})
    out.update(kb)
    if parity:
        out.setdefault("parity", {}).update(parity)
    return out


def _spread(ts):
    q = np.percentile(ts, [10, 50, 90])
    return dict(p10=float(q[0]), median=float(q[1]), p90=float(q[2]), n=len(ts))


def _card():
    import subprocess
    name, plim = None, None
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True,
                           text=True, timeout=20)
        name, plim = [x.strip() for x in r.stdout.strip().splitlines()[0].split(",")]
    except Exception:
        pass
    return name, plim


def kfdb_block(oracle=None, reps=30):
    """DetectLoopCandidates on a server-shaped database (4 agents x 2500 keyframes, ~660 words each, 200 k-word vocabulary): one
    query per call (ccm_kfdb_query + ccm_kfdb_select, host buffers), a batch of 64 queries, CUDA-event time of the kernels, and the
    CPU oracle port of S/Database.cpp on the same database."""
    import importlib
    from . import synth_match as sm
    from .frontend import KeyFrameDatabase
    d = sm.make_place_db(n_clients=4, kf_per_client=2500, n_words=200000, local_words=400, bg_words=150, pool=1200, seed=5)
    K = len(d["uid"])
    idx = {int(u): k for k, u in enumerate(d["uid"])}
    covis = lambda u: sm.place_db_covis(d, idx[int(u)])
    db = KeyFrameDatabase(d["n_words"], 0)
    for k in range(K):
        db.add(d["uid"][k], d["client"][k], *sm.place_db_bow(d, k))
    rows = [K - 1 - i for i in range(64)]
    reqs, mins, info = [], [], []
    for k in rows:
        w, v = sm.place_db_bow(d, k)
        nb = sm.place_db_covis(d, k)
        ms = float(np.float32(db.score_many(w, v, nb).min()) * np.float32(0.8)) if len(nb) else 0.0   # LoopFinder.cpp:125-142
        reqs.append(db.request(w, v, 1 << int(d["client"][k]), np.concatenate([[d["uid"][k]], nb]).astype(np.uint64)))
        mins.append(ms); info.append((int(d["uid"][k]), nb))
    i = [0]

    def one():
        j = i[0] % len(reqs); i[0] += 1
        return db.select(db.query_batch([reqs[j]])[0], covis, False, mins[j])
    for _ in range(5):
        one()
    ts = []
    for _ in range(max(reps, 50)):
        t0 = time.perf_counter(); one(); ts.append((time.perf_counter() - t0) * 1e3)
    out = {"kfdb_query_ms_per_call": statistics.median(ts), "kfdb_query_ms_spread": _spread(ts)}
    db.query_batch(reqs)
    tb = []
    for _ in range(10):
        t0 = time.perf_counter()
        res = db.query_batch(reqs)
        for r, ms in zip(res, mins):
            db.select(r, covis, False, ms)
        tb.append((time.perf_counter() - t0) * 1e3 / len(reqs))
    out["kfdb_query_batch_ms_per_query"] = statistics.median(tb)
    out["kfdb_query_batch_spread"] = _spread(tb)
    out["kfdb_batch"] = len(reqs)
    db.set_timing(True)
    for _ in range(3):
        db.query_batch([reqs[0]])
    tc, tsc, nq = db.timing()
    db.set_timing(True)
    db.query_batch(reqs)
    bc, bsc, bn = db.timing()
    db.set_timing(False)
    out["kfdb_kernel_ms_per_query"] = {"count": tc / nq, "score": tsc / nq, "batch64_count": bc / bn, "batch64_score": bsc / bn}
    first = db.query_batch([reqs[0]])[0]
    out["kfdb_database"] = {"keyframes": K, "clients": 4, "postings": int(len(d["bow_word"])), "vocabulary": d["n_words"],
                            "query_candidates_scored": int(len(first["cand"])), "query_sharing": int(first["n_sharing"])}
    name, plim = _card()
    out["kfdb_card"] = {"name": name, "power_limit": plim}
    if oracle is not None:
        pk = importlib.import_module(oracle.__name__.rsplit(".", 1)[0] + ".pykfdb")
        o = pk.Oracle(d["n_words"], 0)
        for k in range(K):
            o.keyframe(d["uid"][k], d["client"][k], *sm.place_db_bow(d, k))
            o.set_covis(d["uid"][k], sm.place_db_covis(d, k))
        for k in range(K):
            o.add(d["uid"][k])
        by_client = {c: d["uid"][d["client"] == c] for c in range(4)}
        equal = True
        tc = []
        for j, k in enumerate(rows[:16]):
            uid, nb = info[j]
            t0 = time.perf_counter()
            want = o.DetectLoopCandidates(uid, mins[j], nb, by_client[int(d["client"][k])])
            tc.append((time.perf_counter() - t0) * 1e3)
            got = db.select(db.query_batch([reqs[j]])[0], covis, False, mins[j])
            equal = equal and got.tolist() == want.tolist()
        out["cpu_kfdb_query_ms_per_call"] = statistics.median(tc)
        out["cpu_kfdb_query_ms_spread"] = _spread(tc)
        out.setdefault("parity", {})["kfdb_candidates_equal"] = bool(equal)
        o.close()
    db.close()
    return out

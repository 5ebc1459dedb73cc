"""Scenes for the keyframe-database tests: keyframe records, covisibility lists and a sequence of database operations, replayed on
the oracle (oracle/pykfdb.Oracle), on the reference's own Database.cpp (pykfdb.Reference) and on the device (KeyFrameDatabase).

An op is ("add", uid) | ("erase", uid) | ("loop", q_uid, min_score, connected, in_map) | ("mm", q_uid, min_score, assoc_clients)
| ("reloc", frame_id, word, value).  Every (kind, query id) is queried once per scene, as LoopFinder / MapMatcher / Tracking do; a
scene holds at most one relocalisation query (the reference reads mRelocScore left by earlier relocalisation queries, DESIGN.md §5).
"""
import numpy as np

from ccm_slam_b200 import synth_match as sm

SCORINGS = (0, 1, 2, 3, 4, 5)   # L1, L2, ChiSquare, KL, Bhattacharyya, DotProduct


def _rec(uid, client, words, rng, lo=0.2, hi=3.0):
    w = np.unique(np.asarray(words, np.uint32))
    v = rng.uniform(lo, hi, len(w))
    return dict(uid=uid, client=client, word=w, value=v / v.sum())


def hand_scenes():
    """small scenes, one per situation the reference code distinguishes"""
    rng = np.random.default_rng(7)
    out = {}
    # an empty database; a query that shares no word
    q = _rec(1, 0, range(0, 30), rng)
    out["empty"] = dict(n_words=200, kfs=[q], covis={}, ops=[("loop", 1, 0.0, [], [1]), ("mm", 1, 0.0, [0]),
                                                           ("reloc", 900, q["word"], q["value"])])
    kfs = [q, _rec(2, 0, range(100, 140), rng), _rec(3, 1, range(140, 180), rng)]
    out["no_shared_word"] = dict(n_words=200, kfs=kfs, covis={}, ops=[("add", 2), ("add", 3), ("loop", 1, 0.0, [], [1, 2]),
                                                                      ("mm", 1, 0.0, [0]), ("reloc", 901, q["word"], q["value"])])
    # the 0.8 truncation at its boundary: max = 10 -> minCommonWords = 8; 9 shared words are scored, 8 are not
    q = _rec(1, 0, range(0, 10), rng)
    kfs = [q, _rec(2, 0, list(range(0, 10)) + [50, 51], rng), _rec(3, 0, list(range(0, 9)) + [52], rng),
           _rec(4, 0, list(range(0, 8)) + [53, 54], rng), _rec(5, 1, list(range(1, 10)), rng), _rec(6, 1, range(0, 8), rng)]
    covis = {2: [3, 4], 3: [2], 4: [2, 3], 5: [6], 6: [5]}
    out["truncation"] = dict(n_words=100, kfs=kfs, covis=covis, ops=[("add", k) for k in (2, 3, 4, 5, 6)] + [
        ("loop", 1, 0.0, [], [1, 2, 3, 4]), ("mm", 1, 0.0, [0]), ("loop", 1001, 10.0, [], [1001]), ("reloc", 902, q["word"], q["value"])])
    out["truncation"]["kfs"].append(dict(q, uid=1001))
    # everything below minScore
    out["below_min_score"] = dict(n_words=100, kfs=[dict(k) for k in kfs[:6]], covis=covis, ops=[("add", k) for k in (2, 3, 4, 5, 6)] + [
        ("loop", 1, 2.0, [], [1, 2, 3, 4]), ("mm", 1, 2.0, [0])])
    # ties: identical BowVectors -> equal scores and equal accumulated scores; one neighbour is the best of two candidates
    base = _rec(10, 0, range(20, 60), rng)
    kfs = [dict(base, uid=1, client=0)] + [dict(base, uid=u, client=c) for u, c in ((11, 0), (12, 0), (13, 1), (14, 1))] + [
        _rec(15, 0, list(range(20, 50)) + [90], rng), _rec(16, 1, list(range(25, 60)), rng)]
    covis = {11: [15, 12], 12: [15, 11], 13: [16, 14], 14: [16, 13], 15: [11, 12], 16: [13, 14]}
    out["ties_and_shared_best"] = dict(n_words=100, kfs=kfs, covis=covis, ops=[("add", k) for k in (11, 12, 13, 14, 15, 16)] + [
        ("loop", 1, 0.0, [], [1, 11, 12, 15]), ("mm", 1, 0.0, [0]), ("reloc", 903, base["word"], base["value"])])
    # connected keyframes (counted as 1 word by the reference, never listed), keyframes outside the map / of other clients
    kfs = [_rec(1, 0, range(0, 40), rng)] + [_rec(u, u % 3, list(range(0, 40, 1 + u % 4)) + [60 + u], rng) for u in range(2, 14)]
    covis = {u: [v for v in range(2, 14) if v != u][:10] for u in range(2, 14)}
    out["connected_other_maps"] = dict(n_words=100, kfs=kfs, covis=covis, ops=[("add", u) for u in range(2, 14)] + [
        ("loop", 1, 0.0, [3, 6], [1, 3, 5, 6, 8, 9, 11]), ("mm", 1, 0.0, [0, 2])])
    # erase mid-sequence, then re-add: a re-added keyframe moves to the end of its lists
    kfs = [_rec(1, 0, range(0, 20), rng)] + [_rec(u, 1, list(range(0, 20, 1 + u % 3)) + [30 + u], rng) for u in range(2, 10)]
    covis = {u: [v for v in range(2, 10) if v != u] for u in range(2, 10)}
    out["erase_readd"] = dict(n_words=100, kfs=kfs + [dict(kfs[0], uid=101), dict(kfs[0], uid=102)], covis=covis, ops=
                              [("add", u) for u in range(2, 10)] + [("erase", 4), ("erase", 2), ("mm", 1, 0.0, [0]), ("add", 2),
                                                                   ("erase", 7), ("add", 4), ("mm", 101, 0.0, [0]), ("erase", 4),
                                                                   ("erase", 4), ("add", 4), ("mm", 102, 0.0, [0])])
    return out


def generated_scenes(seed=0, n_queries=6):
    """make_place_db(): several agents, revisits, cross-agent overlap; loop / map-match queries for the last keyframes of each agent
    (each is in the database; its covisibility list is its connected set; a few keyframes of its agent are left out of the map), and
    one scene per relocalisation query"""
    db = sm.make_place_db(n_clients=3, kf_per_client=40, n_words=5000, local_words=60, bg_words=25, pool=150, seed=seed)
    rng = np.random.default_rng(seed + 1)
    K = len(db["uid"])
    kfs = []
    for k in range(K):
        w, v = sm.place_db_bow(db, k)
        kfs.append(dict(uid=int(db["uid"][k]), client=int(db["client"][k]), word=w, value=v))
    covis = {int(db["uid"][k]): [int(u) for u in sm.place_db_covis(db, k)] for k in range(K)}
    ops = [("add", int(u)) for u in db["uid"]]
    qrows = rng.choice(np.arange(K // 2, K), size=n_queries, replace=False)
    for j, k in enumerate(qrows):
        uid, c = int(db["uid"][k]), int(db["client"][k])
        same = [int(u) for u, cc in zip(db["uid"], db["client"]) if cc == c]
        in_map = [u for u in same if rng.random() > 0.1] + [uid]
        ops.append(("loop", uid, float([0.0, 0.01, 0.02][j % 3]), covis[uid], in_map))
        ops.append(("mm", uid, float([0.0, 0.015][j % 2]), [c]))
        if j == n_queries // 2:
            ops += [("erase", int(u)) for u in db["uid"][::7]] + [("add", int(u)) for u in db["uid"][::14]]
    scenes = {"place_db": dict(n_words=db["n_words"], kfs=kfs, covis=covis, ops=ops)}
    for j, k in enumerate(qrows[:3]):
        w, v = sm.place_db_bow(db, k)
        scenes[f"place_db_reloc{j}"] = dict(n_words=db["n_words"], kfs=kfs, covis=covis, ops=[("add", int(u)) for u in db["uid"]] +
                                            [("reloc", 5000 + j, w, v)])
    return scenes


def all_scenes():
    s = hand_scenes()
    s.update(generated_scenes())
    return s


def replay_checker(scene, scoring, make):
    """replay on a pykfdb backend (Oracle / Reference); yields (op, returned uids, backend) after every op"""
    b = make(scene["n_words"], scoring)
    for k in scene["kfs"]:
        b.keyframe(k["uid"], k["client"], k["word"], k["value"])
    for u, nb in scene["covis"].items():
        b.set_covis(u, nb)
    for op in scene["ops"]:
        r = None
        if op[0] == "add":
            b.add(op[1])
        elif op[0] == "erase":
            b.erase(op[1])
        elif op[0] == "loop":
            r = b.DetectLoopCandidates(op[1], op[2], op[3], op[4])
        elif op[0] == "mm":
            r = b.DetectMapMatchCandidates(op[1], op[2], op[3])
        else:
            r = b.DetectRelocalizationCandidates(op[1], op[2], op[3])
        yield op, r, b
    b.close()


def replay_device(scene, scoring, db):
    """replay on the device database `db` (KeyFrameDatabase, empty) through its Detect* methods; yields (op, returned uids, the device
    result of the query or None)"""
    rec = {k["uid"]: k for k in scene["kfs"]}
    covis = scene["covis"]
    for op in scene["ops"]:
        if op[0] == "add":
            k = rec[op[1]]
            if op[1] not in db.client_of:          # the reference would list it twice; the device refuses a second add
                db.add(k["uid"], k["client"], k["word"], k["value"])
            yield op, None, None
        elif op[0] == "erase":
            db.erase(op[1])
            yield op, None, None
        elif op[0] == "loop":                       # the public methods: visibility, exclusions and selection are theirs
            q = rec[op[1]]
            got = db.DetectLoopCandidates(op[1], q["word"], q["value"], op[2], op[3], op[4], covis)
            yield op, got, db.last_result
        elif op[0] == "mm":
            q = rec[op[1]]
            got = db.DetectMapMatchCandidates(q["word"], q["value"], op[2], op[3], covis)
            yield op, got, db.last_result
        else:
            got = db.DetectRelocalizationCandidates(op[2], op[3], covis)
            yield op, got, db.last_result

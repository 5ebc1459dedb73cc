"""Generates tests/golden/covisibility.npz: the counter and ordered connections of KeyFrame::UpdateConnections
(cslam/src/KeyFrame.cpp:629-711) on hand-made edge cases, tie storms and random scenes.  The fixture stores each case's inputs (the
keys of synth.make_covisibility) and the answer in the flat layout of ccm_covisibility (conn_ptr, conn_kf, conn_w, n_sel, sel_kf,
sel_w, status).  The answer is the pure-Python witness below (a dict per keyframe, sorted()); the generator refuses to write unless
the oracle (oracle/covis_oracle.cpp) agrees on every case.  Run from the repo root:
    python tests/golden/make_covisibility_golden.py
"""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", ".."))
from ccm_slam_b200 import synth  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(HERE, "covisibility.npz")
IN_KEYS = ("kf_id", "kf_rank", "kf_bad", "mvp_ptr", "mvp", "mp_bad", "obs_ptr", "obs_kf", "obs_idx", "batch")
OUT_KEYS = ("conn_ptr", "conn_kf", "conn_w", "n_sel", "sel_kf", "sel_w", "status")
NAMES = ("edges", "storm", "random", "maps")
# the rows of "edges", by what they exercise (hand_edges below)
EDGE_ROWS = dict(no_points=0, all_bad=1, only_self=2, same_id=3, below_tie=4, at_14_15=9, duplicate=13, bad_observer=16)


def witness(sc, th=15, skip_bad_observers=False, strict=False, ascending_ties=False, last_max=False, self_by_row=False):
    """pure Python; the keyword arguments are the slips the tests must catch"""
    rank = [int(r) for r in sc["kf_rank"]]
    row_of = {r: k for k, r in enumerate(rank)}
    ids = [int(i) for i in sc["kf_id"]]
    o = {k: [] for k in OUT_KEYS}
    o["conn_ptr"].append(0)
    for self in (int(b) for b in sc["batch"]):
        counter = {}
        for p in sc["mvp"][sc["mvp_ptr"][self]:sc["mvp_ptr"][self + 1]]:
            if p < 0 or sc["mp_bad"][p]:
                continue
            for k in (int(k) for k in sc["obs_kf"][sc["obs_ptr"][p]:sc["obs_ptr"][p + 1]]):
                if (k == self) if self_by_row else (ids[k] == ids[self]):
                    continue
                if skip_bad_observers and sc["kf_bad"][k]:
                    continue
                counter[rank[k]] = counter.get(rank[k], 0) + 1
        items = sorted(counter.items())
        base = len(o["conn_kf"])
        for r, w in items:
            o["conn_kf"].append(row_of[r]); o["conn_w"].append(w); o["sel_kf"].append(-1); o["sel_w"].append(0)
        sel = [(w, r) for r, w in items if (w > th if strict else w >= th)]
        sel = sorted(sel, key=lambda e: (-e[0], e[1])) if ascending_ties else sorted(sel, reverse=True)
        if not sel and items:
            nmax, best = 0, None
            for r, w in items:
                if w > nmax or (last_max and w == nmax):
                    nmax, best = w, r
            sel = [(nmax, best)]
        for i, (w, r) in enumerate(sel):
            o["sel_kf"][base + i] = row_of[r]; o["sel_w"][base + i] = w
        o["n_sel"].append(len(sel)); o["status"].append(1 if items else 0)
        o["conn_ptr"].append(len(o["conn_kf"]))
    dt = dict(conn_ptr=np.int64, conn_kf=np.int32, conn_w=np.int32, n_sel=np.int32, sel_kf=np.int32, sel_w=np.int32, status=np.uint8)
    return {k: np.array(v, dt[k]) for k, v in o.items()}


def hand_edges():
    """one scene, a row per edge case (EDGE_ROWS); ranks shuffled"""
    rng = np.random.default_rng(31)
    K = 20
    pk, pm, extra_k, extra_m = [], [], [], []
    P = [0]

    def point(observers):
        p = P[0]; P[0] += 1
        pk.extend(observers); pm.extend([p] * len(observers))
        return p
    # row 0: no points.  Row 1: every point bad (points 0..4, listed below as bad)
    bad = [point([1, 5, 6]) for _ in range(5)]
    # rows 2 and 3 share an mId: row 2's points are seen by row 2 and row 3 only
    for _ in range(6):
        point([2, 3])
    # row 4: weights 9, 9, 9, 5 (rows 5, 6, 7, 8): below 15, a three-way tie at the maximum
    for j in range(9):
        point([4, 5, 6, 7] + ([8] if j < 5 else []))
    # row 9: weights 15 (row 10), 14 (row 11), 15 (row 12), and 15 for row 16 which is bad
    for j in range(15):
        point([9, 10, 12, 16] + ([11] if j < 14 else []))
    # row 13: one point at two indices, seen by rows 13 and 14; another seen by 13, 14, 15
    dup = point([13, 14])
    point([13, 14, 15])
    extra_k.append(13); extra_m.append(dup)
    kf_id = np.arange(K, dtype=np.uint64); kf_id[3] = kf_id[2]
    sc = synth.covis_pack(K, pk, pm, P[0], rng, kf_id=kf_id, extra=(extra_k, extra_m), null_frac=0.2)
    sc["mp_bad"][:] = 0; sc["mp_bad"][bad] = 1
    sc["kf_bad"][:] = 0; sc["kf_bad"][16] = 1
    return sc


def storm(seed=32):
    """tie storms: 14 keyframes, every point seen by the same few, so that whole counters tie; ranks shuffled"""
    rng = np.random.default_rng(seed)
    K, pk, pm, p = 14, [], [], 0
    for a in range(K):
        for group, n in (((a + 1) % K, (a + 2) % K, (a + 3) % K), 16), (((a + 4) % K, (a + 5) % K), 15), (((a + 6) % K, (a + 7) % K), 7):
            for _ in range(n):
                pk.extend((a,) + group); pm.extend([p] * (len(group) + 1)); p += 1
    return synth.covis_pack(K, pk, pm, p, rng, null_frac=0.1, dup_frac=0.02)


def cases():
    return dict(edges=hand_edges(), storm=storm(),
                random=synth.make_covisibility(seed=33, K=50, P=2500, max_deg=8, window=12, same_id_frac=0.1),
                maps=synth.make_covisibility(seed=34, K=60, P=3000, max_deg=10, window=16, n_maps=3, same_id_frac=0.05, batch_frac=0.7))


def load(z, name):
    sc = {k: z[name + "/" + k] for k in IN_KEYS}
    return sc, {k: z[name + "/out/" + k] for k in OUT_KEYS}


def main():
    from oracle import pycv
    arrays = {}
    for name, sc in cases().items():
        want = witness(sc)
        got = pycv.oracle(sc)
        for k in OUT_KEYS:
            if not np.array_equal(want[k], got[k]):
                raise SystemExit("%s: the witness and the oracle differ in %s; not written" % (name, k))
        for k in IN_KEYS:
            arrays[name + "/" + k] = sc[k]
        for k in OUT_KEYS:
            arrays[name + "/out/" + k] = want[k]
    np.savez_compressed(OUT, **arrays)
    print("wrote", OUT)


if __name__ == "__main__":
    main()

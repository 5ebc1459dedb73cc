"""Generates tests/golden/distinctive_descriptors.npz: MapPoint::ComputeDistinctiveDescriptors (cslam/src/MapPoint.cpp:929-994) on
hand-made edge cases and random scenes.  The fixture stores each case's inputs (the keys of synth.make_distinctive) and the answer:
    best         position of the chosen observer in the point's list, bad observers counted; -1 untouched
    best_median  its median distance; desc its 32 bytes (0 when untouched)
The answer is the numpy witness below: survivors, a popcount matrix from np.unpackbits, np.sort of every row, element (N-1)//2,
np.argmin (the first minimum).  Before it writes, every point is recomputed by a second, pure-Python restatement (int.bit_count,
sorted(), the reference's strict < loop); the generator refuses to write on any difference.  Run from the repo root:
    python tests/golden/make_distinctive_golden.py
"""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", ".."))
from ccm_slam_b200 import synth  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(HERE, "distinctive_descriptors.npz")
KEYS = ("kf_bad", "kf_uid", "kf_desc_ptr", "kf_desc", "mp_bad", "obs_ptr", "obs_kf", "obs_feat")   # obs_desc: see load()


def hand_scene(points):
    """points: a list of observer lists [(bad, 32 bytes), ...]; every observer gets a keyframe row of its own with one feature, rows in
    observer order (so a std::map<kfptr> over stand-in keyframes keeps the list order)"""
    bad, desc, ptr = [], [], [0]
    for obs in points:
        for b, d in obs:
            bad.append(b); desc.append(np.asarray(d, np.uint8))
        ptr.append(len(bad))
    E = len(bad)
    desc = np.array(desc, np.uint8).reshape(E, 32)
    return dict(kf_bad=np.array(bad, np.uint8), kf_uid=np.arange(E, dtype=np.uint64) + np.uint64(1000), kf_desc_ptr=np.arange(E + 1, dtype=np.int64),
                kf_desc=desc, mp_bad=np.zeros(len(points), bool), obs_ptr=np.array(ptr, np.int64), obs_kf=np.arange(E, dtype=np.int32),
                obs_feat=np.zeros(E, np.int32), obs_desc=desc)


def hand_cases():
    rng = np.random.default_rng(71)
    rnd = lambda: rng.integers(0, 256, 32, dtype=np.uint8)               # noqa: E731
    near = lambda t, m: t ^ np.bitwise_and.reduce(rng.integers(0, 256, (m, 32), dtype=np.uint8), axis=0) if m else t.copy()  # noqa: E731
    pts = []
    for n in (1, 2, 3, 4, 5, 6, 7, 8):                                  # small N, even and odd, noisy copies of one descriptor
        t = rnd(); pts.append([(0, near(t, 3)) for _ in range(n)])
    for n in (2, 4, 6):                                                 # independent random rows: medians differ little
        pts.append([(0, rnd()) for _ in range(n)])
    x = rnd(); pts.append([(0, x)] * 5)                                 # all equal: every median 0, the first wins
    x = rnd(); pts.append([(0, rnd()), (0, x), (0, x), (0, x)])         # the smallest median tied at positions 1..3: 1 wins
    x = rnd(); pts.append([(0, rnd()), (0, rnd()), (0, x), (0, x), (0, x), (0, rnd())])
    t = rnd(); pts.append([(0, near(t, 2)), (0, t), (0, near(t, 2)), (0, t)])   # even N: lower middle
    t = rnd()
    pts.append([(1, t), (1, rnd()), (0, near(t, 4)), (0, near(t, 4)), (0, near(t, 4))])     # bad at the front
    pts.append([(0, near(t, 4)), (1, t), (1, t), (0, near(t, 4)), (0, near(t, 4))])          # bad in the middle
    pts.append([(0, near(t, 4)), (0, near(t, 4)), (0, rnd()), (1, t), (1, t)])              # bad at the end
    pts.append([(1, near(t, 3)), (0, rnd()), (1, t), (0, near(t, 3)), (1, t), (0, near(t, 3))])  # bad interleaved
    pts.append([(1, rnd()) for _ in range(4)])                          # every observer bad
    pts.append([])                                                      # no observers
    pts.append([(1, rnd())])
    for n in (31, 32, 33, 64, 65, 256, 257, 1024, 1025, 3000):           # N survivors around each kernel path's edge, one in the thousands,
        t = rnd(); m = np.array([0, 3, 4, 5])                          # with 3 bad observers among them
        obs = [(0, near(t, int(rng.choice(m)))) for _ in range(n)]
        for q in sorted(rng.choice(n, 3, replace=False))[::-1]:
            obs.insert(int(q), (1, rnd()))
        pts.append(obs)
    t = rnd(); pts.append([(int(q < 40), near(t, 4)) for q in range(73)])   # 40 bad, then 33 survivors: N crosses 32 only after the skip
    return hand_scene(pts)


def cases():
    """name -> scene"""
    return {"hand": hand_cases(),
            "random": synth.make_distinctive(seed=72, K=40, P=600, max_deg=12, bad_kf_frac=0.15, all_bad_frac=0.03, empty_frac=0.03,
                                             bad_mp_frac=0.03, extra_feat=0, map_order=True),
            "small": synth.make_distinctive(synth.make_config("small"), seed=73, bad_kf_frac=0.05, extra_feat=0, map_order=True)}


def load(z, name):
    """one case of the fixture: (scene, answer); obs_desc is gathered from the keyframes' rows"""
    sc = {k: z["%s_%s" % (name, k)] for k in KEYS}
    sc["obs_desc"] = sc["kf_desc"][sc["kf_desc_ptr"][sc["obs_kf"]] + sc["obs_feat"]]
    return sc, {k: z["%s_%s" % (name, k)] for k in ("best", "best_median", "desc")}


NAMES = ("hand", "random", "small")


def witness(sc):
    """the numpy statement of the rule"""
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
        m = np.sort(dist, axis=1)[:, (len(pos) - 1) // 2]
        a = int(np.argmin(m))
        best[i] = pos[a]; med[i] = m[a]; desc[i] = D[ptr[i] + pos[a]]
    return dict(best=best, best_median=med, desc=desc)


def pure_python(sc):
    """the second statement: Python integers, the reference's loop"""
    ptr, okf, bad = sc["obs_ptr"].tolist(), sc["obs_kf"].tolist(), sc["kf_bad"].tolist()
    rows = [int.from_bytes(bytes(r), "little") for r in sc["obs_desc"]]
    best, med = [], []
    for i in range(len(ptr) - 1):
        pos = [j - ptr[i] for j in range(ptr[i], ptr[i + 1]) if not bad[okf[j]]]
        if not pos:
            best.append(-1); med.append(0); continue
        v = [rows[ptr[i] + p] for p in pos]
        N = len(v)
        bm, bi = 2 ** 31 - 1, 0
        for a in range(N):
            m = sorted((v[a] ^ v[c]).bit_count() for c in range(N))[int(0.5 * (N - 1))]
            if m < bm:
                bm, bi = m, a
        best.append(pos[bi]); med.append(bm)
    return np.array(best, np.int32), np.array(med, np.int32)


def main():
    out = {}
    for name, sc in cases().items():
        w = witness(sc)
        b, m = pure_python(sc)
        if not (np.array_equal(b, w["best"]) and np.array_equal(m, w["best_median"])):
            bad = np.flatnonzero((b != w["best"]) | (m != w["best_median"]))
            raise SystemExit("%s: the two statements disagree at points %s; nothing written" % (name, bad[:10]))
        for k in KEYS:
            out["%s_%s" % (name, k)] = sc[k]
        for k, v in w.items():
            out["%s_%s" % (name, k)] = v
    np.savez_compressed(OUT, **out)
    print("wrote", OUT)


if __name__ == "__main__":
    main()

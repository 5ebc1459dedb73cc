"""Cost of the searches of LocalMapping::SearchInNeighbors per keyframe on one GPU, and what they replace.

  (a) ccm_fuse_neighbours: every (target, slot) and (current keyframe, candidate) pair in one call
  (b) the path it replaces: one ccm_fuse_search per target entry (a target listed twice is searched twice, as the member does), then
      the backward one.  The host prelude that builds each entry's queries (gate_into_kf in shim/ORBmatcher_proj_shim.cpp) is NOT
      timed: it is computed once here in numpy, so (b) is a lower bound of the old path.
  Bytes moved each way are estimates from the array sizes (the 64 x 48 grid of the generated scene for (b)), not measurements.
  (c) the flat oracle (oracle/pyfn.py) on one CPU thread: a proxy for the CPU cost of the searches; the reference's own
      SearchInNeighbors was not measured.
C calls on prebuilt structs; medians of alternating repetitions filling about a second each.  Prints the card and its power limit
from the same process.  python tools/fuse_probe.py [--out DIR]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from ccm_slam_b200 import api  # noqa: E402
from ccm_slam_b200 import synth_match as sm  # noqa: E402
from oracle import pyfn  # noqa: E402


def queries(k, pts, rows):
    """Fuse's prelude into keyframe k for point rows (numpy f32 arithmetic, logf via numpy): the queries ccm_fuse_search takes"""
    f = np.float32
    m = len(rows)
    q = dict(valid=np.zeros(m, np.uint8), uv=np.zeros((m, 2), f), radius=np.zeros(m, f), level=np.zeros(m, np.int32),
             desc=np.zeros((m, 32), np.uint8))
    ok = rows >= 0
    r = np.where(ok, rows, 0)
    ok &= pts["skip"][r] == 0
    P = pts["pos"][r].astype(f)
    T = np.asarray(k["Tcw"], f)
    pc = [((T[i, 0] * P[:, 0] + T[i, 1] * P[:, 1]) + T[i, 2] * P[:, 2]) + T[i, 3] for i in range(3)]
    with np.errstate(all="ignore"):
        ok &= ~(pc[2] < f(0))
        invz = f(1) / pc[2]
        fx, fy, cx, cy = (f(x) for x in k["intr"])
        u = fx * (pc[0] * invz) + cx
        v = fy * (pc[1] * invz) + cy
        x0, y0, x1, y1 = (f(b) for b in k["bounds"])
        ok &= (u >= x0) & (u < x1) & (v >= y0) & (v < y1)
        d = sm.fuse_dist3d(P, k["Ow"])
        ok &= ~((d < f(0.8) * pts["min_d"][r]) | (d > f(1.2) * pts["max_d"][r]))
        PO = (P - np.asarray(k["Ow"], f)).astype(np.float64)
        ok &= ~((PO * pts["normal"][r].astype(np.float64)).sum(1) < 0.5 * d.astype(np.float64))
        lv = np.ceil(np.log(pts["max_d"][r] / d) / f(k["log_scale_factor"]))
        lv = np.clip(np.nan_to_num(lv, nan=0, posinf=0, neginf=0), 0, len(k["scale_factors"]) - 1).astype(np.int32)
    q["valid"][:] = ok; q["uv"][:, 0] = u; q["uv"][:, 1] = v; q["level"][:] = lv
    q["radius"][:] = f(3.0) * np.asarray(k["scale_factors"], f)[lv]
    q["desc"][:] = pts["desc"][r]
    return q


def timed(fn, budget=1.0):
    fn()
    t0 = time.perf_counter(); k = 0
    while True:
        fn(); k += 1
        if time.perf_counter() - t0 > budget / 4:
            break
    return (time.perf_counter() - t0) / k


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--reps", type=int, default=4)
    a = ap.parse_args()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip()
    api.init(0)
    from ccm_slam_b200.frontend import grid_struct, queries_struct
    L = api.lib()
    sc = sm.make_fuse_scene(n_first=20, n_second=5, n=1000, seed=0)
    keep = []
    cur, tg, T, pts, cp, cand = api.fuse_structs(sc, keep)
    n, nc = len(cp), len(cand)
    fwd = np.zeros((T, n), np.int32); bwd = np.zeros(nc, np.int32); settled = C.c_int32()

    def call_a():
        api._chk(L.ccm_fuse_neighbours(C.byref(cur), tg, T, C.byref(pts), api._p(cp), api._p(cand), nc, api._p(fwd), api._p(bwd), C.byref(settled)))
    # (b): structs per entry, built once
    p = sc["points"]
    G = [grid_struct(k, keep) for k in sc["targets"]]
    Gc = grid_struct(sc["cur"], keep)
    il = [np.ascontiguousarray(k["inv_level_sigma2"], np.float32) for k in sc["targets"] + [sc["cur"]]]
    Qe = [queries_struct(queries(sc["targets"][e], p, cp), keep) for e in sc["entries"]]
    Qb = queries_struct(queries(sc["cur"], p, cand), keep)
    best_e = [np.zeros(n, np.int32) for _ in sc["entries"]]
    best_b = np.zeros(nc, np.int32); nf = C.c_int32()

    def call_b():
        for i, e in enumerate(sc["entries"]):
            api._chk(L.ccm_fuse_search(C.byref(G[e]), C.byref(Qe[i]), api._p(il[e]), len(il[e]), api._p(best_e[i]), C.byref(nf)))
        api._chk(L.ccm_fuse_search(C.byref(Gc), C.byref(Qb), api._p(il[-1]), len(il[-1]), api._p(best_b), C.byref(nf)))
    olib = pyfn.lib()
    of = np.zeros((T, n), np.int32); ob = np.zeros(nc, np.int32)

    def call_c():
        olib.orc_fuse_neighbours(C.byref(cur), tg, T, C.byref(pts), api._p(cp), api._p(cand), nc, api._p(of), api._p(ob))
    ta, tb, tc = [], [], []
    for _ in range(a.reps):
        ta.append(timed(call_a)); tb.append(timed(call_b)); tc.append(timed(call_c))
    call_a(); call_b(); call_c()
    agree_b = int(sum((best_e[i] == fwd[e]).sum() for i, e in enumerate(sc["entries"])) + (best_b == bwd).sum())
    total_b = len(sc["entries"]) * n + nc
    # bytes: ESTIMATES from the array sizes, not measured.  (a) the arrays of the one pinned block (the Kf table and the 16-byte padding
    # left out) and one i32 per pair down
    up_a = sum(k["desc"].nbytes + k["kp_xy"].nbytes + k["octave"].nbytes + 4 * (k["cols"] * k["rows"] + 1) + 4 * len(k["octave"])
               for k in sc["targets"] + [sc["cur"]]) + sum(np.asarray(v).nbytes for k, v in p.items() if k != "bad") + cp.nbytes + cand.nbytes
    down_a = 4 * (T * n + nc)
    # (b) per call: the grid's descriptors, keypoints, octaves and cell index, the queries and their descriptors; one (index, distance) pair back per query
    up_b = sum(sc["targets"][e]["desc"].nbytes + 12 * n + 4 * (64 * 48 + 1 + n) + 64 * n for e in sc["entries"]) + \
        sc["cur"]["desc"].nbytes + 12 * n + 4 * (64 * 48 + 1 + n) + 64 * nc
    down_b = 8 * (len(sc["entries"]) * n + nc)
    res = dict(card=card, targets_distinct=T, entries=len(sc["entries"]), features=n, candidates=nc,
               a_ms=1e3 * float(np.median(ta)), b_ms=1e3 * float(np.median(tb)), c_ms=1e3 * float(np.median(tc)),
               a_all=[1e3 * x for x in ta], b_all=[1e3 * x for x in tb], c_all=[1e3 * x for x in tc],
               settled=settled.value, fuse_matches=int((fwd >= 0).sum() + (bwd >= 0).sum()), b_agrees=agree_b, b_pairs=total_b,
               a_bytes_up_est=int(up_a), a_bytes_down_est=int(down_a), b_bytes_up_est=int(up_b), b_bytes_down_est=int(down_b),
               oracle_equal=bool(np.array_equal(of, fwd) and np.array_equal(ob, bwd)))
    print(json.dumps(res))
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "fuse_probe.json"), "w") as fh:
            json.dump(res, fh)


if __name__ == "__main__":
    main()

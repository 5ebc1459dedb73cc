"""Cost of the searches of LoopFinder / MapMerger::SearchAndFuse on one GPU, and what they replace.

Shapes: loop (31 corrected keyframes of 1000 features against about 8000 loop points) and stress (100 x 30000).
  (a) ccm_search_and_fuse: every (keyframe, loop point) pair in one call, host buffers in and out
  (k) k_sf_pairs alone: its device time from torch.profiler's CUDA activity records, in a run of its own after the timed runs
  (h) ccm_search_and_fuse_host: the same contract on one CPU thread
  (b) the path it replaces: one ccm_fuse_search per keyframe on queries built once here in numpy (Fuse(Scw)'s host prelude in
      shim/ORBmatcher_proj_shim.cpp is NOT timed), so (b) is a lower bound of the old path
  (c) the flat oracle (oracle/pysf.py) on one CPU thread
  (s) the whole member on stand-in objects (oracle/pysf.StandIn, the loop shape with held slots and duplicates): the literal restatement
      of LoopFinder::SearchAndFuse against shim/SearchAndFuse_shim.cpp over the real library, one run each on fresh scenes, with the
      number of points the shim searched again because an earlier replacement changed their descriptor
(a), (h) and (c) must give the same pairs, or the probe fails; (b) builds its queries with numpy's log, not logf, so it may differ at
PredictScale boundaries and its agreement is only reported.
Medians of --reps alternating repetitions (default 3), each call synchronised (every entry point returns after its download).  Prints the card, its
power limit and its top SM clock from the same process.  python tools/search_and_fuse_probe.py [--out DIR] [--shapes loop,stress]
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
from oracle import pyoracle, pysf  # noqa: E402
from tools.fuse_probe import queries, timed  # noqa: E402

SHAPES = {"loop": dict(n_kf=31, n=1000, n_loop=8000), "stress": dict(n_kf=100, n=1000, n_loop=30000)}


def kernel_ms(call, reps=20):
    """median device time of k_sf_pairs over `reps` calls, from torch.profiler's CUDA activity records; None when none were recorded"""
    try:
        import torch
        from torch.profiler import ProfilerActivity, profile
    except Exception:
        return None
    call()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            call()
        torch.cuda.synchronize()
    d = [e.device_time_total for e in prof.events() if "k_sf_pairs" in e.name]
    return 1e-3 * float(np.median(d)) if d else None


def run(shape, reps):
    L = api.lib()
    sc = sm.make_search_and_fuse_scene("loop", seed=0, **SHAPES[shape])
    keep = []
    kfs, K, pts = api.search_and_fuse_structs(sc, keep)
    P = pts.n
    best = np.zeros((K, P), np.int32); hbest = np.zeros((K, P), np.int32); obest = np.zeros((K, P), np.int32)
    settled = C.c_int32()

    def call_a():
        api._chk(L.ccm_search_and_fuse(kfs, K, C.byref(pts), api._p(best), C.byref(settled)))

    def call_h():
        api._chk(L.ccm_search_and_fuse_host(kfs, K, C.byref(pts), api._p(hbest), None))
    olib = pyoracle.lib()

    def call_c():
        olib.orc_search_and_fuse(kfs, K, C.byref(pts), C.c_float(4.0), 0, api._p(obest))
    # (b): one grid and one query set per keyframe, built once
    from ccm_slam_b200.frontend import grid_struct, queries_struct
    p = sc["points"]
    rows = np.arange(P)
    G, Q = [], []
    for k in sc["kfs"]:
        q = queries(k, p, rows)
        q["radius"][:] = np.float32(4.0) * np.asarray(k["scale_factors"], np.float32)[q["level"]]
        G.append(grid_struct(k, keep)); Q.append(queries_struct(q, keep))
    bb = [np.zeros(P, np.int32) for _ in range(K)]
    nf = C.c_int32()

    def call_b():
        for k in range(K):
            api._chk(L.ccm_fuse_search(C.byref(G[k]), C.byref(Q[k]), None, 0, api._p(bb[k]), C.byref(nf)))
    ta, th, tb, tc = [], [], [], []
    for _ in range(reps):
        ta.append(timed(call_a)); tb.append(timed(call_b))
        th.append(timed(call_h, budget=0.5)); tc.append(timed(call_c, budget=0.5))
    call_a(); call_h(); call_b(); call_c()
    agree_b = int(sum((bb[k] == best[k]).sum() for k in range(K)))
    assert np.array_equal(best, hbest) and np.array_equal(best, obest), "device, host entry point and oracle disagree"
    return dict(shape=shape, keyframes=K, features=int(sc["kfs"][0]["desc"].shape[0]), loop_points=P, pairs=K * P,
                a_ms=1e3 * float(np.median(ta)), h_ms=1e3 * float(np.median(th)), b_ms=1e3 * float(np.median(tb)),
                c_ms=1e3 * float(np.median(tc)), a_all=[1e3 * x for x in ta], b_all=[1e3 * x for x in tb],
                k_sf_pairs_ms=kernel_ms(call_a), settled=settled.value, found=int((best >= 0).sum()),
                b_agrees=agree_b)


def shim_vs_restatement():
    """(restatement ms, shim ms, repairs) for one LoopFinder::SearchAndFuse member on stand-ins of the loop shape"""
    sc = sm.make_search_and_fuse_scene("loop", seed=1, held_frac=0.3, occupied_frac=0.3, dup=400, **SHAPES["loop"])
    w = pysf.StandIn(sm.make_search_and_fuse_scene("loop", n_kf=2, n=200, seed=2), gpu=True)   # first call: stream and blocks
    w.run(1, False)
    w.close()
    out = []
    for mode in (0, 1):
        s = pysf.StandIn(sc, gpu=True)
        s0 = s.stats()
        t0 = time.perf_counter()
        s.run(mode, False)
        out.append(1e3 * (time.perf_counter() - t0))
        rep = int((s.stats() - s0)[1])
        s.close()
    return dict(restatement_ms=out[0], shim_ms=out[1], repairs=rep)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--shapes", default="loop,stress")
    a = ap.parse_args()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip()
    api.init(0)
    res = dict(card=card, reps=a.reps, shapes=[run(s, a.reps) for s in a.shapes.split(",")], shim=shim_vs_restatement())
    print(json.dumps(res))
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "search_and_fuse_probe.json"), "w") as fh:
            json.dump(res, fh)


if __name__ == "__main__":
    main()

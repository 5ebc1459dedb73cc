"""Measures ccm_covisibility (KeyFrame::UpdateConnections' counting for a whole-map batch) at the cfg4 and full cfg5 observation
structure and prints one JSON line: the kernel time (the k_cv_* kernels' durations in torch.profiler's CUPTI device trace, summed per
call, recorded in the same process as the wall-clock timings that follow), the call wall time with host buffers, ccm_covisibility_host
over the same arrays on one thread, and, as a single-thread proxy for the reference, the literal restatement of UpdateConnections
(std::map counter, AddConnection, UpdateBestCovisibles, parent) over stand-in objects.  On cfg5 the literal runs over a random sample
of keyframes (a scene holding only their points and those points' observers); literal_ms_per_kf is measured on that sample and
literal_ms_whole_map_extrapolated scales it to the batch.  GPU name and power limit are read in the same run.
    python tools/covis_probe.py [--reps 5] [--literal-sample 500]
"""
import argparse
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
import numpy as np  # noqa: E402

from ccm_slam_b200 import api, synth  # noqa: E402


def gpu_info():
    try:
        out = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], text=True).strip().splitlines()[0]
        name, pl = [x.strip() for x in out.split(",")]
        return name, pl
    except Exception as e:  # noqa: BLE001
        return "unknown (%s)" % e, "unknown"


def kernel_ms(sc, cap, reps):
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            api.covisibility(sc, capacity=cap)
        torch.cuda.synchronize()
    per = {}
    for e in prof.events():
        for k in ("k_cv_shared<false>", "k_cv_shared<true>", "k_cv_dense<false>", "k_cv_dense<true>"):
            if k in e.name:
                per.setdefault(k, []).append(e.device_time / 1000.0)
    med = {k: float(np.median(v)) for k, v in per.items()}
    return med, float(sum(med.values())) if med else None


def wall_ms(fn, reps):
    t = []
    for _ in range(reps):
        t0 = time.perf_counter(); fn(); t.append((time.perf_counter() - t0) * 1e3)
    return float(np.median(t))


def literal_sample(sc, rows):
    """the sub-scene of the keyframes `rows`: their points and those points' observers; every keyframe row kept (ranks unchanged)"""
    from oracle import pycv
    pts = np.unique(np.concatenate([sc["mvp"][sc["mvp_ptr"][r]:sc["mvp_ptr"][r + 1]] for r in rows]))
    pts = pts[pts >= 0]
    remap = np.full(len(sc["mp_bad"]), -1, np.int64); remap[pts] = np.arange(len(pts))
    n = np.diff(sc["mvp_ptr"]); keep = np.zeros(len(n), bool); keep[rows] = True
    lens = np.where(keep, n, 0)
    mptr = np.zeros(len(n) + 1, np.int64); mptr[1:] = np.cumsum(lens)
    sel = np.repeat(keep, n)
    mvp = sc["mvp"][sel]; mvp = np.where(mvp >= 0, remap[np.maximum(mvp, 0)], -1).astype(np.int32)
    deg = np.diff(sc["obs_ptr"])[pts]
    optr = np.zeros(len(pts) + 1, np.int64); optr[1:] = np.cumsum(deg)
    idx = np.repeat(sc["obs_ptr"][pts] - optr[:-1], deg) + np.arange(optr[-1])
    sub = dict(sc, mvp_ptr=mptr, mvp=mvp, mp_bad=sc["mp_bad"][pts], obs_ptr=optr, obs_kf=sc["obs_kf"][idx], obs_idx=sc["obs_idx"][idx],
               batch=np.asarray(rows, np.int32))
    s = pycv.StandIn(sub)
    t0 = time.perf_counter(); s.merge(0); t = (time.perf_counter() - t0) * 1e3
    s.close()
    return t


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--literal-sample", type=int, default=500)
    a = ap.parse_args()
    api.init(0)
    name, pl = gpu_info()
    res = dict(gpu=name, power_limit=pl, reps=a.reps, stat="median")
    for cfg in ("cfg4", "cfg5"):
        sc = synth.make_covisibility(synth.make_config(cfg), seed=1)
        h = api.covisibility(sc, host=True)
        cap = int(h["conn_ptr"][-1])
        r = api.covisibility(sc, capacity=cap)                             # warm-up, and the result must be the host's
        assert all(np.array_equal(r[k], h[k]) for k in h), cfg
        n = np.diff(h["conn_ptr"])
        row = dict(keyframes=len(sc["batch"]), points=len(sc["mp_bad"]), map_point_entries=int(len(sc["mvp"])),
                   observations=int(len(sc["obs_kf"])), counter_entries=cap, max_counter=int(n.max()), mean_counter=float(n.mean()))
        row["kernel_ms_each"], row["kernel_ms"] = kernel_ms(sc, cap, a.reps)
        row["call_wall_ms"] = wall_ms(lambda: api.covisibility(sc, capacity=cap), a.reps)
        row["host_entry_ms"] = wall_ms(lambda: api.covisibility(sc, host=True, capacity=cap), max(1, a.reps // 2))
        K = len(sc["batch"])
        rows = np.arange(K) if K <= a.literal_sample else np.sort(np.random.default_rng(2).choice(K, a.literal_sample, replace=False))
        t = literal_sample(sc, rows)
        row["literal_keyframes"] = int(len(rows))
        row["literal_ms_per_kf"] = t / len(rows)
        if len(rows) == K:
            row["literal_ms_whole_map"] = t
        else:
            row["literal_ms_whole_map_extrapolated"] = t / len(rows) * K
        res[cfg] = row
    print(json.dumps(res))


if __name__ == "__main__":
    main()

"""Measures ccm_normal_depth (MapPoint::UpdateNormalAndDepth for a batch) at the cfg4 and full cfg5 observer structure and prints one
JSON line: the kernel time (k_normal_depth's duration in torch.profiler's CUPTI device trace, recorded in the same process as the
wall-clock timings that follow), the call wall time with host buffers, ccm_normal_depth_host over the same arrays on one thread, and
the MapPoint shim's write-back over stand-in objects with and without the batched preparation (a proxy: the reference's own per-point cost is not measured).  GPU name and power limit are read in the same run.
    python tools/normal_depth_probe.py [--reps 5]
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


def kernel_ms(sc, reps):
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            api.normal_depth(sc)
        torch.cuda.synchronize()
    ts = [e.device_time for e in prof.events() if "k_normal_depth" in e.name]
    return float(np.median(ts)) / 1000.0 if ts else None


def wall_ms(fn, reps):
    t = []
    for _ in range(reps):
        t0 = time.perf_counter(); fn(); t.append((time.perf_counter() - t0) * 1e3)
    return float(np.median(t))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    api.init(0)
    name, pl = gpu_info()
    res = dict(gpu=name, power_limit=pl, reps=a.reps, stat="median")
    for cfg in ("cfg4", "cfg5"):
        sc = synth.make_normal_depth(synth.make_config(cfg), seed=1)
        api.normal_depth(sc)                                            # warm-up
        row = dict(points=len(sc["mp_ref"]), observers=int(len(sc["obs_kf"])))
        row["kernel_ms"] = kernel_ms(sc, a.reps)
        row["call_wall_ms"] = wall_ms(lambda: api.normal_depth(sc), a.reps)
        row["host_entry_ms"] = wall_ms(lambda: api.normal_depth(sc, host=True), a.reps)
        if cfg == "cfg4":                                               # stand-in objects: the shim's own loop, with and without batching
            from oracle import pynd
            s = pynd.StandIn(synth.make_normal_depth(synth.make_config(cfg), seed=1, map_order=True), gpu=True)
            row["shim_loop_host_ms"] = wall_ms(lambda: s.shim(prepare=False), a.reps)
            row["shim_loop_batched_ms"] = wall_ms(lambda: s.shim(prepare=True), a.reps)
            s.close()
        res[cfg] = row
    print(json.dumps(res))


if __name__ == "__main__":
    main()

"""Measures ccm_distinctive_descriptors (MapPoint::ComputeDistinctiveDescriptors for a batch) at the cfg4 and full cfg5 observer
structure and prints one JSON line: the kernel time (the k_dd_* kernels' durations in torch.profiler's CUPTI device trace, summed per
call, recorded in the same process as the wall-clock timings that follow), the call wall time with host buffers, the wall time of
ccm_kfstore_distinctive_descriptors over a store holding every keyframe, and ccm_distinctive_descriptors_host over the same arrays on
one thread.  GPU name and power limit are read in the same run.
    python tools/distinctive_probe.py [--reps 5]
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
from ccm_slam_b200.frontend import KP_DTYPE, KeyFrameStore  # noqa: E402


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
            api.distinctive_descriptors(sc)
        torch.cuda.synchronize()
    per = {}
    for e in prof.events():
        for k in ("k_dd_classify", "k_dd_warp", "k_dd_cta"):
            if k in e.name:
                per.setdefault(k, []).append(e.device_time / 1000.0)
    med = {k: float(np.median(v)) for k, v in per.items()}
    return med, float(sum(med.values())) if med else None


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
        sc = synth.make_distinctive(synth.make_config(cfg), seed=1)
        api.distinctive_descriptors(sc)                                 # warm-up
        n = np.diff(sc["obs_ptr"])
        row = dict(points=len(n), observers=int(len(sc["obs_kf"])), max_observers=int(n.max()))
        row["kernel_ms_each"], row["kernel_ms"] = kernel_ms(sc, a.reps)
        row["call_wall_ms"] = wall_ms(lambda: api.distinctive_descriptors(sc), a.reps)
        st = KeyFrameStore()
        for k in range(len(sc["kf_bad"])):
            d = sc["kf_desc"][sc["kf_desc_ptr"][k]:sc["kf_desc_ptr"][k + 1]]
            st.put(int(sc["kf_uid"][k]), np.zeros(len(d), KP_DTYPE), d)
        args = (sc["kf_uid"], sc["kf_bad"], sc["obs_ptr"], sc["obs_kf"], sc["obs_feat"])
        st.distinctive_descriptors(*args)
        row["store_wall_ms"] = wall_ms(lambda: st.distinctive_descriptors(*args), a.reps)
        st.close()
        row["host_entry_ms"] = wall_ms(lambda: api.distinctive_descriptors(sc, host=True), a.reps)
        res[cfg] = row
    print(json.dumps(res))


if __name__ == "__main__":
    main()

"""Measures ccm_sim3_correction (the Sim3 pass of LoopFinder::CorrectLoop / MapMerger::MergeMaps) and prints one JSON line.  Three
shapes: a merge of the whole cfg4 map, a merge of the whole cfg5 map (K = 10^4, P = 10^6) and a loop closure on the cfg4 map (the
current keyframe and its 30 most covisible keyframes), the last with every point of the map and with only the points the entries list
(what shim/Sim3Correction_shim.cpp passes).  For each:
  device_call_ms   ccm_sim3_correction with host buffers in and out (validation, packing, one upload, three launches, one download,
                   synchronised), warmed, median of repetitions
  kernels_ms       the three kernels' device time from torch.profiler's CUDA trace, recorded before the wall-clock timings
  host_entry_ms    ccm_sim3_correction_host over the same arrays, one thread
  oracle_walk_ms   the flat oracle: the reference's sequential walk over the same arrays, one thread.  A proxy for the reference loop
                   itself, which also chases pointers, takes locks and allocates cv::Mat per point; that loop is not measured here.
GPU name and power limit are read in the same run.
    python tools/sim3_correction_probe.py [--reps 7]
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
from oracle import pysc  # noqa: E402

KERNELS = ("k_sc_entries", "k_sc_claim", "k_sc_points")


def gpu_info():
    try:
        out = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                                      text=True).strip().splitlines()[0]
        return [x.strip() for x in out.split(",")]
    except Exception as e:  # noqa: BLE001
        return ["unknown (%s)" % e, "unknown", "unknown"]


def kernels_ms(sc, out, reps):
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            api.sim3_correction(sc, out=out)
        torch.cuda.synchronize()
    per = {}
    for e in prof.events():
        for k in KERNELS:
            if k in e.name:
                per.setdefault(k, []).append(e.device_time / 1000.0)
    return {k: float(np.median(v)) for k, v in per.items()}


def wall_ms(fn, reps):
    fn()
    t = []
    for _ in range(reps):
        t0 = time.perf_counter(); fn(); t.append((time.perf_counter() - t0) * 1e3)
    return float(np.median(t)), float(min(t)), float(max(t))


def listed_only(sc):
    """the scene with only the points some entry lists, renumbered: what shim/Sim3Correction_shim.cpp flattens"""
    keep = np.zeros(len(sc["mp_skip"]), bool)
    keep[sc["slot_mp"][sc["slot_mp"] >= 0]] = True
    new = np.full(len(keep), -1, np.int32); new[keep] = np.arange(int(keep.sum()), dtype=np.int32)
    out = dict(sc)
    out["slot_mp"] = np.where(sc["slot_mp"] >= 0, new[np.maximum(sc["slot_mp"], 0)], -1).astype(np.int32)
    deg = np.diff(sc["obs_ptr"])[keep]
    idx = np.repeat(sc["obs_ptr"][:-1][keep], deg) + (np.arange(int(deg.sum())) - np.repeat(np.cumsum(deg) - deg, deg))
    out["obs_kf"] = sc["obs_kf"][idx]; out["obs_ptr"] = np.concatenate([[0], np.cumsum(deg)]).astype(np.int64)
    for k in ("mp_pos", "mp_skip", "mp_ref", "mp_scale_ref", "mp_scale_last"):
        out[k] = sc[k][keep]
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
    a = ap.parse_args()
    api.init(0)
    name, pl, clk = gpu_info()
    res = dict(gpu=name, power_limit=pl, max_sm_clock=clk, reps=a.reps, stat="median [min, max] ms")
    cfg4 = synth.make_config("cfg4")
    shapes = [("cfg4_merge", lambda: synth.make_sim3_correction(cfg4, kind="merge", seed=1)),
              ("cfg4_loop30", lambda: synth.make_sim3_correction(cfg4, kind="loop", seed=1, n_loop=30)),
              ("cfg4_loop30_listed", lambda: listed_only(synth.make_sim3_correction(cfg4, kind="loop", seed=1, n_loop=30))),
              ("cfg5_merge", lambda: synth.make_sim3_correction(synth.make_config("cfg5"), kind="merge", seed=1))]
    for tag, make in shapes:
        sc = make()
        out = api.sim3_correction_out(len(sc["entry_kf"]), len(sc["mp_skip"]))
        ref = pysc.oracle(sc)
        api.sim3_correction(sc, out=out)                                 # warm-up, and the result checked once
        ok = all(np.array_equal(out[k], ref[k], equal_nan=True) for k in ref)
        row = dict(entries=len(sc["entry_kf"]), slots=int(sc["slot_ptr"][-1]), points=len(sc["mp_skip"]), observers=int(len(sc["obs_kf"])),
                   moved=int((ref["mp_entry"] >= 0).sum()), device_equals_oracle=bool(ok))
        row["kernels_ms"] = kernels_ms(sc, out, a.reps)
        row["device_call_ms"] = wall_ms(lambda: api.sim3_correction(sc, out=out), a.reps)
        hout = api.sim3_correction_out(len(sc["entry_kf"]), len(sc["mp_skip"]))
        row["host_entry_ms"] = wall_ms(lambda: api.sim3_correction(sc, host=True, out=hout), max(3, a.reps // 2))
        row["oracle_walk_ms"] = wall_ms(lambda: pysc.oracle(sc), max(3, a.reps // 2))
        res[tag] = row
        print(tag, json.dumps(row), file=sys.stderr, flush=True)
    print(json.dumps(res))


if __name__ == "__main__":
    main()

"""Measures LocalMapping::CreateNewMapPoints for one keyframe with 20 neighbours of 1000 features each, three ways, alternating, warm,
host clock around calls that end in a synchronise, median over enough repetitions to fill a second per path:
  (a) ccm_new_map_points: the whole member in one call;
  (b) the path it replaces: ccm_match_triangulation per neighbour (device distance matrix, host selection) followed by the oracle's host
      triangulation, with the claims folded into has_mp between neighbours;
  (c) the sequential oracle alone on one CPU thread (the reference's shape: matching and triangulation on the host).
Prints one JSON line with the three times, the bytes each device path moves (computed from the shapes), whether (a) and (b) produce
the same points, and the card's name, power limit and maximum SM clock.  Fails without a GPU.
    python tools/new_points_probe.py [--n-nb 20] [--n 1000] [--seconds 1.0]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
import numpy as np  # noqa: E402

from ccm_slam_b200 import api, synth_match as sm  # noqa: E402


def gpu_info():
    out = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], text=True)
    return [x.strip() for x in out.strip().splitlines()[0].split(",")]


class Prebuilt:
    """the C structs of one scene, built once: what is timed is the library call, not the Python binding"""

    def __init__(self, sc):
        self.keep = []
        self.n, self.B = len(sc["cur"]["octave"]), len(sc["neighbours"])
        self.has = sc["cur"]["has_mp"].copy()                        # (b) folds the claims in here between neighbours
        self.mask = np.ones(self.n, np.uint8)
        self.cur, self.nbs = api.new_points_structs(sc["cur"], sc["neighbours"], self.keep)
        self.cur_has, _ = api.new_points_structs(dict(sc["cur"], has_mp=self.has), [], self.keep)
        self.cur_mask, _ = api.new_points_structs(dict(sc["cur"], has_mp=self.mask), [], self.keep)
        self.has0 = sc["cur"]["has_mp"].copy()
        self.out = np.zeros(self.n * self.B, api.NEW_POINT_DTYPE)
        self.pairs = np.zeros((self.n + 1, 2), np.int32)
        self.n_out = C.c_int32()

    def one_call(self, fn):
        rc = fn(C.byref(self.cur), self.nbs, self.B, api._p(self.out), len(self.out), C.byref(self.n_out), None, None)
        assert rc == 0
        return self.out[:self.n_out.value].copy()

    def oracle(self):
        from oracle import pynp
        rc = pynp.lib().orc_new_map_points(C.byref(self.cur), self.nbs, self.B, api._p(self.out), len(self.out), C.byref(self.n_out), None, None, 0)
        assert rc == 0
        return self.out[:self.n_out.value].copy()

    def per_pair(self, match):
        """(b): per neighbour, `match` = ccm_match_triangulation, then the oracle's triangulation of exactly those pairs (the oracle over
        that neighbour alone with every other feature masked), the accepted features folded into has_mp for the next neighbour"""
        from oracle import pynp
        tri = pynp.lib().orc_new_map_points
        self.has[:] = self.has0
        got = []
        npairs = C.c_int32()
        for b in range(self.B):
            nb = self.nbs[b]
            rc = match(C.byref(self.cur_has.v), C.byref(nb.view.v), nb.F12, C.c_float(nb.ex), C.c_float(nb.ey), C.c_void_p(nb.view.level_sigma2),
                       C.c_void_p(nb.view.scale_factors), nb.view.nlevels, 0, api._p(self.pairs), C.byref(npairs))
            assert rc == 0
            self.mask[:] = 1
            self.mask[self.pairs[:npairs.value, 0]] = 0
            assert tri(C.byref(self.cur_mask), C.byref(nb), 1, api._p(self.out), len(self.out), C.byref(self.n_out), None, None, 0) == 0
            p = self.out[:self.n_out.value].copy()
            p["nb"] = b
            self.has[p["idx1"]] = 1
            got.append(p)
        return np.concatenate(got)


def bytes_moved(sc, n_out):
    views = [sc["cur"]] + sc["neighbours"]
    per = lambda v: len(v["octave"]) * (32 + 1 + 8 + 4) + 2 * 4 * len(v["level_sigma2"]) + 4 * (len(np.unique(v["node"])) + 1) + 4 * len(v["octave"])  # noqa: E731
    n1 = len(sc["cur"]["octave"])
    a_up = sum(per(v) for v in views) + 4 * n1 + 4 * len(np.unique(sc["cur"]["node"])) * len(sc["neighbours"])
    a_down = 4 + 24 * n_out
    b_up = sum(32 * (n1 + len(v["octave"])) for v in sc["neighbours"])
    b_down = sum(2 * n1 * len(v["octave"]) for v in sc["neighbours"])
    return dict(a_upload=a_up, a_download=a_down, b_upload=b_up, b_download=b_down)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n-nb", type=int, default=20); ap.add_argument("--n", type=int, default=1000)
    ap.add_argument("--seconds", type=float, default=1.0); ap.add_argument("--seed", type=int, default=3)
    a = ap.parse_args()
    if api.device_count() == 0:
        sys.exit("new_points_probe: no CUDA device; there is nothing to measure without one")
    api.init(0)
    name, power, clock = gpu_info()
    sc = sm.make_new_points_scene(n_nb=a.n_nb, n=a.n, seed=a.seed)
    pb = Prebuilt(sc)
    L = api.lib()
    paths = dict(a=lambda: pb.one_call(L.ccm_new_map_points), b=lambda: pb.per_pair(L.ccm_match_triangulation), c=pb.oracle)
    res = {k: f() for k, f in paths.items()}                         # warm every path once
    for f in paths.values():
        f()
    t = {k: [] for k in paths}
    spent = {k: 0.0 for k in paths}
    while min(spent.values()) < a.seconds:
        for k, f in paths.items():
            t0 = time.perf_counter(); f(); dt = time.perf_counter() - t0
            t[k].append(dt * 1e3); spent[k] += dt
    out = dict(gpu=name, power_limit=power, max_sm_clock=clock, n_nb=a.n_nb, n=a.n, points=int(len(res["a"])),
               a_one_call_ms=float(np.median(t["a"])), b_per_pair_calls_ms=float(np.median(t["b"])), c_cpu_oracle_ms=float(np.median(t["c"])),
               a_p10_p90_ms=[float(np.percentile(t["a"], q)) for q in (10, 90)], reps=len(t["a"]),
               a_equals_b=bool(res["a"].tobytes() == res["b"].tobytes()), a_equals_c=bool(res["a"].tobytes() == res["c"].tobytes()),
               note="C entry points called on structs built once; (b) and (c) triangulate on the host",
               **bytes_moved(sc, len(res["a"])))
    print(json.dumps(out))
    if not (out["a_equals_b"] and out["a_equals_c"]):
        sys.exit("new_points_probe: the paths disagree")


if __name__ == "__main__":
    main()

"""Cost of the redundancy test of LocalMapping::KeyFrameCullingV3 on one GPU, and what it replaces.

Shapes: 20, 60 and 150 candidates of about 1000 slots, points with 5-20 observers (synth.make_keyframe_culling_scene, two
redundant candidates whose culls reach later ones), and "cascades": 60 candidates with eight redundant ones plus the edge and cascade
blocks.
  (d) ccm_keyframe_culling: one upload, one launch, one download and the host settle, host buffers in and out
  (h) ccm_keyframe_culling_host: the same contract on one CPU thread
  (r) the member restated on stand-in objects (oracle/pykc.StandIn mode 0: KeyFrameCullingV3 with its SetBadFlag / EraseObservation
      paths, over std::map observations), one run on a fresh scene each repetition; scene construction is not timed
(d) and (h) must give the same bytes, or the probe fails.  Each time is a host clock around calls that end in a device synchronise
(every entry point returns after its download); medians of --reps alternating repetitions.  Prints the card, its power limit and its
top SM clock from the same process.  python tools/keyframe_culling_probe.py [--out DIR] [--reps 5]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from ccm_slam_b200 import api, synth  # noqa: E402
from oracle import pykc  # noqa: E402
from tools.fuse_probe import timed  # noqa: E402

SHAPES = {"20x1000": dict(n_c=20, slots=1000, seed=41, edges=False), "60x1000": dict(n_c=60, slots=1000, seed=42, edges=False),
          "150x1000": dict(n_c=150, slots=1000, seed=43, edges=False), "cascades": dict(n_c=60, slots=1000, seed=44, n_redundant=8)}


def run(name, reps):
    sc = synth.make_keyframe_culling_scene(**SHAPES[name])
    d, h = api.keyframe_culling(sc), api.keyframe_culling(sc, host=True)
    for k in d:
        if not np.array_equal(d[k], h[k]):
            raise SystemExit("%s: device and host differ in %s" % (name, k))
    out_d, out_h = api.keyframe_culling_out(len(sc["cand_kf"])), api.keyframe_culling_out(len(sc["cand_kf"]))
    argv_d, keep_d = api.keyframe_culling_args(sc, out_d)
    argv_h, keep_h = api.keyframe_culling_args(sc, out_h)
    L = api.lib()
    td, th, tr = [], [], []
    for _ in range(reps):
        td.append(timed(lambda: api._chk(L.ccm_keyframe_culling(*argv_d))))
        th.append(timed(lambda: api._chk(L.ccm_keyframe_culling_host(*argv_h))))
        s = pykc.StandIn(sc)
        t0 = time.perf_counter(); s.run(0); tr.append(time.perf_counter() - t0)
        s.close()
    ms = lambda v: round(1e3 * float(np.median(v)), 4)  # noqa: E731
    r = dict(shape=name, candidates=len(sc["cand_kf"]), slots=int(sc["slot_ptr"][-1]), points=len(sc["mp_bad"]),
             observations=int(sc["obs_ptr"][-1]), culls=int(d["cull"].sum()), settled=d["n_settled"], device_ms=ms(td), host_ms=ms(th),
             restatement_ms=ms(tr), device_range=[ms([min(td)]), ms([max(td)])], host_range=[ms([min(th)]), ms([max(th)])])
    print(json.dumps(r), flush=True)
    return r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--shapes", default=",".join(SHAPES))
    a = ap.parse_args()
    if api.device_count() == 0:
        raise SystemExit("keyframe_culling_probe: no CUDA device")
    api.init(0)
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip().splitlines()[0]
    print("card:", card, flush=True)
    res = dict(card=card, reps=a.reps, shapes=[run(s, a.reps) for s in a.shapes.split(",")])
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "keyframe_culling_probe.json"), "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()

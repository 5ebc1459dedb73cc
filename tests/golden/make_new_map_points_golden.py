"""Writes tests/golden/new_map_points.npz: two scenes for ccm_new_map_points with the sequential oracle's points, best2 and verdicts.
  small   4 neighbours x 60 features: inputs stored whole (hand-checkable)
  big     20 neighbours x 1000 features: stored as the generator's arguments plus a digest of every input array, so the file stays
          small and a drift of the generator is caught before the outputs are compared
Refuses to write unless the f64 witness check (tests/test_new_map_points.py: numpy.linalg.svd in f64 over the same pairs) passes on
both scenes.
    python tests/golden/make_new_map_points_golden.py
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "..", ".."))
from ccm_slam_b200 import synth_match as sm  # noqa: E402
from oracle import pynp  # noqa: E402
from tests import test_new_map_points as TN  # noqa: E402


def main():
    out = {}
    for name, kw in TN.FIXTURE_SCENES.items():
        sc = sm.make_new_points_scene(**kw)
        pts, b2, vd = pynp.oracle(sc["cur"], sc["neighbours"])
        bad, near, pairs = TN.witness_check(sc, pts, b2, vd)
        if bad or near > TN.NEAR_FRACTION * pairs:
            sys.exit("scene %s fails the f64 witness check (%d wrong, %d of %d near a threshold): nothing written" % (name, bad, near, pairs))
        out[name + "_points"] = pts; out[name + "_best2"] = b2; out[name + "_verdict"] = vd
        out[name + "_digest"] = np.frombuffer(TN.scene_digest(sc), np.uint8)
        if name == "small":
            for i, v in enumerate([sc["cur"]] + sc["neighbours"]):
                for k in TN.VIEW_KEYS + (("F12", "ex", "ey") if i else ()):
                    out["small_v%d_%s" % (i, k)] = np.asarray(v[k])
    np.savez_compressed(os.path.join(HERE, "new_map_points.npz"), **out)
    print("wrote new_map_points.npz:", {k: len(out[k + "_points"]) for k in TN.FIXTURE_SCENES})


if __name__ == "__main__":
    main()

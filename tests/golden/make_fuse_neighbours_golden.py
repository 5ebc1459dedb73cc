"""Regenerates tests/golden/fuse_neighbours.npz: a seeded SearchInNeighbors scene and what the flat oracle (oracle/pyfn.py) answers
for it.  python tests/golden/make_fuse_neighbours_golden.py"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from ccm_slam_b200 import synth_match as sm  # noqa: E402
from oracle import pyfn  # noqa: E402

if __name__ == "__main__":
    sc = sm.make_fuse_scene(n_first=3, n_second=2, n=200, seed=11, boundary=40)
    fwd, bwd = pyfn.oracle(sc)
    np.savez_compressed(os.path.join(os.path.dirname(os.path.abspath(__file__)), "fuse_neighbours.npz"),
                        fwd=fwd, bwd=bwd, **sm.fuse_scene_arrays(sc))
    print("fwd matches %d, bwd matches %d" % ((fwd >= 0).sum(), (bwd >= 0).sum()))

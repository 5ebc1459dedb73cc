"""Regenerates tests/golden/search_and_fuse.npz: a seeded loop scene and a seeded merge scene of LoopFinder / MapMerger::SearchAndFuse
and what the searches answer for them.  Where the reference's own ORBmatcher::Fuse(Scw) is built (oracle/_ref), the answer is written
from it, keyframe by keyframe, and checked against the flat oracle (oracle/pysf.py) first; elsewhere it is the oracle's.
python tests/golden/make_search_and_fuse_golden.py"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from ccm_slam_b200 import synth_match as sm  # noqa: E402
from oracle import pyoracle, pysf  # noqa: E402


def reference(sc):
    """the reference's Fuse(pKF, Scw, vpLoopMapPoints, 4, vpReplacePoints) for each keyframe, or None where it is not built"""
    if pyoracle.ref_match() is None:
        return None
    p = sc["points"]
    pts = dict(pos=p["pos"], normal=p["normal"], min_dist=p["min_d"], max_dist=p["max_d"], desc=p["desc"], bad=p["skip"], do_not_replace=p["dnr"])
    rows = []
    for kf in sc["kfs"]:
        best, _ = pyoracle.ref_fuse(kf, kf["intr"], None, np.full(len(kf["desc"]), -1, np.int32), pts, 4.0, Scw=kf["Scw"])
        rows.append(best)
    return np.stack(rows).astype(np.int32)


def scenes():
    return {"loop": sm.make_search_and_fuse_scene("loop", n_kf=4, n=250, seed=11, boundary=40),
            "merge": sm.make_search_and_fuse_scene("merge", n_kf=4, n=250, seed=12, boundary=40)}


if __name__ == "__main__":
    out = {}
    for name, sc in scenes().items():
        best = pysf.oracle(sc)
        ref = reference(sc)
        if ref is not None:
            assert np.array_equal(ref, best), "the flat oracle disagrees with the reference's Fuse(Scw)"
            best = ref
        out[name + "_best"] = best
        out.update({name + "_" + k: v for k, v in sm.search_and_fuse_scene_arrays(sc).items()})
        print("%s: %d pairs found, written from %s" % (name, (best >= 0).sum(), "the reference" if ref is not None else "the oracle"))
    np.savez_compressed(os.path.join(os.path.dirname(os.path.abspath(__file__)), "search_and_fuse.npz"), **out)

"""Generates tests/golden/normal_depth_cv2.npz: MapPoint::UpdateNormalAndDepth (cslam/src/MapPoint.cpp:779-823) evaluated with
OpenCV's own arithmetic, point by point, on the scenes of synth.make_normal_depth:
    d = X - O_k                   cv2.subtract
    r = cv::norm(d)               cv2.norm
    normal = normal + d / r       cv2.scaleAdd(d, 1.0 / r, normal)   (what MatOp_AddEx evaluates the expression to)
    mNormalVector = normal / n    convertTo(CV_32F, 1.0 / n): x * (float)(1.0 / n) + 0.f.  Python's cv2 has no convertTo; this step is
                                  the scalar tail of convert_scale.simd.hpp's cvt_32f (the scale taken as float), not a cv2 call
    dist = (float) cv2.norm(X - O_ref), mfMaxDistance = dist * scale_ref, mfMinDistance = mfMaxDistance / scale_last (f32).
Before it writes, every value is checked against an independent numpy restatement (f64 squares, fma through an exact f64 product);
the generator refuses to write on any difference.  Run from the repo root (cv2 4.13):
    python tests/golden/make_normal_depth_golden.py
"""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", ".."))
from ccm_slam_b200 import synth  # noqa: E402

# random scenes with every edge case of the reference body: bad observers, points whose observers are all bad, points on an
# observer's centre, reference keyframes that do not observe the point, bad points (the first two in std::map order, so that the
# stand-in MapPoint objects of the shim tests can replay them); and the observer structure of a BA problem, in its own order
CASES = [dict(seed=41, K=60, P=1500, all_bad_frac=0.02, on_centre_frac=0.02, off_ref_frac=0.05, map_order=True),
         dict(seed=42, K=12, P=400, bad_kf_frac=0.3, bad_mp_frac=0.1, all_bad_frac=0.05, on_centre_frac=0.05, off_ref_frac=0.2, map_order=True),
         dict(seed=43, config="small")]


def scene(kw):
    kw = dict(kw)
    cfg = kw.pop("config", None)
    return synth.make_normal_depth(synth.make_config(cfg) if cfg else None, **kw)


def cv2_normal_depth(sc):
    import cv2
    P = len(sc["mp_ref"])
    normal = np.zeros((P, 3), np.float32); dmax = np.zeros(P, np.float32); dmin = np.zeros(P, np.float32); status = np.zeros(P, np.uint8)
    C = sc["kf_centre"].reshape(-1, 3, 1)
    for i in range(P):
        b, e = sc["obs_ptr"][i], sc["obs_ptr"][i + 1]
        if b == e or sc["mp_ref"][i] < 0:
            continue
        X = np.ascontiguousarray(sc["mp_pos"][i].reshape(3, 1))
        nv = np.zeros((3, 1), np.float32); n = 0
        for k in sc["obs_kf"][b:e]:
            if sc["kf_bad"][k]:
                continue
            d = cv2.subtract(X, C[k])
            r = cv2.norm(d)
            with np.errstate(divide="ignore"):
                nv = cv2.scaleAdd(d, np.float64(1.0) / np.float64(r), nv)
            n += 1
        dist = np.float32(cv2.norm(cv2.subtract(X, C[sc["mp_ref"][i]])))
        dmax[i] = np.float32(dist * sc["mp_scale_ref"][i])
        dmin[i] = np.float32(dmax[i] / sc["mp_scale_last"][i])
        with np.errstate(divide="ignore", invalid="ignore"):
            a = np.float32(np.float64(1.0) / np.float64(n))
            normal[i] = (nv.reshape(3) * a) + np.float32(0)
        status[i] = 1
    return dict(normal=normal, max_dist=dmax, min_dist=dmin, status=status)


def numpy_normal_depth(sc):
    """vectorised over points, one observer slot at a time; an independent statement of the same rules"""
    P = len(sc["mp_ref"]); ptr = sc["obs_ptr"]; deg = np.diff(ptr)
    X = sc["mp_pos"].astype(np.float32); C = sc["kf_centre"].astype(np.float32); bad = sc["kf_bad"].astype(bool)
    live = (deg > 0) & (sc["mp_ref"] >= 0)
    nv = np.zeros((P, 3), np.float32); n = np.zeros(P, np.int64)
    with np.errstate(divide="ignore", invalid="ignore"):
        for j in range(int(deg.max(initial=0))):
            sel = np.flatnonzero(live & (deg > j))
            k = sc["obs_kf"][ptr[sel] + j]
            sel, k = sel[~bad[k]], k[~bad[k]]
            d = (X[sel] - C[k]).astype(np.float32)
            d64 = d.astype(np.float64)
            r = np.sqrt((d64[:, 0] * d64[:, 0] + d64[:, 1] * d64[:, 1]) + d64[:, 2] * d64[:, 2])
            a = (1.0 / r).astype(np.float32).astype(np.float64)
            nv[sel] = (d64 * a[:, None] + nv[sel].astype(np.float64)).astype(np.float32)   # the f32 x f32 product is exact in f64: one rounding to f32 (up to double rounding, which the cv2 comparison would expose)
            n[sel] += 1
        ref = np.maximum(sc["mp_ref"], 0)
        pc = (X - C[ref]).astype(np.float64)
        dist = np.sqrt((pc[:, 0] * pc[:, 0] + pc[:, 1] * pc[:, 1]) + pc[:, 2] * pc[:, 2]).astype(np.float32)
        dmax = (dist * sc["mp_scale_ref"]).astype(np.float32)
        dmin = (dmax / sc["mp_scale_last"]).astype(np.float32)
        s = (1.0 / n.astype(np.float64)).astype(np.float32)
        normal = (nv * s[:, None] + np.float32(0)).astype(np.float32)
    normal[~live] = 0; dmax[~live] = 0; dmin[~live] = 0
    return dict(normal=normal, max_dist=dmax, min_dist=dmin, status=live.astype(np.uint8))


def same(a, b):
    return all(np.array_equal(a[k], b[k], equal_nan=True) for k in ("normal", "max_dist", "min_dist", "status"))


if __name__ == "__main__":
    import cv2
    store = {"cv2_version": np.array(cv2.__version__)}
    for c, kw in enumerate(CASES):
        sc = scene(kw)
        r = cv2_normal_depth(sc)
        if not same(r, numpy_normal_depth(sc)):
            raise SystemExit("case %d: cv2 and the numpy restatement disagree; nothing written" % c)
        for k, v in r.items():
            store["case%d_%s" % (c, k)] = v
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "normal_depth_cv2.npz")
    np.savez_compressed(path, **store)
    print("wrote", path, os.path.getsize(path), "bytes")

"""Generates tests/golden/sim3_correction.npz: the Sim3 correction pass of LoopFinder::CorrectLoop (cslam/src/LoopFinder.cpp:568-613)
and MapMerger::MergeMaps (cslam/src/MapMerger.cpp:349-395), evaluated by a witness written here, on the scenes of
synth.make_sim3_correction.  The witness walks the entries in map order as the reference does, with a live table of camera centres:
    Swi = CorrectedSiw.inverse(), Swi.map(Siw.map(P))   f64 scalar operations (Python floats: no FMA) in Eigen's / g2o's order
    P -> f32                                            Converter::toCvMat
    UpdateNormalAndDepth()                              the cv2 evaluation of make_normal_depth_golden.py, against the live centres
    R, t *= (1./s), toCvSE3                             f64, then each element to f32
    SetPose: Ow = -Rwc * tcw                            cv2.gemm on the f32 matrices
Before it writes, every output is checked against the oracle (oracle/libsim3_correction_oracle.so); the generator refuses to write on
any difference.  Inputs and outputs are both stored, so the fixture does not depend on the generator's random streams.  Run from the
repo root (cv2 4.13):
    python tests/golden/make_sim3_correction_golden.py
"""
import importlib.util
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "..", ".."))
from ccm_slam_b200 import api, synth  # noqa: E402

INPUTS = [k for k, _ in api.SIM3_CORRECTION_IN]
OUTPUTS = ("entry_Tcw", "entry_centre", "mp_entry", "mp_pos", "normal", "max_dist", "min_dist", "status")
EDGES = dict(K=14, P=500, window=6, null_frac=0.1, dup_frac=0.1, bad_mp_frac=0.05, tagged_frac=0.05, bad_kf_frac=0.3, all_bad_frac=0.08,
             off_ref_frac=0.3, no_ref_frac=0.03, empty_frac=0.1, null_entry_frac=0.1)
# the last case moves every entry's tx onto a point where tx * (1./s) and tx / s round to different floats (the reference multiplies)
CASES = [dict(kind="loop", seed=71, K=80, P=1500, n_loop=30, unlisted_frac=0.05),
         dict(kind="merge", seed=72, K=40, P=1200, unlisted_frac=0.05),
         dict(kind="loop", seed=73, n_loop=8, **EDGES),
         dict(kind="merge", seed=74, **EDGES),
         dict(kind="merge", seed=75, K=16, P=400, ties=True)]


def tie_translation(s, rng):
    """a translation t for scale s such that float(t * (1./s)) != float(t / s)"""
    inv = 1. / s
    while True:
        m = float(np.float32(rng.uniform(0.5, 4.0)))
        m = m + float(np.spacing(np.float32(m))) / 2            # halfway between two floats
        for t in (m * s, np.nextafter(m * s, 0), np.nextafter(m * s, 10)):
            if np.float32(t * inv) != np.float32(t / s):
                return float(t)


def scene(kw):
    kw = dict(kw)
    ties = kw.pop("ties", False)
    sc = synth.make_sim3_correction(**kw)
    if ties:
        rng = np.random.default_rng(kw["seed"])
        sc["entry_Siw_new"] = sc["entry_Siw_new"].copy()
        for e in range(len(sc["entry_kf"])):
            sc["entry_Siw_new"][e, 4] = tie_translation(sc["entry_Siw_new"][e, 7], rng)
    return sc


def _nd():
    spec = importlib.util.spec_from_file_location("make_normal_depth_golden", os.path.join(HERE, "make_normal_depth_golden.py"))
    mod = importlib.util.module_from_spec(spec); spec.loader.exec_module(mod)
    return mod


def _rotate(q, v):
    qx, qy, qz, qw = q
    ux = qy * v[2] - qz * v[1]; uy = qz * v[0] - qx * v[2]; uz = qx * v[1] - qy * v[0]
    ux = ux + ux; uy = uy + uy; uz = uz + uz
    return [v[0] + qw * ux + (qy * uz - qz * uy), v[1] + qw * uy + (qz * ux - qx * uz), v[2] + qw * uz + (qx * uy - qy * ux)]


def _map(S, v):
    r = _rotate(S[:4], v)
    return [S[7] * r[i] + S[4 + i] for i in range(3)]


def _inverse(S):
    q = [-S[0], -S[1], -S[2], S[3]]
    k = -1. / S[7]
    t = _rotate(q, [k * S[4], k * S[5], k * S[6]])
    return q + t + [1. / S[7]]


def _rotation(S):
    x, y, z, w = S[:4]
    tx, ty, tz = 2 * x, 2 * y, 2 * z
    twx, twy, twz = tx * w, ty * w, tz * w
    txx, txy, txz = tx * x, ty * x, tz * x
    tyy, tyz, tzz = ty * y, tz * y, tz * z
    return [[1 - (tyy + tzz), txy - twz, txz + twy], [txy + twz, 1 - (txx + tzz), tyz - twx], [txz - twy, tyz + twx, 1 - (txx + tyy)]]


def witness(sc):
    import cv2
    nd = _nd()
    E, P = len(sc["entry_kf"]), len(sc["mp_skip"])
    out = api.sim3_correction_out(E, P)
    out["mp_entry"][:] = -1
    out["mp_pos"][:] = sc["mp_pos"]
    centre = np.array(sc["kf_centre"], np.float32)
    tagged = np.array(sc["mp_skip"], bool)
    ptr, obs = sc["obs_ptr"], sc["obs_kf"]
    for e in range(E):
        Snew = [float(v) for v in sc["entry_Siw_new"][e]]; Sold = [float(v) for v in sc["entry_Siw_old"][e]]
        Swi = _inverse(Snew)
        for j in range(sc["slot_ptr"][e], sc["slot_ptr"][e + 1]):
            p = int(sc["slot_mp"][j])
            if p < 0 or tagged[p]:
                continue
            x = [float(v) for v in sc["mp_pos"][p]]
            out["mp_pos"][p] = np.array(_map(Swi, _map(Sold, x)), np.float64).astype(np.float32)
            tagged[p] = True
            out["mp_entry"][p] = e
            one = dict(kf_centre=centre, kf_bad=sc["kf_bad"], mp_pos=out["mp_pos"][p:p + 1], obs_ptr=np.array([0, ptr[p + 1] - ptr[p]], np.int64),
                       obs_kf=obs[ptr[p]:ptr[p + 1]], mp_ref=sc["mp_ref"][p:p + 1], mp_scale_ref=sc["mp_scale_ref"][p:p + 1],
                       mp_scale_last=sc["mp_scale_last"][p:p + 1])
            r = nd.cv2_normal_depth(one)
            for k in ("normal", "max_dist", "min_dist", "status"):
                out[k][p] = r[k][0]
        R = _rotation(Snew)
        inv = 1. / Snew[7]
        t = [Snew[4 + i] * inv for i in range(3)]
        T = np.eye(4, dtype=np.float32)
        T[:3, :3] = np.array(R, np.float64).astype(np.float32); T[:3, 3] = np.array(t, np.float64).astype(np.float32)
        Ow = cv2.gemm(np.ascontiguousarray(T[:3, :3].T), np.ascontiguousarray(T[:3, 3:4]), -1.0, None, 0.0).reshape(3)
        out["entry_Tcw"][e] = T
        out["entry_centre"][e] = Ow
        centre[sc["entry_kf"][e]] = Ow
    return out


def main():
    from oracle import pysc
    z = {}
    for c, kw in enumerate(CASES):
        sc = scene(kw)
        w = witness(sc)
        o = pysc.oracle(sc)
        for k in OUTPUTS:
            if not np.array_equal(w[k], o[k], equal_nan=True):
                raise SystemExit("case %d: witness and oracle differ in %s; not writing" % (c, k))
        for k in INPUTS:
            z["case%d_in_%s" % (c, k)] = np.asarray(sc[k])
        for k in OUTPUTS:
            z["case%d_%s" % (c, k)] = w[k]
        print("case %d: %d entries, %d points moved, %d NaN normals" % (c, len(sc["entry_kf"]), (w["mp_entry"] >= 0).sum(),
                                                                         np.isnan(w["normal"]).any(1).sum()))
    np.savez_compressed(os.path.join(HERE, "sim3_correction.npz"), **z)


if __name__ == "__main__":
    main()

"""Scenes for the single-vertex optimisations (PoseOptimizationClient, OptimizeSim3) at the edges where they go wrong (test
infrastructure): boundary sizes around the `edges().size() < 10` break and the 256-thread stride, Huber thresholds other than 10,
frames whose edges are all gross outliers, bad starts whose edges flip between inlier and outlier across rounds, points behind the
camera, a point at camera depth exactly 0, measurements that are exact on the optical axis (rho == 0), calls that end on a rejected
full step (stale cached errors), frames whose every edge becomes an outlier (no active edge), Sim3 with two different cameras, with
too few surviving pairs, with no rejected pair, and under fix_scale.

Every scene is a dict in the layout of ccm_slam_b200.synth.make_pose_opt / make_sim3_opt, plus "name", and
"underdetermined_from" = the first optimize() call that has fewer residuals than unknowns, where there is one."""
from __future__ import annotations

import numpy as np

from ccm_slam_b200 import synth

EUROC = tuple(np.float32(v) for v in synth.EUROC_INTR)   # 752x480
CAM640 = tuple(np.float32(v) for v in (520.9, 521.0, 325.1, 249.7))   # 640x480, fx ~ 520


def _cut(d, n, keys):
    for k in keys:
        d[k] = d[k][:n]
    return d


def _pose(name, n=300, **kw):
    d = _cut(synth.make_pose_opt(n=max(n, 1), **kw), n, ("Xw", "uv", "inv_sigma2"))
    d["name"] = name
    return d


def pose_all_outliers(n=40, seed=31):
    """every measurement moved by hundreds of pixels: almost every edge leaves after round 1 and the frame ends with one inlier"""
    d = _pose("pose_all_outliers", n=n, seed=seed, outlier_frac=0.0)
    rng = np.random.default_rng(seed)
    d["uv"] = (d["uv"] + rng.choice([-1, 1], (n, 2)) * rng.uniform(300, 600, (n, 2))).astype(np.float32)
    d["underdetermined_from"] = 1    # rounds 2-4 keep one or two edges: fewer residuals than the 6 unknowns
    return d


def pose_bad_start(n=200, seed=41):
    """a start far from the truth with many outliers: edges flip between inlier and outlier across the four rounds"""
    return _pose("pose_bad_start", n=n, seed=seed, outlier_frac=0.3, pose_noise=(0.12, 0.35), noise_px=1.5)


def pose_behind(n=120, seed=51):
    """a tenth of the points behind the camera (negative depth): finite errors of the wrong sign of projection"""
    d = _pose("pose_behind", n=n, seed=seed, outlier_frac=0.05)
    T = d["Tcw0"]
    k = np.arange(0, n, 10)
    q, t = T[:4], T[4:]
    # X_w of a camera point (x, y, -z): X_w = R^T (X_c - t)
    qi = np.array([-q[0], -q[1], -q[2], q[3]])
    rng = np.random.default_rng(seed + 1)
    for i in k:
        Xc = np.array([rng.uniform(-1, 1), rng.uniform(-1, 1), -rng.uniform(1.0, 4.0)])
        d["Xw"][i] = synth._quat_rot(qi, Xc - t).astype(np.float32)
    return d


def pose_depth_zero(n=30, seed=61):
    """point 0 at camera depth exactly 0 at the start (identity rotation, t_z = -X_z, both exactly representable): its error is
    infinite, H and b are NaN in round 1, every Cholesky factorisation fails and the trial is rejected with tempChi = DBL_MAX"""
    d = _pose("pose_depth_zero", n=n, seed=seed, outlier_frac=0.1, pose_noise=(0.0, 0.05))
    X = d["Xw"].astype(np.float64)
    tz = np.float64(-0.25)
    d["Tcw0"] = np.array([0.0, 0.0, 0.0, 1.0, d["Tcw0"][4], d["Tcw0"][5], tz])
    d["Xw"][:, 2] = (X[:, 2] + 0.5).astype(np.float32)
    d["Xw"][0] = np.array([0.375, -0.125, 0.25], np.float32)        # z_c = 0.25 + (-0.25) = 0 exactly
    return d


def pose_on_axis(n=12, seed=71):
    """every point on the optical axis of an identity pose with its exact measurement (cx, cy): chi2 = 0, b = 0, x = 0 and
    the first trial ends the call with rho == 0"""
    fx, fy, cx, cy = EUROC
    Z = np.linspace(2.0, 8.0, n)
    Xw = np.stack([np.zeros(n), np.zeros(n), Z], 1).astype(np.float32)
    uv = np.tile(np.array([cx, cy], np.float32), (n, 1))
    return dict(name="pose_on_axis", Tcw0=np.array([0.0, 0.0, 0.0, 1.0, 0.0, 0.0, 0.0]), Xw=Xw, uv=uv,
                inv_sigma2=np.ones(n, np.float32), intr=EUROC)


def pose_weightless(n=12, seed=91):
    """inv_sigma2 = 0 on every edge: H = 0, b = 0, lambda = 1e-5 * 0 = 0, so every factorisation of H + lambda I fails and every
    call ends after ten rejected trials"""
    d = _pose("pose_weightless", n=n, seed=seed, outlier_frac=0.0)
    d["inv_sigma2"] = np.zeros(n, np.float32)
    return d


FAR_PX = np.float32(1e25)


def pose_stale(n=120, seed=201):
    """a bad start plus one measurement 1e25 px away.  That edge's Huber cost (~7e25) swamps the chi2 sum: the other edges' change
    under a step is below one ulp of the total, so the first trial of round 1 gives tempChi == currentChi exactly, is rejected,
    and ends the call with rho == 0.  Its weight rho' ~ 1e-25 leaves H and b to the other edges, so that trial is a full
    Gauss-Newton step: the errors the classification reads are those of a state the estimate never took."""
    d = _pose("pose_stale", n=n, seed=seed, outlier_frac=0.15, pose_noise=(0.05, 0.2))
    d["uv"][0] = FAR_PX
    return d


def pose_heavy(n=60, seed=203):
    """inv_sigma2 = 1e6: no edge stays under 5.991, so every edge is an outlier after round 1, rounds 2-4 have no active edge
    (optimize returns -1) and classify every edge from errors recomputed at the reset estimate"""
    d = _pose("pose_heavy", n=n, seed=seed, outlier_frac=0.0)
    d["inv_sigma2"] = np.full(n, 1e6, np.float32)
    return d


def pose_size(n, seed=None):
    return _pose(f"pose_n{n}", n=n, seed=1000 + n if seed is None else seed, outlier_frac=0.1 if n >= 3 else 0.0)


POSE_SIZES = (0, 1, 2, 3, 9, 10, 11, 255, 256, 257, 5000)


def pose_scenes():
    out = [pose_size(n) for n in POSE_SIZES]
    out += [pose_all_outliers(), pose_bad_start(), pose_behind(), pose_depth_zero(), pose_on_axis(), pose_weightless(), pose_stale(),
            pose_heavy(),
            _pose("pose_clean", n=60, seed=81, outlier_frac=0.0, noise_px=0.3)]
    return out


# ---- Sim3 ---------------------------------------------------------------------------------------------------------------------
def _reproject(d, K1, K2, seed, noise_px=0.7, outlier_frac=0.2):
    """measurements of d's points in two cameras K1 / K2 (the points stay those of make_sim3_opt)"""
    rng = np.random.default_rng(seed)
    n = len(d["P1c"])
    proj = lambda P, K: np.stack([K[0] * P[:, 0] / P[:, 2] + K[2], K[1] * P[:, 1] / P[:, 2] + K[3]], 1)
    s1, s2 = 1 / np.sqrt(d["w1"]), 1 / np.sqrt(d["w2"])
    uv1 = proj(d["P1c"].astype(np.float64), K1) + rng.standard_normal((n, 2)) * noise_px * s1[:, None]
    uv2 = proj(d["P2c"].astype(np.float64), K2) + rng.standard_normal((n, 2)) * noise_px * s2[:, None]
    bad = rng.random(n) < outlier_frac
    uv1[bad] += rng.uniform(-40, 40, (int(bad.sum()), 2))
    d.update(uv1=uv1.astype(np.float32), uv2=uv2.astype(np.float32), K1=K1, K2=K2)
    return d


def _sim3(name, th2=10.0, cams=None, n=120, **kw):
    d = _cut(synth.make_sim3_opt(n=max(n, 1), **kw), n, ("P1c", "P2c", "uv1", "uv2", "w1", "w2"))
    if cams is not None:
        d = _reproject(d, cams[0], cams[1], kw.get("seed", 0) + 7, outlier_frac=kw.get("outlier_frac", 0.2))
    d["th2"] = np.float32(th2)
    d["name"] = name
    return d


def sim3_stale(n=60, seed=202):
    """pair 0 measured 1e25 px away in keyframe 1: as pose_stale, the first call ends after one rejected full step (rho == 0)
    and the first classification reads the errors of that step"""
    d = _sim3("sim3_stale", n=n, seed=seed)
    d["uv1"][0] = FAR_PX
    return d


def sim3_scenes():
    return [
        _sim3("sim3_two_cams", n=100, seed=101, cams=(EUROC, CAM640)),
        _sim3("sim3_two_cams_rev", n=80, seed=102, cams=(CAM640, EUROC)),
        _sim3("sim3_two_cams_fix", n=90, seed=103, cams=(EUROC, CAM640), fix_scale=True),
        _sim3("sim3_th5991", n=100, seed=104, th2=5.991, cams=(EUROC, CAM640)),
        _sim3("sim3_th20", n=100, seed=105, th2=20.0, cams=(CAM640, EUROC)),
        _sim3("sim3_fix_scale", n=120, seed=106, fix_scale=True),
        _sim3("sim3_too_few", n=14, seed=107, outlier_frac=0.7),
        _sim3("sim3_no_reject", n=40, seed=108, outlier_frac=0.0, noise_px=0.2),
        _sim3("sim3_n127", n=127, seed=109, cams=(EUROC, CAM640)),
        _sim3("sim3_n128", n=128, seed=110),
        _sim3("sim3_n129", n=129, seed=111, cams=(CAM640, EUROC)),
        _sim3("sim3_n9", n=9, seed=112, outlier_frac=0.0),
        _sim3("sim3_n10", n=10, seed=113, outlier_frac=0.0, noise_px=0.2),
        dict(_sim3("sim3_n1", n=1, seed=114, outlier_frac=0.0), underdetermined_from=0),   # 4 residuals, 7 unknowns
        _sim3("sim3_n0", n=0, seed=115),
        _sim3("sim3_n600", n=600, seed=116, outlier_frac=0.15, cams=(EUROC, CAM640)),
        sim3_stale(),
    ]


def by_name(scenes):
    return {d["name"]: d for d in scenes}

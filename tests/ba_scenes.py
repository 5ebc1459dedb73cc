"""Global-BA scenes built to sit where the linearisation, the pose update and the trial chi2 go wrong (tests/test_ba_ref.py,
tests/test_gpu_ba_steps.py).

Cameras on a 3 m baseline face one field of points, so any subset of them sees any point (the geometry of test_gpu_fused_z.py).
Every scene has:
  * four distinct f32 cameras, assigned per keyframe, with obs_uv projected from ground truth through each keyframe's own camera
    plus pixel noise of its octave; invSigma2 of all 8 octaves; 5 % gross outliers;
  * fixed keyframes among the free ones, and a landmark only fixed keyframes see;
  * edges without a kernel (flag bit 1), inactive edges (bit 0), and both bits together;
  * far points at depths 1e3-1e4 (their Hll is ~1e-8 of the largest entry);
  * a point behind every camera, observed by active edges;
  * inactive edges whose points sit at depth exactly 0 and 1e-300 in a fixed keyframe (0, at the identity pose) and in a free one
    (DEPTH0_FREE_KF, at the identity rotation with t_z = 0), so that k_linearize, k_pose_pass and k_residual all meet them;
  * edges whose chi2 at the start lies in the Huber band between float(delta^2) and double(delta^2), or one float ulp either side
    of float(delta^2), for HUBER_GBA and HUBER_LOCAL, tuned through the f32 weight and kept only where the restatement confirms it.
"multicam" adds near points 0.05 in front of two fixed keyframes (the largest diagonal entry is then in Hll).
"sizes" has landmarks of 1, 2, 32, 33, 97, 127, 128, 129 and 300 observations around the 128-observation chunks of k_linearize; its
depth-0 point has 130 observations, all inactive, so it spans two chunks, and its Huber-band edges sit on the largest landmarks.  It
has no near points, so its largest diagonal entry is in Hpp.
"""
from __future__ import annotations

import numpy as np

from ccm_slam_b200 import api, synth
from tests import ba_ref

CAMERAS = np.array([[458.654, 457.296, 367.215, 248.375],
                    [435.2, 435.2, 367.2, 252.2],
                    [520.9, 521.0, 325.1, 249.7],
                    [381.5, 383.25, 300.0, 230.5]], np.float32).astype(np.float64)
SPECIAL = [1, 2, 32, 33, 97, 127, 128, 129, 300]
DELTAS = (api.HUBER_GBA, api.HUBER_LOCAL)


def _cameras(rng, K):
    """camera centres on a 3 m baseline with a few centimetres of jitter; keyframe 0 at the origin"""
    C = np.stack([np.linspace(-1.5, 1.5, K), rng.uniform(-0.1, 0.1, K), rng.uniform(-0.1, 0.1, K)], 1)
    C[0] = 0.0
    return C


def _observers(rng, K, sizes):
    kf = np.concatenate([np.sort(rng.choice(K, s, replace=False)) for s in sizes]).astype(np.int32)
    mp = np.repeat(np.arange(len(sizes)), sizes).astype(np.int32)
    return kf, mp


def _finish(rng, C, X, kf, mp, intr, fixed_idx, name, extra_uv=None):
    """observations through each keyframe's own camera with octave noise and outliers, perturbed free poses (orientation near the
    identity), perturbed points, and edge flags"""
    K, E = len(C), kf.size
    Xc = X[mp] - C[kf]
    octave = np.arange(E) % 8
    rng.shuffle(octave)
    sigma = synth.SCALE_FACTOR ** octave
    I = intr[kf]
    with np.errstate(all="ignore"):
        uv = np.stack([I[:, 0] * Xc[:, 0] / Xc[:, 2] + I[:, 2], I[:, 1] * Xc[:, 1] / Xc[:, 2] + I[:, 3]], 1)
    uv += rng.normal(size=(E, 2)) * sigma[:, None]
    out = rng.random(E) < 0.05
    uv[out] += rng.uniform(10, 50, (out.sum(), 1)) * rng.choice([-1.0, 1.0], (out.sum(), 2))
    if extra_uv is not None:
        m = extra_uv[0]
        uv[m] = extra_uv[1]
    q_gt = np.tile([0.0, 0.0, 0.0, 1.0], (K, 1)); t_gt = -C
    drot = synth._rotvec_to_quat(rng.normal(size=(K, 3)) * 0.01)
    q0 = synth._quat_mul(drot, q_gt)
    t0 = synth._quat_rot(drot, t_gt) + rng.normal(size=(K, 3)) * 0.03
    fixed = np.zeros(K, np.uint8); fixed[fixed_idx] = 1
    q0[fixed == 1] = q_gt[fixed == 1]; t0[fixed == 1] = t_gt[fixed == 1]
    q0 /= np.linalg.norm(q0, axis=-1, keepdims=True)
    pts0 = X.copy()
    ordinary = np.abs(X[:, 2]) < 100
    pts0[ordinary] += rng.normal(size=(ordinary.sum(), 3)) * 0.05
    pts0 = pts0.astype(np.float32).astype(np.float64)
    flags = np.zeros(E, np.uint8)
    u = rng.random(E)
    flags[u < 0.03] = 1
    flags[(u >= 0.03) & (u < 0.06)] = 3
    flags[(u >= 0.06) & (u < 0.2)] = 2
    return synth.BAProblem(poses=np.ascontiguousarray(np.concatenate([q0, t0.astype(np.float32).astype(np.float64)], -1)),
                           intr=np.ascontiguousarray(intr), fixed=fixed, points=np.ascontiguousarray(pts0),
                           obs_kf=kf, obs_mp=mp, obs_uv=np.ascontiguousarray(uv.astype(np.float32)),
                           obs_w=(1.0 / sigma ** 2).astype(np.float32), edge_flags=flags, name=name)


DEPTH0_FREE_KF = 2     # a free keyframe put at the identity rotation with t_z = 0: the depth-0 points sit at depth 0 in it too


def _far(rng, K, n):
    return [(np.array([rng.uniform(-200, 200), rng.uniform(-100, 100), rng.uniform(1e3, 1e4)]), np.sort(rng.choice(K, 6, replace=False)))
            for _ in range(n)]


def _with_extras(X, kf, mp, extra):
    """append the extra (point, observers) landmarks to the scene arrays; returns X, kf, mp and the first extra landmark index"""
    n0 = len(X)
    X = np.concatenate([X, np.stack([x for x, _ in extra])])
    kf = np.concatenate([kf] + [np.asarray(o, np.int32) for _, o in extra])
    mp = np.concatenate([mp] + [np.full(len(o), n0 + j, np.int32) for j, (_, o) in enumerate(extra)])
    return X, kf, mp, n0


def _depth0(p, mp, depth0, X):
    """keyframe 0 (fixed) at the identity pose and keyframe DEPTH0_FREE_KF (free) at the identity rotation with t_z = 0: the depth-0
    points (world z = 0 and 1e-300) sit at depth exactly 0 and 1e-300 in both.  Every edge of those points is inactive (flag bit 0);
    returns the edges at depth 0 / 1e-300"""
    p.poses[0] = [0, 0, 0, 1, 0, 0, 0]
    p.poses[DEPTH0_FREE_KF, :4] = [0, 0, 0, 1]
    p.poses[DEPTH0_FREE_KF, 6] = 0.0
    p.points[depth0] = X[depth0]
    on = np.isin(mp, depth0) & np.isin(p.obs_kf, [0, DEPTH0_FREE_KF])
    p.edge_flags[np.isin(mp, depth0)] = 1
    return np.flatnonzero(on)


def make_multicam(seed=41, K=40, n_base=500):
    rng = np.random.default_rng(seed)
    C = _cameras(rng, K)
    intr = CAMERAS[np.arange(K) % len(CAMERAS)]
    fixed_idx = [0, 9, 23]
    sizes = [int(s) for s in rng.integers(3, 9, n_base)]
    X = np.stack([rng.uniform(-1, 1, n_base), rng.uniform(-0.6, 0.6, n_base), rng.uniform(6, 10, n_base)], 1)
    kf, mp = _observers(rng, K, sizes)
    extra = [  # (point, its observers)
        *_far(rng, K, 6),                                           # far
        (C[9] + [0.01, 0.005, 0.05], [9]), (C[23] + [-0.01, -0.004, 0.05], [23]),   # near, in front of fixed keyframes
        (np.array([0.3, 0.1, -3.0]), [3, 17, 35]),                  # behind every camera
        (np.array([0.2, -0.1, 7.0]), [0, 9]),                       # seen only by fixed keyframes
        (np.array([1.0, 2.0, 0.0]), [0, DEPTH0_FREE_KF]), (np.array([1.0, 2.0, 1e-300]), [0, DEPTH0_FREE_KF]),   # depth 0 and 1e-300
    ]
    X, kf, mp, n0 = _with_extras(X, kf, mp, extra)
    far, near, behind, only_fixed, depth0 = (np.arange(n0, n0 + 6), np.arange(n0 + 6, n0 + 8), n0 + 8, n0 + 9, np.arange(n0 + 10, n0 + 12))
    rnd = np.flatnonzero(np.isin(mp, depth0) | (mp == behind))
    p = _finish(rng, C, X, kf, mp, intr, fixed_idx, "multicam", extra_uv=(rnd, rng.uniform([0, 0], [752, 480], (rnd.size, 2))))
    p.points[near] = X[near].astype(np.float32)     # unperturbed: a depth of 0.05 stays 0.05
    p.obs_w[np.isin(mp, near)] = 1.0                # octave 0
    fl = p.edge_flags
    fl[np.isin(mp, np.concatenate([far, near, [behind, only_fixed]]))] &= 2     # active, kernel as drawn
    fl[mp == behind] = 0
    d0 = _depth0(p, mp, depth0, X)
    p.special = dict(depth0=d0, behind=np.flatnonzero(mp == behind), far=np.flatnonzero(np.isin(mp, far)),
                     near=np.flatnonzero(np.isin(mp, near)), only_fixed_point=only_fixed)
    tune_band(p)
    return p


def make_sizes(seed=5, K=320, n_base=900):
    """like multicam, without near points (so that the largest diagonal entry is in Hpp); the depth-0 point is a landmark of 130
    observations, all inactive, so that it spans two chunks of k_linearize, and the Huber band sits on the largest landmarks first"""
    rng = np.random.default_rng(seed)
    C = _cameras(rng, K)
    intr = CAMERAS[np.arange(K) % len(CAMERAS)]
    fixed_idx = [0, 1, 100, 201]
    sizes = [int(s) for s in rng.integers(3, 9, n_base)]
    at = np.sort(rng.choice(n_base, len(SPECIAL), replace=False))
    for i, s in sorted(zip(at, SPECIAL), reverse=True):
        sizes.insert(int(i), s)
    P = len(sizes)
    X = np.stack([rng.uniform(-1, 1, P), rng.uniform(-0.6, 0.6, P), rng.uniform(6, 10, P)], 1)
    kf, mp = _observers(rng, K, sizes)
    others = np.setdiff1d(np.arange(K), [0, DEPTH0_FREE_KF])
    extra = [
        *_far(rng, K, 6),
        (np.array([0.3, 0.1, -3.0]), [3, 150, 290]),                # behind every camera
        (np.array([0.2, -0.1, 7.0]), [100, 201]),                   # seen only by fixed keyframes
        (np.array([1.0, 2.0, 0.0]), np.sort(np.concatenate([[0, DEPTH0_FREE_KF], rng.choice(others, 128, replace=False)]))),
        (np.array([1.0, 2.0, 1e-300]), [0, DEPTH0_FREE_KF]),
    ]
    X, kf, mp, n0 = _with_extras(X, kf, mp, extra)
    far, behind, only_fixed, depth0 = np.arange(n0, n0 + 6), n0 + 6, n0 + 7, np.arange(n0 + 8, n0 + 10)
    rnd = np.flatnonzero(np.isin(mp, depth0) | (mp == behind))
    p = _finish(rng, C, X, kf, mp, intr, fixed_idx, "sizes", extra_uv=(rnd, rng.uniform([0, 0], [752, 480], (rnd.size, 2))))
    fl = p.edge_flags
    fl[np.isin(mp, np.concatenate([far, [behind, only_fixed]]))] &= 2
    fl[mp == behind] = 0
    d0 = _depth0(p, mp, depth0, X)
    p.special = dict(depth0=d0, behind=np.flatnonzero(mp == behind), far=np.flatnonzero(np.isin(mp, far)),
                     near=np.zeros(0, np.int64), only_fixed_point=only_fixed, depth0_landmark=int(depth0[0]))
    tune_band(p, prefer_large=True)
    return p


def band_targets(delta):
    """the chi2 intervals of the Huber band for delta: between double(delta^2) and float(delta^2), and one float ulp either side
    of float(delta^2)"""
    dd = delta * delta
    df = float(np.float32(dd))
    up = float(np.nextafter(np.float32(df), np.float32(np.inf)))
    dn = float(np.nextafter(np.float32(df), np.float32(-np.inf)))
    return [(min(dd, df), max(dd, df)), (dn, dn), (up, up)]


def tune_band(p, per_target=3, prefer_large=False):
    """retune the f32 weight of a few edges per band target so that their chi2 at the start state lands in it; an edge is kept only
    where the restated chi2, with its bound, lies strictly inside [lo, hi] (or on the side of float(delta^2) its target names).
    prefer_large: edges of landmarks with more than one 128-observation chunk first"""
    lin = ba_ref.Lin(p, delta=api.HUBER_GBA)
    with np.errstate(all="ignore"):
        s = (lin.err ** 2).sum(1)
    cand = np.flatnonzero((p.edge_flags == 0) & (s > 0.5) & (s < 50) & (lin.depth > 1))
    rng = np.random.default_rng(7)
    cand = rng.permutation(cand)
    if prefer_large:
        big = np.bincount(p.obs_mp)[p.obs_mp[cand]] > 128
        cand = np.concatenate([cand[big], cand[~big]])
    used = 0
    band = []
    w0 = p.obs_w.copy()
    for delta in DELTAS:
        df = float(np.float32(delta * delta))
        for lo, hi in band_targets(delta):
            got = 0
            while got < per_target and used < cand.size:
                i = cand[used]; used += 1
                for w in _weights_near(0.5 * (lo + hi) / s[i]):
                    if _confirm(p, i, w, lo, hi, df):
                        p.obs_w[i] = w
                        band.append((i, delta, lo, hi)); got += 1
                        break
                else:
                    p.obs_w[i] = w0[i]
    p.band = band


def _weights_near(w):
    w = np.float32(w)
    out = [w]
    a = b = w
    for _ in range(4):
        a = np.nextafter(a, np.float32(np.inf)); b = np.nextafter(b, np.float32(0))
        out += [a, b]
    return out


def _confirm(p, i, w, lo, hi, df):
    """the restated chi2 of edge i with weight w, and its bound, inside the target: strictly inside [lo, hi] for the band, and on
    the right side of float(delta^2) for the one-ulp targets"""
    kf, mp = int(p.obs_kf[i]), int(p.obs_mp[i])
    _, _, _, _, c = ba_ref.edge_terms(p.poses[kf], p.points[mp], p.obs_uv[i].astype(np.float64), p.intr[kf], float(w), ba_ref.R)
    v, e = float(c.v), c.e
    if lo == hi:                           # one float ulp from float(delta^2): within half an ulp of it, on its side
        half = abs(lo - df) / 2
        return abs(v - lo) + e < half
    return lo + e < v < hi - e


def states(oracle, p, delta=api.HUBER_GBA, iters=10):
    """the scene at its start, half-way along the oracle's run and at the oracle's end state"""
    r = oracle.ba_solve(p, iterations=iters, huber_delta=delta)
    end_q, end_x = r["poses"], r["points"]
    qa, qb = p.poses[:, :4], end_q[:, :4]
    qb = np.where((qa * qb).sum(1, keepdims=True) >= 0, qb, -qb)
    q = (qa + qb) / np.linalg.norm(qa + qb, axis=1, keepdims=True)
    mid_q = np.concatenate([q, (p.poses[:, 4:] + end_q[:, 4:]) / 2], 1)
    mid_q[p.fixed == 1] = p.poses[p.fixed == 1]
    mid_x = (p.points + end_x) / 2
    return [("start", p.poses, p.points), ("midway", mid_q, mid_x), ("end", end_q, end_x)]


def turned(poses, seed=3):
    """the poses turned by 2.5 rad about random axes (left-multiplied, w >= 0): far from the identity, so that exp(x) * T meets
    products with w < 0"""
    rng = np.random.default_rng(seed)
    ax = rng.normal(size=(len(poses), 3))
    r = synth._rotvec_to_quat(ax / np.linalg.norm(ax, axis=1, keepdims=True) * 2.5)
    q = synth._quat_mul(r, np.asarray(poses)[:, :4])
    q = np.where(q[:, 3:4] < 0, -q, q)
    q /= np.linalg.norm(q, axis=1, keepdims=True)
    return np.ascontiguousarray(np.concatenate([q, np.asarray(poses)[:, 4:]], 1))


def with_state(p, poses, points):
    q = p.copy()
    q.poses = np.ascontiguousarray(poses, np.float64); q.points = np.ascontiguousarray(points, np.float64)
    return q


_cache = {}


def scene(name):
    """the named scene, built once with every deliberate defect of ba_ref.MUT switched off"""
    if name not in _cache:
        saved = dict(ba_ref.MUT)
        ba_ref.MUT.update({k: False for k in ba_ref.MUT})
        try:
            _cache[name] = make_multicam() if name == "multicam" else make_sizes()
        finally:
            ba_ref.MUT.update(saved)
    return _cache[name]


SCENES = ("multicam", "sizes")

"""Seeded synthetic BA / pose-graph problems with the shapes BASELINE.json names.

No EuRoC data and no ROS exist in this environment, so configs 1-4 are realised as synthetic problems of
EuRoC-like shape (SURVEY.md §8(d), BASELINE.md §3); config 5 is synthetic by definition.  Distributions
follow BASELINE.md: pose noise N(0, 0.02 rad / 0.05 m), point noise N(0, 0.05 m), pixel noise
N(0, sigma_octave) with the octave drawn proportionally to the per-level ORB quotas
217:181:151:126:105:87:73:60 (S/ORBextractor.cpp:604-615), invSigma2 = 1.2^(-2 octave)
(S/ORBextractor.cpp:584-600), 5 % gross outliers.  Intrinsics: cslam/conf/vi_euroc.yaml:9-12.

Pure numpy; shared by tests, bench.py and the oracle legs so that CPU and GPU paths see identical bytes.
"""
from __future__ import annotations

import dataclasses

import numpy as np

EUROC_INTR = (458.654, 457.296, 367.215, 248.375)
OCTAVE_QUOTAS = np.array([217, 181, 151, 126, 105, 87, 73, 60], dtype=np.float64)
SCALE_FACTOR = 1.2

# named configurations (BASELINE.json "configs"); (est.) shapes from BASELINE.md §3
CONFIGS = {
    "cfg1": dict(kind="local", n_local=15, n_fixed=10, P=2000, obs_per_point=6, seed=1),
    "cfg2": dict(kind="local", n_local=15, n_fixed=10, P=2000, obs_per_point=6, seed=1),
    "cfg3": dict(kind="global", K=400, P=25000, obs_per_point=6, window=24, n_agents=2, seed=2),
    "cfg4": dict(kind="global", K=800, P=50000, obs_per_point=6, window=24, n_agents=4, seed=3),
    "cfg5": dict(kind="global", K=10000, P=1000000, obs_per_point=20, window=40, n_agents=1, seed=4),
    # small shapes for parity tests
    "tiny": dict(kind="global", K=3, P=20, obs_per_point=3, window=3, n_agents=1, seed=7),
    "small": dict(kind="global", K=40, P=1500, obs_per_point=5, window=12, n_agents=2, seed=11),
}


@dataclasses.dataclass
class BAProblem:
    poses: np.ndarray      # (K,7) f64: qx qy qz qw tx ty tz  (Tcw)
    intr: np.ndarray       # (K,4) f64: fx fy cx cy (f32-representable)
    fixed: np.ndarray      # (K,) u8
    points: np.ndarray     # (P,3) f64 (f32-representable)
    obs_kf: np.ndarray     # (E,) i32
    obs_mp: np.ndarray     # (E,) i32
    obs_uv: np.ndarray     # (E,2) f32
    obs_w: np.ndarray      # (E,) f32  invSigma2
    edge_flags: np.ndarray | None = None  # (E,) u8
    gt_poses: np.ndarray | None = None
    gt_points: np.ndarray | None = None
    name: str = ""

    @property
    def K(self): return int(self.poses.shape[0])
    @property
    def P(self): return int(self.points.shape[0])
    @property
    def E(self): return int(self.obs_kf.shape[0])

    def copy(self):
        return dataclasses.replace(self, **{f.name: (getattr(self, f.name).copy() if isinstance(getattr(self, f.name), np.ndarray) else getattr(self, f.name)) for f in dataclasses.fields(self)})


def _quat_mul(a, b):
    ax, ay, az, aw = a[..., 0], a[..., 1], a[..., 2], a[..., 3]
    bx, by, bz, bw = b[..., 0], b[..., 1], b[..., 2], b[..., 3]
    return np.stack([aw * bx + ax * bw + ay * bz - az * by,
                     aw * by + ay * bw + az * bx - ax * bz,
                     aw * bz + az * bw + ax * by - ay * bx,
                     aw * bw - ax * bx - ay * by - az * bz], axis=-1)


def _quat_rot(q, v):
    u = np.cross(q[..., :3], v)
    u = u + u
    return v + q[..., 3:4] * u + np.cross(q[..., :3], u)


def _rotvec_to_quat(rv):
    th = np.linalg.norm(rv, axis=-1, keepdims=True)
    half = 0.5 * th
    k = np.where(th > 1e-12, np.sin(half) / np.maximum(th, 1e-300), 0.5)
    return np.concatenate([rv * k, np.cos(half)], axis=-1)


def _mat_to_quat(R):
    """Shepperd-style branchy conversion (vectorised); sign fixed to w>=0 and normalised like SE3Quat."""
    from scipy.spatial.transform import Rotation
    q = Rotation.from_matrix(R).as_quat()  # x y z w
    q = np.where(q[..., 3:4] < 0, -q, q)
    return q / np.linalg.norm(q, axis=-1, keepdims=True)


def _helix_cameras(K, rng, radius=2.0, dtheta=0.02, dz=0.002, phase=0.0, z0=0.0):
    """Ground-truth world->camera poses on a helix, optical axis pointing radially outward."""
    k = np.arange(K)
    th = phase + dtheta * k
    C = np.stack([radius * np.cos(th), radius * np.sin(th), z0 + dz * k], axis=-1)  # camera centres
    zc = np.stack([np.cos(th), np.sin(th), np.zeros(K)], axis=-1)                   # look direction
    up = np.tile(np.array([0.0, 0.0, 1.0]), (K, 1))
    xc = np.cross(up, zc); xc /= np.linalg.norm(xc, axis=-1, keepdims=True)
    yc = np.cross(zc, xc)
    Rcw = np.stack([xc, yc, zc], axis=1)  # rows are camera axes in world -> Xc = Rcw (X - C)
    tcw = -np.einsum("kij,kj->ki", Rcw, C)
    return Rcw, tcw, C, zc


def make_global_ba(K, P, obs_per_point, window, n_agents=1, seed=0, outlier_frac=0.05,
                   pose_noise=(0.02, 0.05), point_noise=0.05, shared_frac=0.10, name="") -> BAProblem:
    rng = np.random.default_rng(seed)
    Ka = K // n_agents
    Rs, ts, Cs, Zs = [], [], [], []
    # the covisibility window spans 0.4 rad of the circle so that co-observers stay inside the 752x480 FOV
    dtheta = 0.4 / max(window, obs_per_point)
    for a in range(n_agents):
        n = Ka if a < n_agents - 1 else K - Ka * (n_agents - 1)
        R, t, C, z = _helix_cameras(n, rng, phase=0.0 + 0.3 * a, z0=0.15 * a, dtheta=dtheta)
        Rs.append(R); ts.append(t); Cs.append(C); Zs.append(z)
    Rcw = np.concatenate(Rs); tcw = np.concatenate(ts); C = np.concatenate(Cs); zdir = np.concatenate(Zs)
    agent_of = np.concatenate([np.full(len(r), a) for a, r in enumerate(Rs)])
    agent_start = np.concatenate([[0], np.cumsum([len(r) for r in Rs])])

    # each landmark: centre keyframe c (spread uniformly), placed in front of c at depth U[2,10]
    centre = np.sort(rng.integers(0, K, size=P))
    depth = rng.uniform(2.0, 10.0, size=P)
    lat = rng.uniform(-0.25, 0.25, size=(P, 2)) * depth[:, None]  # lateral offsets in the camera frame
    Xc = np.stack([lat[:, 0], lat[:, 1], depth], axis=-1)
    gt_pts = np.einsum("pji,pj->pi", Rcw[centre], Xc - tcw[centre])  # R^T (Xc - t)

    n_obs = obs_per_point
    w = max(window, n_obs)
    a_of_c = agent_of[centre]
    lo = np.maximum(agent_start[a_of_c], centre - w // 2)
    hi = np.minimum(agent_start[a_of_c + 1], lo + w)
    lo = np.maximum(agent_start[a_of_c], hi - w)
    span = hi - lo
    # choose n_obs distinct offsets in [0, span) per landmark
    keys = rng.random((P, w))
    keys[np.arange(w)[None, :] >= span[:, None]] = 2.0
    sel = np.sort(np.argpartition(keys, n_obs - 1, axis=1)[:, :n_obs], axis=1)
    valid = sel < span[:, None]
    kf = lo[:, None] + sel
    # inter-agent sharing: a fraction of landmarks gets half of its observers moved to another agent's
    # keyframes at the same trajectory phase (map-merge overlap)
    if n_agents > 1 and shared_frac > 0:
        shared = rng.random(P) < shared_frac
        other = (a_of_c + 1 + rng.integers(0, n_agents - 1, size=P)) % n_agents
        rel = centre - agent_start[a_of_c] + np.rint(0.3 * (a_of_c - other) / dtheta).astype(np.int64)  # same phase
        oc = agent_start[other] + np.clip(rel, 0, (agent_start[other + 1] - agent_start[other]) - 1)
        half = n_obs // 2
        okf = oc[:, None] + np.arange(-(half // 2), half - half // 2)[None, :]
        okf = np.clip(okf, agent_start[other][:, None], agent_start[other + 1][:, None] - 1)
        kf[shared, :half] = okf[shared]
        kf.sort(axis=1)
        dup = np.zeros_like(valid)
        dup[:, 1:] = kf[:, 1:] == kf[:, :-1]
        valid &= ~dup
    mp = np.broadcast_to(np.arange(P)[:, None], kf.shape)
    kf = kf[valid].astype(np.int32); mp = mp[valid].astype(np.int32)

    # ground-truth projections
    fx, fy, cx, cy = EUROC_INTR
    Xcam = np.einsum("eij,ej->ei", Rcw[kf], gt_pts[mp]) + tcw[kf]
    good = (Xcam[:, 2] > 0.5) & (np.abs(fx * Xcam[:, 0] / Xcam[:, 2]) < 1.1 * cx) & (np.abs(fy * Xcam[:, 1] / Xcam[:, 2]) < 1.1 * cy)
    kf, mp, Xcam = kf[good], mp[good], Xcam[good]
    E = kf.shape[0]
    octave = rng.choice(8, size=E, p=OCTAVE_QUOTAS / OCTAVE_QUOTAS.sum())
    sigma = SCALE_FACTOR ** octave
    uv = np.stack([fx * Xcam[:, 0] / Xcam[:, 2] + cx, fy * Xcam[:, 1] / Xcam[:, 2] + cy], axis=-1)
    uv += rng.normal(size=(E, 2)) * sigma[:, None]
    out = rng.random(E) < outlier_frac
    ang = rng.uniform(0, 2 * np.pi, size=E)
    mag = rng.uniform(10.0, 50.0, size=E)
    uv[out] += (np.stack([np.cos(ang), np.sin(ang)], -1) * mag[:, None])[out]
    inv_sigma2 = (1.0 / (SCALE_FACTOR ** (2 * octave))).astype(np.float32)

    # perturbed initial estimates
    q_gt = _mat_to_quat(Rcw)
    drot = _rotvec_to_quat(rng.normal(size=(K, 3)) * pose_noise[0])
    dt = rng.normal(size=(K, 3)) * pose_noise[1]
    q0 = _quat_mul(drot, q_gt)
    t0 = _quat_rot(drot, tcw) + dt
    fixed = np.zeros(K, np.uint8); fixed[0] = 1
    q0[0] = q_gt[0]; t0[0] = tcw[0]
    q0 = np.where(q0[:, 3:4] < 0, -q0, q0)
    q0 /= np.linalg.norm(q0, axis=-1, keepdims=True)
    pts0 = (gt_pts + rng.normal(size=(P, 3)) * point_noise).astype(np.float32).astype(np.float64)
    t0 = t0.astype(np.float32).astype(np.float64)  # translations arrive as f32 (S/Converter.cc:48)

    intr = np.tile(np.array(EUROC_INTR, np.float32).astype(np.float64), (K, 1))
    return BAProblem(poses=np.ascontiguousarray(np.concatenate([q0, t0], -1)), intr=intr, fixed=fixed,
                     points=np.ascontiguousarray(pts0), obs_kf=np.ascontiguousarray(kf),
                     obs_mp=np.ascontiguousarray(mp), obs_uv=np.ascontiguousarray(uv.astype(np.float32)),
                     obs_w=np.ascontiguousarray(inv_sigma2),
                     gt_poses=np.concatenate([q_gt, tcw], -1), gt_points=gt_pts, name=name)


def make_local_ba(n_local=15, n_fixed=10, P=2000, obs_per_point=6, seed=1, name="") -> BAProblem:
    """LocalBundleAdjustmentClient-shaped window: the newest n_local KFs are free, the n_fixed older ones that
    co-observe the local points are fixed (S/Optimizer.cpp:351-404)."""
    K = n_local + n_fixed
    p = make_global_ba(K, P, obs_per_point, window=K, n_agents=1, seed=seed, name=name)
    p.fixed[:] = 0
    p.fixed[:n_fixed] = 1
    # fixed keyframes are consistent with the map in the reference (they were optimised before): keep them at GT
    gt = p.gt_poses[:n_fixed].copy()
    gt[:, 4:] = gt[:, 4:].astype(np.float32)
    p.poses[:n_fixed] = gt
    return p


def make_awkward_ba(seed=21) -> BAProblem:
    """A global-BA problem built to sit on the edges of the Schur path's schedules (tests/test_gpu_schur.py checks it):
    199 free keyframes, fixed keyframes among the free ones, co-observations at free-pose offsets 43, 44 and beyond, landmarks with
    more than 160 observations (more than one 128-observation chunk of the landmark schedule), runs of two-observation landmarks,
    one keyframe pair sharing more than 4096 landmarks, a landmark only fixed keyframes see, one seen once, edges with flag bits
    0 and 1, and observations in shuffled order.
    The added landmarks are not geometrically consistent (only the linear system at the initial state is of interest)."""
    rng = np.random.default_rng(seed)
    p = make_global_ba(203, 3000, 6, window=50, n_agents=1, seed=seed)
    K = p.K
    fixed = np.zeros(K, np.uint8)
    fixed[[0, 13, 50, 101]] = 1                       # 199 free; 13, 50 and 101 sit among the free poses
    free_idx = np.flatnonzero(fixed == 0)
    obs = [(p.obs_kf, p.obs_mp, p.obs_uv, p.obs_w)]
    pts = [p.points]
    centre = [np.bincount(p.obs_mp, weights=p.obs_kf, minlength=p.P) / np.maximum(np.bincount(p.obs_mp, minlength=p.P), 1)]
    nxt = p.P

    def add(kfs):
        nonlocal nxt
        kfs = np.asarray(kfs, np.int32)
        n = kfs.size
        uv = np.stack([rng.uniform(0, 752, n), rng.uniform(0, 480, n)], 1).astype(np.float32)
        w = (1.0 / SCALE_FACTOR ** (2 * rng.integers(0, 8, n))).astype(np.float32)
        obs.append((kfs, np.full(n, nxt, np.int32), uv, w))
        pts.append(np.array([[rng.uniform(-0.5, 0.5), rng.uniform(-0.5, 0.5), rng.uniform(0.0, 0.4)]]).astype(np.float32).astype(np.float64))
        centre.append(np.array([kfs.mean()]))
        nxt += 1

    a = free_idx[30]
    for d in (43, 44, 47, 60):                        # co-observations at growing free-pose offsets
        add([a, free_idx[30 + d]])
    for _ in range(2):                                # more observations than a chunk of the landmark schedule
        add(np.sort(rng.choice(np.arange(20, 200), 170, replace=False)))
    for _ in range(4200):                             # one pair of keyframes sharing > 4096 landmarks, as two-observation landmarks
        add([free_idx[70], free_idx[71]])
    add([0, 13])                                      # seen only by fixed keyframes
    add([free_idx[120]])                              # seen once
    kf = np.concatenate([o[0] for o in obs]); mp = np.concatenate([o[1] for o in obs])
    uv = np.concatenate([o[2] for o in obs]); w = np.concatenate([o[3] for o in obs])
    points = np.concatenate(pts)
    # landmark numbering by mean observing keyframe, as a map's landmark order follows its trajectory
    order = np.argsort(np.concatenate(centre), kind="stable")
    relabel = np.empty_like(order); relabel[order] = np.arange(order.size)
    mp = relabel[mp].astype(np.int32); points = points[order]
    flags = np.zeros(kf.size, np.uint8)
    u = rng.random(kf.size)
    flags[u < 0.03] = 1                               # level 1: left out of the optimisation
    flags[(u >= 0.03) & (u < 0.3)] = 2                # no robust kernel
    perm = rng.permutation(kf.size)                   # not grouped by landmark
    p.fixed = fixed
    p.points = np.ascontiguousarray(points)
    p.obs_kf, p.obs_mp = np.ascontiguousarray(kf[perm]), np.ascontiguousarray(mp[perm])
    p.obs_uv, p.obs_w, p.edge_flags = np.ascontiguousarray(uv[perm]), np.ascontiguousarray(w[perm]), flags[perm]
    p.gt_points = None
    p.name = "awkward"
    return p


def make_config(name: str, **over) -> BAProblem:
    cfg = dict(CONFIGS[name]); cfg.update(over)
    kind = cfg.pop("kind")
    if kind == "local":
        return make_local_ba(name=name, **cfg)
    return make_global_ba(name=name, **cfg)


@dataclasses.dataclass
class PGOProblem:
    sim3: np.ndarray      # (K,8) qx qy qz qw tx ty tz s
    fixed: np.ndarray     # (K,) u8
    edge_i: np.ndarray    # (E,) i32
    edge_j: np.ndarray    # (E,) i32
    meas: np.ndarray      # (E,8) Sji
    fix_scale: bool = False
    gt: np.ndarray | None = None


def _sim3_mul(a, b):
    q = _quat_mul(a[..., :4], b[..., :4])
    t = a[..., 7:8] * _quat_rot(a[..., :4], b[..., 4:7]) + a[..., 4:7]
    return np.concatenate([q, t, a[..., 7:8] * b[..., 7:8]], -1)


def _sim3_inv(a):
    qc = a[..., :4] * np.array([-1, -1, -1, 1.0])
    t = _quat_rot(qc, (-1.0 / a[..., 7:8]) * a[..., 4:7])
    return np.concatenate([qc, t, 1.0 / a[..., 7:8]], -1)


def make_pgo(K=200, n_loop=6, n_covis=3, seed=5, drift=(0.002, 0.01, 0.002), fix_scale=False) -> PGOProblem:
    """Essential-graph-shaped Sim3 pose graph: spanning-tree chain + covisibility edges to the previous
    n_covis keyframes + a few loop edges (S/Optimizer.cpp:1389-1508).  Measurements are built like the
    reference does (Sji = Sjw * Swi from the *current*, drifted estimate) except for the loop edges which
    come from ground truth - that is what creates the error the optimisation distributes."""
    rng = np.random.default_rng(seed)
    Rcw, tcw, _, _ = _helix_cameras(K, rng, dtheta=2 * np.pi / K * 1.0, dz=0.0)
    q = _mat_to_quat(Rcw)
    gt = np.concatenate([q, tcw, np.ones((K, 1))], -1)
    # accumulate drift along the chain
    est = gt.copy()
    acc = np.array([0, 0, 0, 1.0, 0, 0, 0, 1.0])
    for k in range(1, K):
        d = np.concatenate([_rotvec_to_quat(rng.normal(size=3) * drift[0]), rng.normal(size=3) * drift[1],
                            [np.exp(rng.normal() * drift[2] * (0 if fix_scale else 1))]])
        acc = _sim3_mul(d, acc)
        est[k] = _sim3_mul(acc, gt[k])
    ei, ej, meas = [], [], []
    def add(i, j, src):
        ei.append(i); ej.append(j)
        meas.append(_sim3_mul(src[j], _sim3_inv(src[i])))
    for k in range(1, K):
        add(k, k - 1, est)
        for c in range(2, n_covis + 2):
            if k - c >= 0: add(k, k - c, est)
    for l in range(n_loop):
        i = K - 1 - l * 2
        j = l * 2
        add(i, j, gt)
    fixed = np.zeros(K, np.uint8); fixed[0] = 1
    return PGOProblem(sim3=est, fixed=fixed, edge_i=np.array(ei, np.int32), edge_j=np.array(ej, np.int32),
                      meas=np.ascontiguousarray(np.array(meas)), fix_scale=fix_scale, gt=gt)


# ---- single-vertex problems: PoseOptimizationClient (one frame against its map points), OptimizeSim3 (two keyframes) ----
def make_pose_opt(n=300, seed=11, outlier_frac=0.15, noise_px=0.8, pose_noise=(0.03, 0.08)):
    """One frame: n map points in front of a camera, pixel noise scaled by the octave, a share of gross outliers, and a
    perturbed initial pose.  Returns dict(Tcw0, Xw, uv, inv_sigma2, intr, Tcw_gt)."""
    rng = np.random.default_rng(seed)
    fx, fy, cx, cy = [np.float32(v) for v in EUROC_INTR]
    q_gt = _rotvec_to_quat(rng.standard_normal(3) * 0.3); t_gt = rng.standard_normal(3) * 0.5
    Xc = np.stack([rng.uniform(-2.0, 2.0, n), rng.uniform(-1.2, 1.2, n), rng.uniform(2.0, 8.0, n)], 1)
    qc = np.array([-q_gt[0], -q_gt[1], -q_gt[2], q_gt[3]])
    Xw = np.stack([_quat_rot(qc, x - t_gt) for x in Xc]).astype(np.float32)
    octave = rng.integers(0, 8, n)
    sigma = (1.2 ** octave)
    Xcf = np.stack([_quat_rot(q_gt, x.astype(np.float64)) + t_gt for x in Xw])
    uv = np.stack([fx * Xcf[:, 0] / Xcf[:, 2] + cx, fy * Xcf[:, 1] / Xcf[:, 2] + cy], 1) + rng.standard_normal((n, 2)) * noise_px * sigma[:, None]
    bad = rng.random(n) < outlier_frac
    uv[bad] += rng.uniform(-60, 60, (int(bad.sum()), 2))
    q0 = _quat_mul(_rotvec_to_quat(rng.standard_normal(3) * pose_noise[0]), q_gt)
    t0 = t_gt + rng.standard_normal(3) * pose_noise[1]
    return dict(Tcw0=np.concatenate([q0 / np.linalg.norm(q0), t0]), Xw=Xw, uv=uv.astype(np.float32),
                inv_sigma2=(1.0 / (sigma * sigma)).astype(np.float32), intr=(fx, fy, cx, cy), Tcw_gt=np.concatenate([q_gt, t_gt]))


def make_sim3_opt(n=120, seed=12, outlier_frac=0.2, noise_px=0.7, scale=1.15, fix_scale=False):
    """Two keyframes seeing the same n points, each with its own copy of the point in its own camera frame (map 2 is scaled
    against map 1).  Returns dict(S12_0, P1c, P2c, uv1, uv2, w1, w2, K1, K2, th2, fix_scale, S12_gt)."""
    rng = np.random.default_rng(seed)
    K = tuple(np.float32(v) for v in EUROC_INTR)
    s = 1.0 if fix_scale else scale
    q12 = _rotvec_to_quat(rng.standard_normal(3) * 0.2); t12 = rng.standard_normal(3) * 0.4
    P2c = np.stack([rng.uniform(-1.5, 1.5, n), rng.uniform(-1.0, 1.0, n), rng.uniform(2.5, 7.0, n)], 1)
    P1c = np.stack([s * _quat_rot(q12, x) + t12 for x in P2c])
    octave1, octave2 = rng.integers(0, 8, n), rng.integers(0, 8, n)
    s1, s2 = 1.2 ** octave1, 1.2 ** octave2
    proj = lambda P: np.stack([K[0] * P[:, 0] / P[:, 2] + K[2], K[1] * P[:, 1] / P[:, 2] + K[3]], 1)
    uv1 = proj(P1c) + rng.standard_normal((n, 2)) * noise_px * s1[:, None]
    uv2 = proj(P2c) + rng.standard_normal((n, 2)) * noise_px * s2[:, None]
    bad = rng.random(n) < outlier_frac
    uv1[bad] += rng.uniform(-40, 40, (int(bad.sum()), 2))
    P1c_n = P1c + rng.standard_normal((n, 3)) * 0.01; P2c_n = P2c + rng.standard_normal((n, 3)) * 0.01
    q0 = _quat_mul(_rotvec_to_quat(rng.standard_normal(3) * 0.02), q12)
    S0 = np.concatenate([q0 / np.linalg.norm(q0), t12 + rng.standard_normal(3) * 0.05, [s * (1.0 if fix_scale else 1.03)]])
    return dict(S12_0=S0, P1c=P1c_n.astype(np.float32), P2c=P2c_n.astype(np.float32), uv1=uv1.astype(np.float32), uv2=uv2.astype(np.float32),
                w1=(1.0 / (s1 * s1)).astype(np.float32), w2=(1.0 / (s2 * s2)).astype(np.float32), K1=K, K2=K, th2=np.float32(10.0),
                fix_scale=fix_scale, S12_gt=np.concatenate([q12, t12, [s]]))


def make_map_update(K=200, P=5000, seed=0, new_kf_frac=0.15, outside_frac=0.03, n_origins=2, chain=0.7):
    """A map as Map::RunGBA (S/Map.cpp:1441-1570) finds it when MapFusionGBA returns: a spanning forest over K keyframes rooted at
    n_origins origins (chain-like: with probability `chain` a keyframe hangs under its predecessor), f32 poses, a BA result for the
    keyframes that existed when the BA started and none for those added meanwhile (new_kf_frac, never an origin), a few keyframes
    outside the tree (outside_frac, some of them holding a BA result), points with and without a BA result, bad points, points
    without a reference keyframe."""
    rng = np.random.default_rng(seed)

    def se3(n, rot=0.6, trans=8.0):
        w = rng.normal(0, rot, (n, 3)); th = np.linalg.norm(w, axis=1, keepdims=True); k = w / np.maximum(th, 1e-12)
        Kx = np.zeros((n, 3, 3)); Kx[:, 0, 1] = -k[:, 2]; Kx[:, 0, 2] = k[:, 1]; Kx[:, 1, 0] = k[:, 2]; Kx[:, 1, 2] = -k[:, 0]; Kx[:, 2, 0] = -k[:, 1]; Kx[:, 2, 1] = k[:, 0]
        R = np.eye(3) + np.sin(th)[:, :, None] * Kx + (1 - np.cos(th))[:, :, None] * (Kx @ Kx)
        T = np.tile(np.eye(4), (n, 1, 1)); T[:, :3, :3] = R; T[:, :3, 3] = rng.normal(0, trans, (n, 3))
        return T
    parent = np.full(K, -2, np.int32)
    n_origins = min(n_origins, K)
    outside = np.zeros(K, bool)
    if K > n_origins:
        outside[n_origins:] = rng.random(K - n_origins) < outside_frac
    last_in = []
    for k in range(K):
        if k < n_origins:
            parent[k] = -1
        elif not outside[k]:
            parent[k] = last_in[-1] if rng.random() < chain else last_in[int(rng.integers(0, len(last_in)))]
        if not outside[k]:
            last_in.append(k)
    optimized = rng.random(K) >= new_kf_frac
    optimized[:n_origins] = True
    Tcw = se3(K).astype(np.float32)
    corr = se3(K, rot=0.02, trans=0.15)
    gba = (corr @ Tcw.astype(np.float64)).astype(np.float32)
    gba[~optimized] = np.float32(np.nan)                      # mTcwGBA is an empty Mat there; the update must never read it
    state = rng.choice(np.array([0, 1, 2], np.uint8), P, p=[0.05, 0.8, 0.15]) if P else np.zeros(0, np.uint8)
    ref = rng.integers(0, K, P).astype(np.int32) if K and P else np.full(P, -1, np.int32)
    if P:
        ref[rng.random(P) < 0.03] = -1
    pos = rng.normal(0, 12.0, (P, 3)).astype(np.float32)
    pos_gba = (pos + rng.normal(0, 0.05, (P, 3))).astype(np.float32)
    pos_gba[state != 1] = np.float32(np.nan)
    return dict(kf_parent=parent, kf_optimized=optimized.astype(np.uint8), kf_Tcw=Tcw, kf_TcwGBA=gba, mp_state=state, mp_ref=ref, mp_pos=pos,
                mp_pos_gba=pos_gba)


def scale_factors(n_levels=8, scale_factor=SCALE_FACTOR):
    """ORBextractor's mvScaleFactor (S/ORBextractor.cpp:584-590): f32, each level the previous one times the factor"""
    s = np.ones(n_levels, np.float32)
    for i in range(1, n_levels):
        s[i] = np.float32(s[i - 1] * np.float32(scale_factor))
    return s


def make_normal_depth(p: BAProblem | None = None, seed=0, K=60, P=2000, bad_kf_frac=0.05, bad_mp_frac=0.02, off_ref_frac=0.03,
                      all_bad_frac=0.0, on_centre_frac=0.0, map_order=False):
    """Inputs of ccm_normal_depth (MapPoint::UpdateNormalAndDepth over a batch, include/ccm_b200.h) for the map of a BA problem `p`
    (None: a random one of K keyframes and P points): keyframe centres -R^T t and bad flags, every point's observers in the problem's
    observation order, a reference keyframe among them (off_ref_frac: one that does not observe the point, whose keypoint 0 then
    gives the octave), scale factors of an 8-level pyramid.  Bad points (bad_mp_frac) are passed with no observers, as the shim passes
    them.  all_bad_frac: points whose observers are all bad keyframes (NaN normal); on_centre_frac: points moved onto an observer's centre.
    map_order: each point's observers unique and in ascending row, the order a std::map<kfptr> keeps when the keyframes lie in
    memory in row order (the stand-in scenes of the shim tests).
    Extra keys describe the scene behind the flat arrays: obs_octave, kf_oct0, mp_bad, ref_observes."""
    rng = np.random.default_rng(seed)
    if p is None:
        cen = rng.normal(0, 3.0, (K, 3)).astype(np.float32)
        deg = rng.integers(1, 9, P)
        obs_mp = np.repeat(np.arange(P, dtype=np.int32), deg)
        obs_kf = rng.integers(0, K, len(obs_mp)).astype(np.int32)
        pos = rng.normal(0, 8.0, (P, 3)).astype(np.float32)
    else:
        K, P = p.K, p.P
        q = p.poses[:, :4]; t = p.poses[:, 4:7]
        x, y, z, w = q[:, 0], q[:, 1], q[:, 2], q[:, 3]
        R = np.stack([1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w),
                      2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w),
                      2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)], 1).reshape(K, 3, 3)
        cen = (-np.einsum("kji,kj->ki", R, t)).astype(np.float32)
        order = np.argsort(p.obs_mp, kind="stable")
        obs_mp, obs_kf = p.obs_mp[order].astype(np.int32), p.obs_kf[order].astype(np.int32).copy()
        pos = p.points.astype(np.float32)
    if map_order:
        pair = np.unique(obs_mp.astype(np.int64) * K + obs_kf)
        obs_mp, obs_kf = (pair // K).astype(np.int32), (pair % K).astype(np.int32)
    deg = np.bincount(obs_mp, minlength=P)
    ptr = np.zeros(P + 1, np.int64); ptr[1:] = np.cumsum(deg)
    kf_bad = (rng.random(K) < bad_kf_frac).astype(np.uint8)
    mp_bad = rng.random(P) < bad_mp_frac
    obs_octave = rng.choice(8, len(obs_kf), p=OCTAVE_QUOTAS / OCTAVE_QUOTAS.sum()).astype(np.int32)
    kf_oct0 = rng.integers(0, 8, K).astype(np.int32)
    bad_rows = np.flatnonzero(kf_bad)
    if len(bad_rows):
        for i in np.flatnonzero((rng.random(P) < all_bad_frac) & (deg > 0) & (deg <= len(bad_rows))):
            pick = rng.choice(bad_rows, deg[i], replace=False)
            obs_kf[ptr[i]:ptr[i + 1]] = np.sort(pick) if map_order else pick
    sf = scale_factors()
    ref = np.full(P, -1, np.int32); ref_observes = np.zeros(P, bool); sref = np.ones(P, np.float32)
    for i in np.flatnonzero(deg > 0):
        b, e = ptr[i], ptr[i + 1]
        if rng.random() < off_ref_frac:
            ref[i] = rng.integers(0, K)
        else:
            ref[i] = obs_kf[rng.integers(b, e)]
        hit = np.flatnonzero(obs_kf[b:e] == ref[i])
        ref_observes[i] = len(hit) > 0
        sref[i] = sf[obs_octave[b + hit[0]]] if len(hit) else sf[kf_oct0[ref[i]]]
    for i in np.flatnonzero((rng.random(P) < on_centre_frac) & (deg > 0)):
        pos[i] = cen[obs_kf[ptr[i]]]
    keep = np.repeat(~mp_bad, deg)                              # a bad point goes in with no observers
    dk = np.where(mp_bad, 0, deg)
    fptr = np.zeros(P + 1, np.int64); fptr[1:] = np.cumsum(dk)
    return dict(kf_centre=cen, kf_bad=kf_bad, mp_pos=pos, obs_ptr=fptr, obs_kf=obs_kf[keep], mp_ref=ref, mp_scale_ref=sref,
                mp_scale_last=np.full(P, sf[-1], np.float32), obs_octave=obs_octave[keep], kf_oct0=kf_oct0, mp_bad=mp_bad,
                ref_observes=ref_observes)


def make_distinctive(p: BAProblem | None = None, seed=0, K=60, P=2000, max_deg=8, bad_kf_frac=0.05, bad_mp_frac=0.0, all_bad_frac=0.0,
                     empty_frac=0.0, forced_n=(), extra_feat=8, map_order=False):
    """Inputs of ccm_distinctive_descriptors (MapPoint::ComputeDistinctiveDescriptors over a batch, include/ccm_b200.h) for the
    observation lists of a BA problem `p` (None: a random map of K keyframes and P points, 1..max_deg observers each).
    Every point has a "true" 32-byte descriptor; each observation of it is that descriptor with random bit flips at a per-point rate
    (none, 1/128 .. 1/8), so rows repeat and medians tie often.  Each keyframe holds its observed features, at shuffled indices, plus
    up to extra_feat unobserved ones.  bad_kf_frac: bad keyframes (skipped observers); all_bad_frac: points whose observers are all
    bad; empty_frac: points with no observers; bad_mp_frac: bad points, passed with no observers as the shim passes them; forced_n:
    extra points appended at the end, one per value, with exactly that many observers, all of keyframes that are not bad.
    map_order: each point's observers unique and in ascending row (the order std::map<kfptr> keeps for the stand-in scenes).
    Returns kf_bad, kf_uid (u64), kf_nfeat, kf_desc_ptr (K+1), kf_desc (sum nfeat, 32), obs_ptr, obs_kf, obs_feat, obs_desc (E, 32),
    mp_bad."""
    rng = np.random.default_rng(seed)
    if p is None:
        deg = rng.integers(1, max_deg + 1, P)
        obs_mp = np.repeat(np.arange(P, dtype=np.int64), deg)
        obs_kf = rng.integers(0, K, len(obs_mp)).astype(np.int64)
    else:
        K, P = p.K, p.P
        order = np.argsort(p.obs_mp, kind="stable")
        obs_mp, obs_kf = p.obs_mp[order].astype(np.int64), p.obs_kf[order].astype(np.int64)
    if map_order:
        pair = np.unique(obs_mp * K + obs_kf)
        obs_mp, obs_kf = pair // K, pair % K
    kf_bad = (rng.random(K) < bad_kf_frac).astype(np.uint8)
    good = np.flatnonzero(kf_bad == 0)
    if len(forced_n):
        add_mp, add_kf = [], []
        for t, n in enumerate(forced_n):
            pick = rng.choice(good, n, replace=n > len(good) and not map_order)
            add_mp.append(np.full(n, P + t, np.int64)); add_kf.append(np.sort(pick) if map_order else pick)
        obs_mp = np.concatenate([obs_mp] + add_mp); obs_kf = np.concatenate([obs_kf] + add_kf)
        P += len(forced_n)
    n_forced = len(forced_n)
    free = np.arange(P) < P - n_forced
    empty = free & (rng.random(P) < empty_frac)
    obs_keep = ~empty[obs_mp]
    obs_mp, obs_kf = obs_mp[obs_keep], obs_kf[obs_keep]
    deg = np.bincount(obs_mp, minlength=P)
    ptr = np.zeros(P + 1, np.int64); ptr[1:] = np.cumsum(deg)
    bad_rows = np.flatnonzero(kf_bad)
    if len(bad_rows):
        for i in np.flatnonzero(free & (rng.random(P) < all_bad_frac) & (deg > 0) & (deg <= len(bad_rows))):
            pick = rng.choice(bad_rows, deg[i], replace=False)
            obs_kf[ptr[i]:ptr[i + 1]] = np.sort(pick) if map_order else pick
    mp_bad = free & (rng.random(P) < bad_mp_frac)
    keep = np.repeat(~mp_bad, deg)                              # a bad point goes in with no observers
    obs_mp, obs_kf = obs_mp[keep], obs_kf[keep]
    deg = np.where(mp_bad, 0, deg)
    ptr = np.zeros(P + 1, np.int64); ptr[1:] = np.cumsum(deg)
    E = len(obs_kf)
    # descriptors: truth xor a mask whose bits are set with probability 2^-m (m per point; m = 0: an exact copy)
    truth = rng.integers(0, 256, (P, 32), dtype=np.uint8)
    m_pt = rng.choice(np.array([0, 3, 4, 5, 6, 7]), P)
    obs_desc = np.empty((E, 32), np.uint8)
    for c0 in range(0, E, 1 << 20):
        c1 = min(E, c0 + (1 << 20))
        m = m_pt[obs_mp[c0:c1]][:, None]
        mask = np.where(m > 0, np.uint8(255), np.uint8(0)) * np.ones((1, 32), np.uint8)
        for r in range(7):
            mask &= np.where(r < m, rng.integers(0, 256, (c1 - c0, 32), dtype=np.uint8), np.uint8(255))
        obs_desc[c0:c1] = truth[obs_mp[c0:c1]] ^ mask
    # features: each keyframe's observations at shuffled indices, then unobserved features
    order = np.lexsort((rng.random(E), obs_kf))
    per_kf = np.bincount(obs_kf, minlength=K)
    start = np.zeros(K + 1, np.int64); start[1:] = np.cumsum(per_kf)
    obs_feat = np.empty(E, np.int64)
    obs_feat[order] = np.arange(E) - start[obs_kf[order]]
    nfeat = per_kf + rng.integers(0, extra_feat + 1, K)
    kptr = np.zeros(K + 1, np.int64); kptr[1:] = np.cumsum(nfeat)
    kf_desc = rng.integers(0, 256, (int(kptr[-1]), 32), dtype=np.uint8)
    kf_desc[kptr[obs_kf] + obs_feat] = obs_desc
    kf_uid = (np.uint64(3) << np.uint64(40)) + np.arange(K, dtype=np.uint64) * np.uint64(7) + np.uint64(11)
    return dict(kf_bad=kf_bad, kf_uid=kf_uid, kf_nfeat=nfeat.astype(np.int32), kf_desc_ptr=kptr, kf_desc=kf_desc, obs_ptr=ptr,
                obs_kf=obs_kf.astype(np.int32), obs_feat=obs_feat.astype(np.int32), obs_desc=obs_desc, mp_bad=mp_bad)


def covis_pack(K, pair_kf, pair_mp, P, rng, kf_id=None, kf_rank=None, null_frac=0.0, dup_frac=0.0, bad_mp_frac=0.0, bad_kf_frac=0.0,
               extra=None, batch=None):
    """The arrays of a covisibility scene (synth.make_covisibility) from (keyframe, point) observation pairs, made unique.  Each
    keyframe's mvpMapPoints holds its points at shuffled indices, with null_frac nulls and dup_frac of its points at a second index;
    extra: (kf, mp) entries appended to mvpMapPoints without an observation (a point the keyframe lists but that does not list it)."""
    key = np.unique(np.asarray(pair_kf, np.int64) * max(P, 1) + np.asarray(pair_mp, np.int64))
    pk, pm = key // max(P, 1), key % max(P, 1)
    kf_id = np.arange(K, dtype=np.uint64) if kf_id is None else np.asarray(kf_id, np.uint64)
    kf_rank = rng.permutation(K).astype(np.uint32) if kf_rank is None else np.asarray(kf_rank, np.uint32)
    ek, em = [pk], [pm]
    if null_frac > 0:
        n = rng.binomial(np.bincount(pk, minlength=K), null_frac)
        ek.append(np.repeat(np.arange(K), n)); em.append(np.full(int(n.sum()), -1, np.int64))
    if dup_frac > 0:
        d = np.flatnonzero(rng.random(len(pk)) < dup_frac)
        ek.append(pk[d]); em.append(pm[d])
    if extra is not None:
        ek.append(np.asarray(extra[0], np.int64)); em.append(np.asarray(extra[1], np.int64))
    ek, em = np.concatenate(ek), np.concatenate(em)
    o = np.lexsort((rng.random(len(ek)), ek))
    ek, em = ek[o], em[o]
    mvp_ptr = np.zeros(K + 1, np.int64); mvp_ptr[1:] = np.cumsum(np.bincount(ek, minlength=K))
    # observers of each point in ascending rank (std::map<kfptr,size_t>'s order), idx = the point's first index in the keyframe
    o = np.lexsort((kf_rank[pk], pm))
    obs_mp, obs_kf = pm[o], pk[o]
    obs_ptr = np.zeros(P + 1, np.int64); obs_ptr[1:] = np.cumsum(np.bincount(obs_mp, minlength=P))
    pos = np.arange(len(ek)) - mvp_ptr[ek]
    live = em >= 0
    ekey = ek[live] * max(P, 1) + em[live]
    first = np.lexsort((pos[live], ekey))
    ukey, at = np.unique(ekey[first], return_index=True)
    okey = obs_kf * max(P, 1) + obs_mp
    obs_idx = pos[live][first][at][np.searchsorted(ukey, okey)] if len(okey) else np.zeros(0, np.int64)
    return dict(kf_id=kf_id, kf_rank=kf_rank, kf_bad=(rng.random(K) < bad_kf_frac).astype(np.uint8), mvp_ptr=mvp_ptr,
                mvp=em.astype(np.int32), mp_bad=(rng.random(P) < bad_mp_frac).astype(np.uint8), obs_ptr=obs_ptr,
                obs_kf=obs_kf.astype(np.int32), obs_idx=obs_idx.astype(np.int32),
                batch=np.arange(K, dtype=np.int32) if batch is None else np.asarray(batch, np.int32))


def make_covisibility(p: BAProblem | None = None, seed=0, K=60, P=2000, max_deg=8, window=None, n_maps=1, null_frac=0.05, dup_frac=0.01,
                      bad_mp_frac=0.03, bad_kf_frac=0.05, same_id_frac=0.0, hub=0, batch_frac=1.0):
    """Inputs of ccm_covisibility (KeyFrame::UpdateConnections over a batch, include/ccm_b200.h) for the observation lists of a BA
    problem `p` (None: K keyframes and P points, 1..max_deg observers each, drawn from a window of `window` consecutive rows when
    given, so that weights spread around the threshold).  Keyframe ids: n_maps maps of consecutive rows, mId = (index in its map, map)
    packed as map << 32 | index; same_id_frac of the rows take the mId of another row of their map (the self test compares mId, not
    the row).  Address ranks are a random permutation.  hub > 0: row 0 is co-observed with every one of `hub` other keyframes
    (K grows to hub + 1 if needed) through extra points, two to six observers each.  batch_frac < 1: a random subset of rows.
    Returns kf_id (u64), kf_rank (u32), kf_bad, mvp_ptr (K+1), mvp (-1 null), mp_bad, obs_ptr, obs_kf, obs_idx, batch."""
    rng = np.random.default_rng(seed)
    if p is None:
        if hub:
            K = max(K, hub + 1)
        deg = rng.integers(1, max_deg + 1, P)
        mp = np.repeat(np.arange(P, dtype=np.int64), deg)
        if window:
            start = rng.integers(0, max(K - window, 1), P)
            kf = np.repeat(start, deg) + rng.integers(0, min(window, K), len(mp))
        else:
            kf = rng.integers(0, K, len(mp))
    else:
        K, P = p.K, p.P
        kf, mp = p.obs_kf.astype(np.int64), p.obs_mp.astype(np.int64)
    if hub:
        n_hub = (hub + 1) // 2
        hp = P + np.arange(n_hub)
        others = 1 + (np.arange(2 * n_hub) % hub)
        extra_n = rng.integers(0, 5, n_hub)
        kf = np.concatenate([kf, np.zeros(n_hub, np.int64), others, rng.integers(1, K, int(extra_n.sum()))])
        mp = np.concatenate([mp, hp, np.repeat(hp, 2), np.repeat(hp, extra_n)])
        P += n_hub
    per_map = -(-K // n_maps)
    m, first = np.arange(K) // per_map, np.arange(K) % per_map
    same = np.flatnonzero((rng.random(K) < same_id_frac) & (first > 1))
    first[same] = first[same] - 1                                       # the mId of the row before it
    kf_id = (m.astype(np.uint64) << np.uint64(32)) | first.astype(np.uint64)
    batch = np.arange(K) if batch_frac >= 1 else np.sort(rng.choice(K, max(1, int(K * batch_frac)), replace=False))
    return covis_pack(K, kf, mp, P, rng, kf_id=kf_id, null_frac=null_frac, dup_frac=dup_frac, bad_mp_frac=bad_mp_frac,
                      bad_kf_frac=bad_kf_frac, batch=batch)


def _eigen_quat(R):
    """Eigen's Quaterniond(Matrix3d) (vectorised, f64): the branches of ba_math.cuh's R_to_quat, no normalisation, as
    g2o::Sim3(R, t, s) keeps it.  R (n,3,3) -> (n,4) qx qy qz qw"""
    R = np.asarray(R, np.float64).reshape(-1, 3, 3)
    q = np.zeros((len(R), 4))
    for i in range(len(R)):
        m = R[i]
        t = m[0, 0] + m[1, 1] + m[2, 2]
        if t > 0:
            t = np.sqrt(t + 1.0); w = 0.5 * t; t = 0.5 / t
            q[i] = [(m[2, 1] - m[1, 2]) * t, (m[0, 2] - m[2, 0]) * t, (m[1, 0] - m[0, 1]) * t, w]
        else:
            a = 0 if (m[0, 0] >= m[1, 1] and m[0, 0] >= m[2, 2]) else (1 if m[1, 1] >= m[2, 2] else 2)
            b, c = (a + 1) % 3, (a + 2) % 3
            t = np.sqrt(m[a, a] - m[b, b] - m[c, c] + 1.0)
            v = np.zeros(3); v[a] = 0.5 * t; t = 0.5 / t
            w = (m[c, b] - m[b, c]) * t; v[b] = (m[b, a] + m[a, b]) * t; v[c] = (m[c, a] + m[a, c]) * t
            q[i] = [v[0], v[1], v[2], w]
    return q


def _f32_gemm4(A, B):
    """A @ B for f32 4x4 stacks, each element summed left to right in f32 (cv::gemm's small-matrix path)"""
    A = np.asarray(A, np.float32); B = np.asarray(B, np.float32)
    C = A[..., :, 0:1] * B[..., 0:1, :]
    for k in range(1, 4):
        C = (C + A[..., :, k:k + 1] * B[..., k:k + 1, :]).astype(np.float32)
    return C


def _f32_pose_inverse(T):
    """KeyFrame::SetPose's Twc from f32 Tcw stacks: [R^T | -(R^T t)], the product summed left to right in f32"""
    T = np.asarray(T, np.float32)
    R, t = T[..., :3, :3], T[..., :3, 3]
    ow = R[..., 0, :] * t[..., 0:1]
    ow = (ow + R[..., 1, :] * t[..., 1:2]).astype(np.float32)
    ow = (ow + R[..., 2, :] * t[..., 2:3]).astype(np.float32)
    W = np.zeros(T.shape, np.float32)
    W[..., :3, :3] = np.swapaxes(R, -1, -2); W[..., :3, 3] = -ow; W[..., 3, 3] = 1
    return W


def make_sim3_correction(p: BAProblem | None = None, kind="loop", seed=0, K=60, P=2000, max_deg=8, window=12, n_loop=30, null_frac=0.05,
                         dup_frac=0.02, bad_mp_frac=0.03, tagged_frac=0.03, bad_kf_frac=0.05, all_bad_frac=0.0, off_ref_frac=0.05,
                         no_ref_frac=0.0, empty_frac=0.0, null_entry_frac=0.0, unlisted_frac=0.0, scale=1.07):
    """Inputs of ccm_sim3_correction (the Sim3 pass of LoopFinder::CorrectLoop / MapMerger::MergeMaps, include/ccm_b200.h) over the map
    of a BA problem `p` (None: K keyframes and P points, 1..max_deg observers each drawn from a window of `window` consecutive rows).
    f32 poses and centres as SetPose leaves them; mvpMapPoints and observer lists from covis_pack (null slots, a point at two slots, bad
    points and keyframes); address ranks a random permutation, so the entries' map order differs from their row order.
    kind="merge": every keyframe is an entry (CorrectedSim3All); kind="loop": a current keyframe and its n_loop most covisible
    keyframes (CorrectedSim3), so observers and reference keyframes fall before, after, on and outside the entries.
    Corrected Sim3s as the sites build them: the current keyframe's Scw = (drift correction with scale `scale`) * Sim3(Tcw, 1);
    for the others Sic = Sim3(R, t, 1) of the f32 product Tiw*Twc and CorrectedSiw = Sic * Scw; NonCorrectedSim3 = Sim3(Riw, tiw, 1).
    Knobs: tagged_frac (points already tagged with the current mId, passed as skipped), all_bad_frac (points whose observers are all bad),
    off_ref_frac (mpRefKF any keyframe), no_ref_frac (no mpRefKF), empty_frac (entries with no slots), null_entry_frac (entries whose
    slots are all null), unlisted_frac (slots turned null while the point keeps the observation: an entry that observes a point
    without listing it, so that observers fall before the claiming entry).  Extra keys: kf_Tcw (K,4,4) f32, kf_rank, mp_bad, mp_tagged, cur (row of the current keyframe)."""
    rng = np.random.default_rng(seed)
    if p is None:
        Rcw, tcw, C, zc = _helix_cameras(K, rng, radius=6.0, dtheta=0.05, dz=0.01)
        Tcw = np.tile(np.eye(4), (K, 1, 1)); Tcw[:, :3, :3] = Rcw; Tcw[:, :3, 3] = tcw
        deg = rng.integers(1, max_deg + 1, P)
        mp = np.repeat(np.arange(P, dtype=np.int64), deg)
        start = rng.integers(0, max(K - window, 1), P)
        kf = np.repeat(start, deg) + rng.integers(0, min(window, K), len(mp))
        base = np.clip(start + min(window, K) // 2, 0, K - 1)
        pos = C[base] + zc[base] * rng.uniform(2.0, 8.0, (P, 1)) + rng.normal(0, 1.0, (P, 3))
    else:
        K, P = p.K, p.P
        q = p.poses[:, :4]; x, y, z, w = q[:, 0], q[:, 1], q[:, 2], q[:, 3]
        R = np.stack([1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w),
                      2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w),
                      2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)], 1).reshape(K, 3, 3)
        Tcw = np.tile(np.eye(4), (K, 1, 1)); Tcw[:, :3, :3] = R; Tcw[:, :3, 3] = p.poses[:, 4:7]
        kf, mp = p.obs_kf.astype(np.int64), p.obs_mp.astype(np.int64)
        pos = p.points
    Tcw = Tcw.astype(np.float32)
    cen = _f32_pose_inverse(Tcw)[:, :3, 3].copy()
    pk = covis_pack(K, kf, mp, P, rng, null_frac=null_frac, dup_frac=dup_frac, bad_mp_frac=bad_mp_frac, bad_kf_frac=bad_kf_frac)
    rank = pk["kf_rank"].astype(np.int64)
    obs_ptr, obs_kf = pk["obs_ptr"], pk["obs_kf"].copy()
    deg = np.diff(obs_ptr)
    kf_bad = pk["kf_bad"]
    cur = int(rng.integers(0, K))
    if kind == "merge":
        rows = np.arange(K)
    elif kind == "loop":
        # the current keyframe and its most covisible keyframes (shared points)
        mine = pk["mvp"][pk["mvp_ptr"][cur]:pk["mvp_ptr"][cur + 1]]
        mine = np.unique(mine[mine >= 0])
        sel = np.concatenate([obs_kf[obs_ptr[i]:obs_ptr[i + 1]] for i in mine]) if len(mine) else np.zeros(0, np.int64)
        cnt = np.bincount(sel, minlength=K); cnt[cur] = 0
        nb = np.argsort(-cnt, kind="stable")[:n_loop]
        rows = np.concatenate([[cur], nb[cnt[nb] > 0]])
    else:
        raise ValueError(kind)
    entry_kf = rows[np.argsort(rank[rows], kind="stable")].astype(np.int32)     # std::map<kfptr> order
    E = len(entry_kf)
    # corrected Sim3s as the sites build them
    corr_q = _rotvec_to_quat(rng.normal(0, 0.05, 3)); corr_q = corr_q / np.linalg.norm(corr_q)
    S_corr = np.concatenate([corr_q, rng.normal(0, 0.3, 3), [scale]])
    Tc = Tcw[cur].astype(np.float64)
    S_cur = np.concatenate([_eigen_quat(Tc[:3, :3])[0], Tc[:3, 3], [1.0]])
    Scw = _sim3_mul(S_corr, S_cur)
    Twc = _f32_pose_inverse(Tcw[cur])
    Tic = _f32_gemm4(Tcw[entry_kf], Twc)
    Sic = np.concatenate([_eigen_quat(Tic[:, :3, :3].astype(np.float64)), Tic[:, :3, 3].astype(np.float64), np.ones((E, 1))], 1)
    Siw_new = np.array([Scw if k == cur else _sim3_mul(Sic[e], Scw) for e, k in enumerate(entry_kf)]).reshape(E, 8)
    Siw_old = np.concatenate([_eigen_quat(Tcw[entry_kf, :3, :3].astype(np.float64)), Tcw[entry_kf, :3, 3].astype(np.float64),
                              np.ones((E, 1))], 1)
    # slots: each entry's mvpMapPoints
    mptr, mvp = pk["mvp_ptr"], pk["mvp"]
    lists = [mvp[mptr[k]:mptr[k + 1]].copy() for k in entry_kf]
    for e in range(E):
        lists[e][rng.random(len(lists[e])) < unlisted_frac] = -1
        u = rng.random()
        if u < empty_frac:
            lists[e] = lists[e][:0]
        elif u < empty_frac + null_entry_frac:
            lists[e][:] = -1
    slot_ptr = np.zeros(E + 1, np.int64); slot_ptr[1:] = np.cumsum([len(s) for s in lists])
    slot_mp = np.concatenate(lists).astype(np.int32) if E else np.zeros(0, np.int32)
    # points
    mp_bad = pk["mp_bad"].astype(bool)
    tagged = rng.random(P) < tagged_frac
    bad_rows = np.flatnonzero(kf_bad)
    if len(bad_rows):
        for i in np.flatnonzero((rng.random(P) < all_bad_frac) & (deg > 0) & (deg <= len(bad_rows))):
            pick = rng.choice(bad_rows, deg[i], replace=False)
            obs_kf[obs_ptr[i]:obs_ptr[i + 1]] = pick[np.argsort(rank[pick])]
    sf = scale_factors()
    ref = np.full(P, -1, np.int32)
    has = deg > 0
    pick = obs_ptr[:-1] + (rng.random(P) * np.maximum(deg, 1)).astype(np.int64)
    ref[has] = obs_kf[pick[has]]
    off = has & (rng.random(P) < off_ref_frac)
    ref[off] = rng.integers(0, K, int(off.sum()))
    ref[rng.random(P) < no_ref_frac] = -1
    sref = sf[rng.choice(8, P, p=OCTAVE_QUOTAS / OCTAVE_QUOTAS.sum())].astype(np.float32)
    return dict(kf_centre=cen.astype(np.float32), kf_bad=kf_bad.astype(np.uint8), entry_kf=entry_kf, entry_Siw_new=Siw_new,
                entry_Siw_old=Siw_old, slot_ptr=slot_ptr, slot_mp=slot_mp, mp_pos=np.asarray(pos, np.float32),
                mp_skip=(mp_bad | tagged).astype(np.uint8), obs_ptr=obs_ptr, obs_kf=obs_kf.astype(np.int32), mp_ref=ref,
                mp_scale_ref=sref, mp_scale_last=np.full(P, sf[-1], np.float32), kf_Tcw=Tcw, kf_rank=pk["kf_rank"], mp_bad=mp_bad,
                mp_tagged=tagged, cur=cur)


class _KcMap:
    """A small mutable map for make_keyframe_culling_scene: keyframes with slots (point row or -1, keypoint octave), points with
    observers (keyframe row, slot index) in mObservations order, nObs and mpRefKF."""

    def __init__(self):
        self.kf_bad, self.kf_not_erase, self.kf_id, self.slots = [], [], [], []
        self.mp_bad, self.mp_nobs, self.mp_ref, self.obs = [], [], [], []

    def kf(self, bad=0, not_erase=0, id=None):
        self.kf_bad.append(bad); self.kf_not_erase.append(not_erase); self.slots.append([])
        self.kf_id.append(len(self.kf_id) + 2 if id is None else id)
        return len(self.kf_bad) - 1

    def pt(self, observers, nobs=None, ref=0, bad=0):
        """observers: (keyframe row, octave) each, in mObservations order; each gets a slot that holds the point.  ref: position in
        observers of mpRefKF, or None for a null mpRefKF"""
        p = len(self.mp_bad)
        o = []
        for k, octave in observers:
            o.append((k, len(self.slots[k])))
            self.slots[k].append((p, int(octave)))
        self.obs.append(o)
        self.mp_bad.append(bad)
        self.mp_nobs.append(len(o) if nobs is None else nobs)
        self.mp_ref.append(-1 if ref is None or not o else o[ref][0])
        return p

    def slot(self, k, p, octave):
        """a slot of keyframe k that holds point p (or -1) without an observation of it"""
        self.slots[k].append((p, int(octave)))

    def redundant_points(self, k, n, observers, octave=0):
        """n points in k's slots, each seen by k at `octave` and by every keyframe of `observers` at octave 0"""
        return [self.pt([(k, octave)] + [(g, 0) for g in observers]) for _ in range(n)]

    def arrays(self):
        ids = np.asarray(self.kf_id, np.int64)
        K, P = len(self.kf_bad), len(self.mp_bad)
        obs = [sorted(o, key=lambda e: ids[e[0]]) if not self.mp_bad[p] else [] for p, o in enumerate(self.obs)]   # a bad point has none
        sptr = np.zeros(K + 1, np.int64); sptr[1:] = np.cumsum([len(s) for s in self.slots])
        smp = np.asarray([s[0] for row in self.slots for s in row], np.int32).reshape(-1)
        soct = np.asarray([s[1] for row in self.slots for s in row], np.int32).reshape(-1)
        optr = np.zeros(P + 1, np.int64); optr[1:] = np.cumsum([len(o) for o in obs])
        okf = np.asarray([e[0] for o in obs for e in o], np.int32).reshape(-1)
        oidx = np.asarray([e[1] for o in obs for e in o], np.int32).reshape(-1)
        return dict(kf_bad=np.asarray(self.kf_bad, np.uint8), kf_not_erase=np.asarray(self.kf_not_erase, np.uint8), kf_id=ids.astype(np.int64),
                    kf_slot_ptr=sptr, kf_slot_mp=smp, kf_slot_octave=soct, mp_bad=np.asarray(self.mp_bad, np.uint8).reshape(P),
                    mp_nobs=np.asarray(self.mp_nobs, np.int32).reshape(P), mp_ref=np.asarray(self.mp_ref, np.int32).reshape(P),
                    obs_ptr=optr, obs_kf=okf, obs_idx=oidx, obs_octave=soct[sptr[okf] + oidx] if len(okf) else np.zeros(0, np.int32))


def keyframe_culling_candidates(sc):
    """The flat candidate arrays of ccm_keyframe_culling for a map scene: the query's covisible keyframes, in order, without mId.first 0
    or 1 and without the recently added ones (Mapping.cpp:799-805), each with its slots."""
    recent = set(int(k) for k in sc["recent"])
    cand = np.asarray([k for k in sc["covis"] if sc["kf_id"][k] not in (0, 1) and int(k) not in recent], np.int32)
    sptr = sc["kf_slot_ptr"]
    n = sptr[cand + 1] - sptr[cand]
    ptr = np.zeros(len(cand) + 1, np.int64); ptr[1:] = np.cumsum(n)
    idx = (np.repeat(sptr[cand] - ptr[:-1], n) + np.arange(ptr[-1])).astype(np.int64)
    return dict(cand_kf=cand, cand_not_erase=sc["kf_not_erase"][cand], slot_ptr=ptr, slot_mp=sc["kf_slot_mp"][idx],
                slot_octave=sc["kf_slot_octave"][idx])


def make_keyframe_culling_scene(n_c=20, slots=1000, obs=(5, 20), seed=0, n_redundant=2, fresh_frac=0.1, null_frac=0.03, dup_frac=0.01,
                                bad_mp_frac=0.02, bad_kf_frac=0.03, no_ref_frac=0.002, edges=True, red_thres=0.98, split=None):
    """Inputs of ccm_keyframe_culling (the redundancy test of LocalMapping::KeyFrameCullingV3, include/ccm_b200.h) as a whole map:
    keyframe rows with mvpMapPoints slots and keypoint octaves, points with observers, nObs and mpRefKF; the picked keyframe `query`,
    its covisible list `covis` (rows 0 and 1 have mId.first 0 and 1) and mlpRecentAddedKFs `recent`; and the flat candidate arrays
    (keyframe_culling_candidates).

    Server-shaped part: n_c candidates of about `slots` slots each, points with obs[0]..obs[1] observers among the candidates and
    n_c // 2 + 8 other keyframes, octaves drawn by the ORB level quotas; fresh_frac of each slot list holds points with two or three
    observers (so an ordinary candidate stays below 0.98), null slots, a point at two slots, bad points and bad observers, points with
    no mpRefKF.  n_redundant candidates see every point at octave 7 and are culled; their culls reach later candidates.

    edges=True adds, each on its own keyframes: the 0.98 ties at nMPs 50 and 100; a point with Observations() == 3 and three other
    observers; observers at octave level + 1 and level + 2; a point whose other counted observer is only the candidate itself; nMPs ==
    0; a redundant candidate with mbNotErase and an already bad one; and three cascades (a cull drops a point to nObs <= 2 and turns a
    later verdict to cull; a cull was mpRefKF of a point whose observers left are all bad, which changes an already bad candidate's
    counts; a cull reaches points with no mpRefKF, one it does not observe).  split=(n, k): one candidate with n points of which k are
    redundant, for the threshold test, and no other part."""
    rng = np.random.default_rng(seed)
    m = _KcMap()
    order = []   # the candidates in covisibility order, built as a list of groups that keep their internal order
    m.kf(id=0); m.kf(id=1)
    query = m.kf()
    recent = [m.kf(), m.kf()]
    if split is not None:
        n, k = split
        c = m.kf()
        g = [m.kf() for _ in range(4)]
        m.redundant_points(c, k, g)
        for _ in range(n - k):
            m.pt([(c, 0), (g[0], 0), (g[1], 0)])
        order.append([c])
        n_c = 0
    cands = [m.kf(bad=int(rng.random() < 0.05)) for _ in range(n_c)]
    extras = [m.kf(bad=int(rng.random() < bad_kf_frac)) for _ in range(n_c // 2 + 8)]
    if n_c:
        designed = set(int(c) for c in rng.choice(cands, min(n_redundant, n_c), replace=False)) if n_redundant else set()
        for c in designed:
            m.kf_bad[c] = 0
        pool = np.asarray(cands + extras + recent + [0, 1])
        plain = np.asarray([k for k in pool if k not in designed])
        q = OCTAVE_QUOTAS / OCTAVE_QUOTAS.sum()
        avg = (obs[0] + obs[1]) / 2.0
        P = int(slots * len(pool) * (1 - fresh_frac) / avg)
        for _ in range(P):
            d = min(int(rng.integers(obs[0], obs[1] + 1)), len(pool))
            who = rng.choice(pool, d, replace=False)
            octs = rng.choice(8, d, p=q)
            octs[np.isin(who, list(designed))] = 7
            m.pt(list(zip(who.tolist(), octs.tolist())), ref=int(rng.integers(d)) if rng.random() >= no_ref_frac else None,
                 bad=int(rng.random() < bad_mp_frac))
        for _ in range(int(slots * len(plain) * fresh_frac / 2.5)):
            d = int(rng.integers(2, 4))
            who = rng.choice(plain, d, replace=False)
            m.pt(list(zip(who.tolist(), rng.choice(8, d, p=q).tolist())), ref=int(rng.integers(d)))
        for c in cands:
            held = [s[0] for s in m.slots[c] if s[0] >= 0]
            for _ in range(int(len(held) * null_frac)):
                m.slot(c, -1, int(rng.integers(8)))
            for p in rng.choice(held, int(len(held) * dup_frac), replace=False) if held else []:
                m.slot(c, int(p), 7 if c in designed else int(rng.integers(8)))
        order += [[c] for c in cands]
    if edges:
        def good(n):
            return [m.kf() for _ in range(n)]
        for n in (50, 100):                                       # ties: nRedundant == 0.98 * nMPs exactly
            c, g = m.kf(), good(4)
            m.redundant_points(c, n - n // 50, g)
            for _ in range(n // 50):
                m.pt([(c, 0), (g[0], 0), (g[1], 0), (m.kf(bad=1), 0)])   # nObs 4, two counted others: the candidate itself is not one
            order.append([c])
        c, g = m.kf(), good(4)                                    # Observations() == 3 with three other observers: not redundant
        m.redundant_points(c, 49, g)
        m.slot(c, m.pt([(g[0], 0), (g[1], 0), (g[2], 0)]), 0)
        order.append([c])
        c, g = m.kf(), good(4)                                    # observers at level + 1 count (a cull) ...
        for _ in range(50):
            m.pt([(c, 2)] + [(x, 3) for x in g])
        order.append([c])
        c, g = m.kf(), good(4)                                    # ... at level + 2 they do not
        for _ in range(50):
            m.pt([(c, 2)] + [(x, 4) for x in g])
        order.append([c])
        c = m.kf()                                                # nMPs == 0: null slots and bad points only
        for _ in range(3):
            m.slot(c, -1, 0)
        for _ in range(2):
            m.pt([(c, 0)] + [(x, 0) for x in good(4)], bad=1)
        order.append([c])
        for flag in ("not_erase", "bad"):                         # redundant, reported, no effect; a later candidate shares its points
            c = m.kf(bad=int(flag == "bad"), not_erase=int(flag == "not_erase"))
            later, g = m.kf(), good(4)
            for _ in range(50):
                m.pt([(c, 7), (later, 0), (g[0], 0), (g[1], 0)])   # three counted others for later only while c is not bad
            order.append([c, later])
        a, b, g, g1 = m.kf(), m.kf(), good(4), m.kf()             # cascade 1: A's cull drops X to nObs 2, B then culls
        m.redundant_points(a, 50, g, octave=7)
        m.redundant_points(b, 49, g)
        m.pt([(a, 7), (b, 0), (g1, 0)])
        order.append([a, b])
        a, c, g = m.kf(), m.kf(bad=1), good(4)                    # cascade 2: A was mpRefKF of Y, every observer left is bad
        m.redundant_points(a, 50, g, octave=7)
        m.redundant_points(c, 10, g, octave=7)
        m.pt([(a, 0), (m.kf(bad=1), 0), (m.kf(bad=1), 0), (m.kf(bad=1), 0), (c, 7)], ref=0)
        order.append([a, c])
        a, b, g = m.kf(), m.kf(), good(4)                         # cascade 3: points with no mpRefKF, one not observed by A
        m.redundant_points(a, 50, g, octave=7)
        m.redundant_points(b, 49, g)
        m.pt([(a, 7), (b, 0)] + [(x, 5) for x in g], ref=None)
        w2 = m.pt([(b, 0)] + [(x, 5) for x in g], ref=None)
        m.slot(a, w2, 7)
        order.append([a, b])
    # interleave the groups at random, keeping each group's order, then add the filtered rows
    flat = []
    groups = [list(g) for g in order]
    while groups:
        i = int(rng.integers(len(groups)))
        flat.append(groups[i].pop(0))
        if not groups[i]:
            groups.pop(i)
    for k in (0, 1) + tuple(recent):
        flat.insert(int(rng.integers(len(flat) + 1)), k)
    sc = m.arrays()
    sc.update(query=query, covis=np.asarray(flat, np.int32), recent=np.asarray(recent, np.int32), th_obs=3, red_thres=float(red_thres))
    sc.update(keyframe_culling_candidates(sc))
    return sc

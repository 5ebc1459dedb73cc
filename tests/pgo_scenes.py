"""Essential graphs of the shapes OptimizeEssentialGraph{LoopClosure,MapFusion} hand to ccm_pgo_solve, and the Sim3 inputs of the
branch tests.  Rows are in ascending keyframe-uid order (agent by agent), as the shim orders them; measurements are Sji = Sjw * Swi
from the current estimate for covisibility / spanning-tree edges and from ground truth for loop and map-fusion edges, like
synth.make_pgo (which stays as it is: the older tests and the golden fixtures use it).

  two_agent_merge  two drifted agents in different frames, each with covisibility edges, joined by map-fusion edges; the one fixed
                   vertex (the loop keyframe) sits in the middle of agent B's rows, so the free-index map has a gap before it
  ragged           several fixed vertices (edges between two of them are dropped), free vertices without edges, duplicate (i, j)
                   edges, pairs in both orders, a free vertex whose only edge goes to a fixed one
  tiny2 / tiny3    K = 2 with one edge (n = 1, one coarse node); K = 3
  far              two_agent_merge 500 m from the origin: the numeric Jacobians are at their noisiest
  large6k / 12k    four agents, K = 6000 (n * 32 >= 1024 * SMs on any H100: the 512-thread PCG CTA) and K = 12000
"""
import numpy as np

from ccm_slam_b200 import synth
from ccm_slam_b200.synth import PGOProblem, _helix_cameras, _mat_to_quat, _rotvec_to_quat, _sim3_inv, _sim3_mul

THETA_GRID = (0.0, 1e-12, 1e-5 * (1 - 1e-9), 1e-5 * (1 + 1e-9), 1e-3, 1.0, np.pi - 1e-6)
# the log decides small rotation on d = (tr R - 1) / 2 > 1 - 1e-5, i.e. theta < acos(1 - 1e-5)
THETA_LOG_EDGE = float(np.arccos(1 - 1e-5))


def _sim3(rotvec, t, s):
    return np.concatenate([_rotvec_to_quat(np.asarray(rotvec, np.float64)), np.asarray(t, np.float64), [s]])


def op_grid(seed=3):
    """(u (n,7), a (n,8), b (n,8)) over the branch grid: theta and sigma on both sides of every 1e-5 boundary (for exp on |omega|
    and sigma, for log on d and log s), d near -1, scales 1e-3 .. 1e3, translations up to 1 km"""
    rng = np.random.default_rng(seed)
    sig = sorted({0.0} | {sg * v for v in THETA_GRID[1:5] for sg in (1, -1)} | {np.log(1e-3), np.log(1e3), 0.3})
    thetas = list(THETA_GRID) + [THETA_LOG_EDGE * (1 - 1e-6), THETA_LOG_EDGE * (1 + 1e-6)]
    us, As, Bs = [], [], []
    for th in thetas:
        for sg in sig:
            for tm in (1.0, 1e3):
                ax = rng.normal(size=3); ax /= np.linalg.norm(ax)
                ups = rng.normal(size=3); ups *= tm / np.linalg.norm(ups)
                us.append(np.concatenate([th * ax, ups, [sg]]))
                As.append(_sim3(th * ax, rng.normal(size=3) * tm, np.exp(sg)))
                Bs.append(_sim3(rng.normal(size=3), rng.normal(size=3) * tm, np.exp(rng.uniform(-7, 7))))
    return np.array(us), np.array(As), np.array(Bs)


def _agents(sizes, seed, fix_scale, n_covis=3, n_fuse=4, n_loop=2, offset=0.0, fixed_agent=1):
    rng = np.random.default_rng(seed)
    gts, ests, starts = [], [], []
    o = 0
    for a, K in enumerate(sizes):
        Rcw, tcw, _, _ = _helix_cameras(K, rng, radius=2.0 + a, dtheta=2 * np.pi / 400, dz=0.01, phase=0.7 * a, z0=3.0 * a)
        gt = np.concatenate([_mat_to_quat(Rcw), tcw, np.ones((K, 1))], -1)
        est = gt.copy()
        acc = np.array([0, 0, 0, 1.0, 0, 0, 0, 1.0])
        for k in range(1, K):
            d = _sim3(rng.normal(size=3) * 0.002, rng.normal(size=3) * 0.01, np.exp(rng.normal() * 0.002 * (0 if fix_scale else 1)))
            acc = _sim3_mul(d, acc)
            est[k] = _sim3_mul(acc, gt[k])
        if a:   # a different world frame: the map-fusion edges carry the misalignment
            est = _sim3_mul(est, _sim3(rng.normal(size=3) * 0.03, rng.normal(size=3) * 0.2, 1.0 if fix_scale else 1.03))
        gts.append(gt); ests.append(est); starts.append(o)
        o += K
    gt, est = np.concatenate(gts), np.concatenate(ests)
    ei, ej, src = [], [], []
    for a, K in enumerate(sizes):
        s0 = starts[a]
        for c in range(1, n_covis + 1):
            k = np.arange(c, K)
            ei.append(s0 + k); ej.append(s0 + k - c); src.append(np.zeros(len(k), bool))
        L = np.arange(n_loop)
        ei.append(s0 + K - 1 - 3 * L); ej.append(s0 + 5 * L); src.append(np.ones(n_loop, bool))
    for a in range(1, len(sizes)):
        i = starts[a] + rng.choice(sizes[a], n_fuse, replace=False)
        j = starts[a - 1] + rng.choice(sizes[a - 1], n_fuse, replace=False)
        ei.append(i); ej.append(j); src.append(np.ones(n_fuse, bool))
    ei, ej, src = np.concatenate(ei), np.concatenate(ej), np.concatenate(src)
    S = np.where(src[:, None], 1.0, 0.0)
    meas = S * _sim3_mul(gt[ej], _sim3_inv(gt[ei])) + (1 - S) * _sim3_mul(est[ej], _sim3_inv(est[ei]))
    fixed = np.zeros(len(est), np.uint8)
    fixed[starts[fixed_agent] + sizes[fixed_agent] // 2] = 1
    if offset:
        shift = _sim3(np.zeros(3), -np.array([offset, 0.6 * offset, -0.3 * offset]), 1.0)   # world moved by |offset| ~ 1.2 x
        est = _sim3_mul(est, shift)
    return PGOProblem(sim3=np.ascontiguousarray(est), fixed=fixed, edge_i=ei.astype(np.int32), edge_j=ej.astype(np.int32),
                      meas=np.ascontiguousarray(meas), fix_scale=fix_scale, gt=gt)


def two_agent_merge(fix_scale=False, offset=0.0):
    return _agents((90, 80), seed=11, fix_scale=fix_scale, offset=offset)


def far(fix_scale=False):
    return two_agent_merge(fix_scale, offset=500.0 / np.sqrt(1 + 0.36 + 0.09))


def ragged(fix_scale=False):
    p = _agents((40,), seed=12, fix_scale=fix_scale, n_loop=1, fixed_agent=0)
    K = 40
    fixed = np.zeros(K, np.uint8)
    fixed[[0, 17, 18, 30]] = 1
    keep = ~np.isin(p.edge_i, [25, 33, 39]) & ~np.isin(p.edge_j, [25, 33, 39])      # 25 and 33: free, no edge; 39: see below
    ei, ej, meas = list(p.edge_i[keep]), list(p.edge_j[keep]), list(p.meas[keep])
    est, gt = p.sim3, p.gt
    add = lambda i, j, src: (ei.append(i), ej.append(j), meas.append(_sim3_mul(src[j], _sim3_inv(src[i]))))
    add(10, 9, gt)            # duplicate of a spanning-tree edge, other measurement (a new loop connection that is also the parent)
    add(10, 9, est)           # exact duplicate
    add(9, 10, gt)            # the same pair in the other order
    add(22, 21, gt); add(21, 22, est)
    add(39, 0, gt)            # 39 is free and its only edge goes to the fixed vertex 0
    add(18, 17, gt); add(30, 18, est)   # both ends fixed: dropped
    return PGOProblem(sim3=est, fixed=fixed, edge_i=np.array(ei, np.int32), edge_j=np.array(ej, np.int32),
                      meas=np.ascontiguousarray(np.array(meas)), fix_scale=fix_scale, gt=gt)


def tiny(K, fix_scale=False):
    p = synth.make_pgo(K=max(K, 4), n_loop=0, n_covis=1, seed=13, fix_scale=fix_scale)
    sim3 = p.sim3[:K].copy()
    if K == 2:
        ei, ej = [1], [0]
    else:
        ei, ej = [1, 2, 2], [0, 1, 0]
    gt = p.gt[:K]
    meas = np.array([_sim3_mul(gt[j], _sim3_inv(gt[i])) for i, j in zip(ei, ej)])
    fixed = np.zeros(K, np.uint8); fixed[0] = 1
    return PGOProblem(sim3=sim3, fixed=fixed, edge_i=np.array(ei, np.int32), edge_j=np.array(ej, np.int32), meas=meas,
                      fix_scale=fix_scale, gt=gt)


def large(K, fix_scale=False):
    return _agents((K // 4,) * 4, seed=14, fix_scale=fix_scale)


SCENES = {
    "two_agent_merge": two_agent_merge,
    "ragged": ragged,
    "tiny2": lambda fix_scale=False: tiny(2, fix_scale),
    "tiny3": lambda fix_scale=False: tiny(3, fix_scale),
    "far": far,
    "large6k": lambda fix_scale=False: large(6000, fix_scale),
    "large12k": lambda fix_scale=False: large(12000, fix_scale),
}

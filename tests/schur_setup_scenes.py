"""Global-BA scenes that each sit exactly on one edge of the reduced camera system's set-up (test infrastructure, numpy only).

The edges, as ccm_ba_create and its kernels define them (ccm_slam_b200/csrc/ba_solver.cu, ba_kernels.cuh):
  * k_row_products keeps a block row's cursors in shared memory when the row has nu <= ROWP_CUR upper blocks, the diagonal block
    included, and in global memory otherwise;
  * the schedule of k_schur_mma cuts a row of n upper blocks into ceil(n / SCHUR_TASK) tasks;
  * the stable radix sort that groups observations by block row keys an observation by its pose slot, or by Kf when the pose is
    fixed, and sorts `bits` bits with 2^bits > Kf: one bit more at Kf = 2^k;
  * the covisibility bitmap holds a row in ceil(Kf / 32) 32-bit words.
Pose slots number the free poses in increasing pose order.  `row_lengths` restates nu for every slot; `EDGES` says where each scene
sits, and tests/test_gpu_schur_setup.py checks both, so that a later change to a builder cannot drift a scene off its edge.

Added landmarks copy the position and the first observation of a landmark their first keyframe sees; the other observations are
random pixels (outliers to the robust kernel).  Only the loop-closure scene is run through LM against the oracle.
"""
from __future__ import annotations

import numpy as np

from ccm_slam_b200 import synth

ROWP_CUR = 512     # k_row_products: most upper blocks of a row whose cursors stay in shared memory
SCHUR_TASK = 64    # k_schur_mma: most blocks of one task


def _base(K, fixed, P, window=8, obs=4, seed=0):
    p = synth.make_global_ba(K, P, obs, window=window, n_agents=1, seed=seed)
    p.fixed = np.zeros(K, np.uint8)
    p.fixed[np.asarray(fixed, np.int64)] = 1
    return p


def _add(p, groups, seed=1):
    """p plus one landmark per list of keyframes in groups, each seen by exactly those keyframes"""
    rng = np.random.default_rng(seed)
    q = p.copy()
    kf, mp, uv, w, pts = [p.obs_kf], [p.obs_mp], [p.obs_uv], [p.obs_w], [p.points]
    nxt = p.P
    for g in groups:
        g = np.asarray(g, np.int32)
        own = np.flatnonzero(p.obs_kf == g[0])
        src = own[0] if own.size else 0
        u = np.stack([rng.uniform(0, 752, g.size), rng.uniform(0, 480, g.size)], 1).astype(np.float32)
        u[0] = p.obs_uv[src]
        kf.append(g); mp.append(np.full(g.size, nxt, np.int32)); uv.append(u)
        w.append((1.0 / synth.SCALE_FACTOR ** (2 * rng.integers(0, 4, g.size))).astype(np.float32))
        pts.append(p.points[p.obs_mp[src]][None])
        nxt += 1
    q.points = np.ascontiguousarray(np.concatenate(pts))
    q.obs_kf = np.ascontiguousarray(np.concatenate(kf)); q.obs_mp = np.ascontiguousarray(np.concatenate(mp))
    q.obs_uv = np.ascontiguousarray(np.concatenate(uv)); q.obs_w = np.ascontiguousarray(np.concatenate(w))
    q.gt_points = None
    return q


def _keep(p, sel):
    q = p.copy()
    q.obs_kf, q.obs_mp, q.obs_uv, q.obs_w = (np.ascontiguousarray(a[sel]) for a in (p.obs_kf, p.obs_mp, p.obs_uv, p.obs_w))
    return q


def free_poses(p):
    return np.flatnonzero(np.asarray(p.fixed) == 0)


def covis_pairs(p):
    """(a, b) slot pairs with a <= b of the upper pattern of S: free poses sharing a landmark, and every diagonal"""
    free = free_poses(p)
    slot = np.full(p.K, -1, np.int64); slot[free] = np.arange(free.size)
    s = slot[p.obs_kf]
    m = s >= 0
    s, lm = s[m], np.asarray(p.obs_mp, np.int64)[m]
    o = np.lexsort((s, lm)); s, lm = s[o], lm[o]
    ptr = np.searchsorted(lm, np.arange(p.P + 1))
    n = np.diff(ptr)
    keys = [np.arange(free.size, dtype=np.int64) * (free.size + 1)]
    for c in np.unique(n[n > 0]):
        ls = np.flatnonzero(n == c)
        iu, ju = np.triu_indices(c)
        idx = ptr[ls][:, None] + np.arange(c)[None, :]
        a, b = s[idx[:, iu]].ravel(), s[idx[:, ju]].ravel()
        keys.append(np.minimum(a, b) * free.size + np.maximum(a, b))
    k = np.unique(np.concatenate(keys))
    return k // max(free.size, 1), k % max(free.size, 1)


def row_lengths(p):
    """nu of every block row (slot order): its upper blocks, the diagonal included"""
    a, _ = covis_pairs(p)
    return np.bincount(a, minlength=free_poses(p).size)


def sort_bits(Kf):
    """the radix sort's key width in ccm_ba_create: keys 0..Kf (Kf for a fixed pose) need 2^bits > Kf"""
    bits = 1
    while (1 << bits) <= Kf:
        bits += 1
    return bits


def _spans(K, every, spans, P, seed):
    """K poses, every `every`-th fixed (from 0), one landmark per span (first slot, length) seen by that many consecutive free poses"""
    p = _base(K, np.arange(0, K, every), P, seed=seed)
    free = free_poses(p)
    return _add(p, [free[s:s + n] for s, n in spans], seed=seed)


def _with_kf(Kf, every, window=12, seed=0):
    """Kf free poses with a fixed pose every `every` poses (from 0)"""
    K = Kf
    while K - len(range(0, K, every)) < Kf:
        K += 1
    return _base(K, np.arange(0, K, every), 10 * K, window=window, seed=seed)


def loop_closure():
    """980 free poses: rows of exactly ROWP_CUR + 1 (slot 20) and ROWP_CUR (slot 100) upper blocks, and slot 1 a loop-closure
    keyframe sharing a landmark with every other keyframe (a row of Kf - 1 blocks).  Every long row is a star of two-observation
    landmarks, so S stays sparse enough for the oracle's exact factorisation."""
    p = _base(1000, np.arange(0, 1000, 50), 8000, seed=3)
    free = free_poses(p)
    stars = [[free[s], free[s + j]] for s, n in ((20, ROWP_CUR + 1), (100, ROWP_CUR)) for j in range(1, n)]
    return _add(p, stars + [[free[1], k] for k in range(p.K) if k != free[1]], seed=4)


def task_cut():
    """rows of exactly 64, 65, 128 and 129 upper blocks (slots 10, 80, 150, 160): one, two, two and three tasks"""
    return _spans(300, 40, [(10, SCHUR_TASK), (80, SCHUR_TASK + 1), (150, 2 * SCHUR_TASK), (160, 2 * SCHUR_TASK + 1)], 2400, seed=5)


def word_edge(Kf):
    """Kf free poses, a fixed pose every 10; free slot 0 also shares a landmark with slots 30, 31, 32 and Kf - 1"""
    p = _with_kf(Kf, 10, window=6, seed=Kf)
    free = free_poses(p)
    return _add(p, [[free[0], free[j]] for j in sorted({30, 31, 32, Kf - 1}) if 0 < j < Kf], seed=Kf)


def empty_rows():
    """free pose 50 and the last pose without observations; free pose 90 sees only landmarks no other free pose sees (fixed
    poses 0, 37, 80 and 85 still do): a row with its diagonal block only"""
    p = _base(120, [0, 37, 80, 85], 1500, window=10, seed=7)
    kf, mp = p.obs_kf, p.obs_mp
    lonely = np.zeros(p.P, bool); lonely[mp[kf == 90]] = True
    drop = (kf == 50) | (kf == p.K - 1) | (lonely[mp] & (kf != 90) & (p.fixed[kf] == 0))
    return _keep(p, ~drop)


def diag_only(K=150, fixed=(0, 70, 71, 149)):
    """every landmark seen by one free pose (its first free observer) and any fixed ones: the only upper blocks are diagonals"""
    p = _base(K, list(fixed), 10 * K, window=10, seed=9)
    freek = p.fixed[p.obs_kf] == 0
    o = np.lexsort((p.obs_kf, p.obs_mp))
    first = np.zeros(p.E, bool)
    fm = o[freek[o]]
    head = np.ones(fm.size, bool); head[1:] = p.obs_mp[fm[1:]] != p.obs_mp[fm[:-1]]
    first[fm[head]] = True
    return _keep(p, first | ~freek)


def one_free_pose():
    """one free pose among eleven fixed ones: one diagonal block, one task, a one-CTA launch"""
    return diag_only(K=12, fixed=[k for k in range(12) if k != 5])


def cfg4_shard():
    from tests.test_gpu_schur_order import _shard
    return _shard(synth.make_config("cfg4"), 20000, 35000)


def cfg4_dense_rows():
    from tests.test_gpu_schur_order import _seen_by_all
    return _seen_by_all(synth.make_config("cfg4"))


KF_EDGE = 8   # Kf = 2^k - 1, 2^k, 2^k + 1

SCENES = {
    "loop_closure": loop_closure,
    "task_cut": task_cut,
    **{f"kf{(1 << KF_EDGE) + d}": (lambda d=d: _with_kf((1 << KF_EDGE) + d, 16, seed=11 + d)) for d in (-1, 0, 1)},
    **{f"kf{n}": (lambda n=n: word_edge(n)) for n in (31, 32, 33, 63, 64, 65)},
    "empty_rows": empty_rows,
    "diag_only": diag_only,
    "one_free_pose": one_free_pose,
    "cfg4_shard": cfg4_shard,
    "cfg4_dense_rows": cfg4_dense_rows,
}

# where each scene sits: rows {slot: nu} that must have exactly that many upper blocks, Kf, and other properties
EDGES = {
    "loop_closure": dict(rows={20: ROWP_CUR + 1, 100: ROWP_CUR, 1: 979}, Kf=980),
    "task_cut": dict(rows={10: SCHUR_TASK, 80: SCHUR_TASK + 1, 150: 2 * SCHUR_TASK, 160: 2 * SCHUR_TASK + 1}),
    **{f"kf{(1 << KF_EDGE) + d}": dict(Kf=(1 << KF_EDGE) + d, fixed_among_free=True) for d in (-1, 0, 1)},
    **{f"kf{n}": dict(Kf=n, fixed_among_free=True) for n in (31, 32, 33, 63, 64, 65)},
    "empty_rows": dict(no_obs=[50, 119], diag_only_rows=[90]),
    "diag_only": dict(max_row=1),
    "one_free_pose": dict(Kf=1, max_row=1),
    "cfg4_shard": dict(empty_rows=True),
    "cfg4_dense_rows": dict(longest_over=ROWP_CUR),
}

"""The Schur product lists, entry by entry: every upper block's list (the diagonal ones included) holds exactly the observation pairs a
numpy restatement derives from the observation arrays, in increasing order of the row-side observation (landmark order), and two
handles created from the same input give bit-identical lists, S, b_schur, Hpp and final state (the final state with the PCG's coarse
level off: its set-up sums with atomics, so only the solve without it is deterministic)."""
import numpy as np
import pytest

from ccm_slam_b200 import api, synth
from tests.test_gpu_schur import SHAPES

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module", autouse=True)
def _dev():
    assert api.device_count() > 0, "no CUDA device: the product path has no CPU fallback"
    api.init(0)


def _shard(p, L0, L1):
    """the problem restricted to landmarks [L0, L1): every pose, the shard's points and their observations"""
    sel = (p.obs_mp >= L0) & (p.obs_mp < L1)
    return synth.BAProblem(poses=p.poses, intr=p.intr, fixed=p.fixed, points=p.points[L0:L1], obs_kf=p.obs_kf[sel],
                           obs_mp=(p.obs_mp[sel] - L0).astype(np.int32), obs_uv=p.obs_uv[sel], obs_w=p.obs_w[sel],
                           edge_flags=None if p.edge_flags is None else p.edge_flags[sel])


def _seen_by_all(p):
    """p plus one landmark every keyframe observes: rows of up to K-1 upper blocks (more than k_row_products keeps in shared memory)"""
    q = p.copy()
    q.points = np.concatenate([p.points, p.points[:1]])
    kf = np.arange(p.K, dtype=np.int32)
    q.obs_kf = np.concatenate([p.obs_kf, kf]); q.obs_mp = np.concatenate([p.obs_mp, np.full(p.K, p.P, np.int32)])
    q.obs_uv = np.concatenate([p.obs_uv, np.tile(p.obs_uv[:1], (p.K, 1))]); q.obs_w = np.concatenate([p.obs_w, np.ones(p.K, np.float32)])
    return q


LIST_CASES = dict(SHAPES)
LIST_CASES["cfg4_shard"] = lambda: _shard(synth.make_config("cfg4"), 20000, 35000)   # the poses outside the shard have empty rows
LIST_CASES["cfg4_dense_rows"] = lambda: _seen_by_all(synth.make_config("cfg4"))


def _expected(p):
    """every pair (e, o) of observations of one landmark with e seen by a free pose a, o by a free pose b, and b > a or o == e, as
    positions in the landmark-sorted order; sorted by block (a, b), then e, then o"""
    order = np.argsort(p.obs_mp, kind="stable")
    kf = p.obs_kf[order].astype(np.int64)
    lm = p.obs_mp[order].astype(np.int64)
    ptr = np.searchsorted(lm, np.arange(p.P + 1))
    n = ptr[lm + 1] - ptr[lm]                                   # observations of each e's landmark
    e = np.repeat(np.arange(kf.size), n)
    o = np.repeat(ptr[lm], n) + (np.arange(e.size) - np.repeat(np.cumsum(n) - n, n))
    free = p.fixed[kf] == 0
    keep = free[e] & free[o] & ((kf[o] > kf[e]) | (o == e))
    e, o = e[keep], o[keep]
    s = np.lexsort((o, e, kf[o], kf[e]))
    return kf[e][s], kf[o][s], e[s], o[s]


@pytest.mark.parametrize("name", list(LIST_CASES))
def test_product_lists_are_the_pairs_in_landmark_order(name):
    p = LIST_CASES[name]()
    h = api.BAHandle(p)
    try:
        got = h.debug_products()
    finally:
        h.close()
    blk, ptr, pairs = got["blk"], got["ptr"], got["pairs"]
    n = np.diff(ptr)
    assert np.all(blk[:, 0] <= blk[:, 1])
    row = np.repeat(blk[:, 0], n); col = np.repeat(blk[:, 1], n)
    first = np.zeros(pairs.shape[0], bool); first[ptr[:-1][n > 0]] = True
    assert np.all((np.diff(pairs[:, 0]) > 0) | first[1:]), f"{name}: a list is not strictly increasing in e"
    a, b, e, o = _expected(p)
    assert pairs.shape[0] == e.size, f"{name}: {pairs.shape[0]} products, expected {e.size}"
    assert np.array_equal(row, a) and np.array_equal(col, b), f"{name}: products in the wrong blocks"
    assert np.array_equal(pairs[:, 0], e) and np.array_equal(pairs[:, 1], o), f"{name}: lists differ from the restatement"
    if name == "awkward":
        assert np.bincount(blk[:, 0]).max() > 64   # rows longer than one task of k_schur_mma's schedule
    if name == "cfg4_dense_rows":
        assert np.bincount(blk[:, 0]).max() > 512


def _collect(h, lam=1e-3, flags=None):
    """lists, linear system, S and b_schur at lam, and a 5-iteration state with per-edge chi2 and depth; with flags, another 5
    iterations from the start after set_edge_flags(flags)"""
    out = dict(lists=h.debug_products(), build=h.debug_build())
    out["schur"] = h.debug_schur(lam)
    out["blocks"] = h.debug_schur_blocks()
    h.reset()
    out["final"] = h.optimize(iterations=5, want_edges=True)
    if flags is not None:
        h.set_edge_flags(flags)
        h.reset()
        out["flagged"] = h.optimize(iterations=5, want_edges=True)
    for run in ("final", "flagged"):
        for k in ("t_setup_ms", "t_optimize_ms", "t_download_ms", "t_optimize_event_ms"):
            out.get(run, {}).pop(k, None)
    return out


def _everything(p, lam=1e-3, flags=None):
    h = api.BAHandle(p)
    try:
        return _collect(h, lam, flags)
    finally:
        h.close()


def _shuffled(p, seed):
    """p with its observations (and edge flags) in random order"""
    perm = np.random.default_rng(seed).permutation(p.E)
    q = p.copy()
    q.obs_kf, q.obs_mp, q.obs_uv, q.obs_w = p.obs_kf[perm], p.obs_mp[perm], p.obs_uv[perm], p.obs_w[perm]
    q.edge_flags = None if p.edge_flags is None else p.edge_flags[perm]
    return q


def _grouped(q):
    """q's observations grouped by landmark with a stable sort, as ccm_ba_create groups them, and the permutation that did it"""
    order = np.argsort(q.obs_mp, kind="stable")
    g = q.copy()
    g.obs_kf, g.obs_mp, g.obs_uv, g.obs_w = q.obs_kf[order], q.obs_mp[order], q.obs_uv[order], q.obs_w[order]
    g.edge_flags = None if q.edge_flags is None else q.edge_flags[order]
    return g, order


def _in_grouped_order(out, order):
    """_collect's outputs of a create from ungrouped observations, their per-observation arrays (W, chi2, depth) put in grouped order"""
    out["build"]["W"] = out["build"]["W"][order]
    for run in ("final", "flagged"):
        if run in out:
            out[run]["chi2"] = out[run]["chi2"][order]
            out[run]["depth_pos"] = out[run]["depth_pos"][order]
    return out


def _same_as_grouped(q, label, flags=None):
    """a create from the ungrouped observations of q against one from the same observations grouped: bit-identical through the
    permutation (run with the PCG's coarse level off: its set-up sums with atomics); flags in q's order"""
    g, order = _grouped(q)
    _same(_everything(g, flags=None if flags is None else flags[order]), _in_grouped_order(_everything(q, flags=flags), order),
          f"{label} (ungrouped against grouped)")


def _same(x, y, path):
    if isinstance(x, dict):
        for k in x:
            _same(x[k], y[k], f"{path}.{k}")
    elif isinstance(x, np.ndarray):
        assert x.tobytes() == y.tobytes(), f"{path} differs between two creates"
    elif isinstance(x, float):
        assert np.float64(x).tobytes() == np.float64(y).tobytes(), f"{path} differs between two creates"
    else:
        assert x == y, f"{path} differs between two creates"


@pytest.mark.parametrize("name", ["small", "cfg4", "awkward"])
def test_two_creates_give_bit_identical_systems(name, monkeypatch):
    monkeypatch.setenv("CCM_PCG_NC", "0")   # read by ccm_ba_create
    p = SHAPES[name]()
    first = _everything(p, 1e-3)
    second = _everything(p, 1e-3)
    _same(first, second, name)

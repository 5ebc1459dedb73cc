"""CPU checks of the f64 Schur restatement (tests/schur_ref.py) the GPU Schur and PCG tests compare against: it agrees with the
oracle's BlockSolver restatement entry by entry, its tolerance fails on the kinds of mistake a Schur kernel makes, and the awkward
shape really has the features it is built for."""
import numpy as np
import pytest

from ccm_slam_b200 import api, synth
from tests import schur_ref as R


def _lams(b):
    md = max(np.abs(np.einsum("kii->ki", b["Hpp"])).max(), np.abs(np.einsum("kii->ki", b["Hll"])).max())
    return {"lm_start": 1e-5 * md, "heavy": 1e-1 * md}


@pytest.mark.parametrize("robust", [True, False])
@pytest.mark.parametrize("lam_kind", ["lm_start", "heavy"])
@pytest.mark.parametrize("name", ["tiny", "small", "cfg2"])
def test_restatement_matches_oracle(oracle, name, lam_kind, robust):
    p = synth.make_config(name)
    b = oracle.ba_build(p, robust=robust, huber_delta=api.HUBER_GBA)
    lam = _lams(b)[lam_kind]
    ref = R.schur_reference(p, b, lam)
    orc = oracle.ba_schur_solve(p, lam, robust=robust, huber_delta=api.HUBER_GBA, dense=True)
    assert orc["rc"] == 0
    S, T = ref.dense()
    assert R.ratio(orc["S"] - S, T) < 0.1
    assert R.ratio(orc["bschur"].reshape(-1, 6) - ref.bschur, ref.bschur_tol) < 0.1
    d, dt = ref.dx_point(orc["dx_pose"])
    assert R.ratio(orc["dx_point"] - d, dt) < 0.1


def test_awkward_shape_has_its_features():
    p = synth.make_awkward_ba()
    free = np.flatnonzero(p.fixed == 0)
    Kf = free.size
    assert Kf % 8 and Kf % 3 and Kf % 4
    slot = np.full(p.K, -1); slot[free] = np.arange(Kf)
    fixed = np.flatnonzero(p.fixed)
    assert np.any(fixed > 0) and any(f // 8 != g // 8 for f, g in zip(fixed[1:], fixed[2:]))   # fixed keyframes inside panels
    assert not np.all(np.diff(p.obs_mp) >= 0)                                                 # not grouped by landmark
    key = p.obs_mp.astype(np.int64) * p.K + p.obs_kf
    assert np.unique(key).size == p.E                                                          # no repeated (pose, landmark)
    cnt = np.bincount(p.obs_mp, minlength=p.P)
    assert cnt.max() > 160 and np.any(cnt == 1)
    nfree = np.bincount(p.obs_mp[p.fixed[p.obs_kf] == 0], minlength=p.P)
    assert np.any((cnt > 0) & (nfree == 0))                                                    # seen by fixed keyframes only
    run = np.convolve(cnt, np.ones(33, int), "valid")
    assert np.any(run <= 160)                                                                  # stages capped at 32 landmarks
    assert np.any(p.edge_flags & 1) and np.any(p.edge_flags & 2)
    # co-observation offsets in free-pose slots, and the largest product list of an off-diagonal block
    o = np.lexsort((p.obs_kf, p.obs_mp))
    mp, sl = p.obs_mp[o], slot[p.obs_kf[o]]
    pairs = {}
    offs = set()
    for l in np.unique(mp[cnt[mp] <= 10]):
        s = sl[mp == l]; s = s[s >= 0]
        for i in range(s.size):
            for j in range(i + 1, s.size):
                offs.add(int(s[j] - s[i]))
                pairs[(s[i], s[j])] = pairs.get((s[i], s[j]), 0) + 1
    assert {43, 44} <= offs and max(offs) > 44
    assert max(pairs.values()) > 4096


# ---- mutation checks: each mistake must exceed the tolerance by at least 100 x -------------------------------------------------
@pytest.fixture(scope="module")
def awkward(oracle):
    p = synth.make_awkward_ba()
    b = oracle.ba_build(p, robust=True, huber_delta=api.HUBER_GBA)
    lam = _lams(b)["lm_start"]
    ref = R.schur_reference(p, b, lam)
    return p, ref


def _export(ref):
    return dict(rowptr=ref.rowptr.copy(), col=ref.col.copy(), val=ref.val.copy(), bschur=ref.bschur.copy())


def _products(p, ref, a, b):
    """the Schur products Z_a Z_b^T of block (a, b), one per common active landmark"""
    act = (np.zeros(p.E, np.uint8) if p.edge_flags is None else p.edge_flags) & 1 == 0
    ea = np.flatnonzero((p.obs_kf == a) & act); eb = np.flatnonzero((p.obs_kf == b) & act)
    common, ia, ib = np.intersect1d(p.obs_mp[ea], p.obs_mp[eb], return_indices=True)
    return np.stack([ref.Z[ea[i]] @ ref.Z[eb[j]].T for i, j in zip(ia, ib)]) if common.size else np.zeros((0, 6, 6))


def _pos(ref, a, b):
    q = ref.rowptr[a] + np.searchsorted(ref.col[ref.rowptr[a]:ref.rowptr[a + 1]], b)
    assert ref.col[q] == b
    return q


def _drop(ref, got, a, b, P):
    got["val"][_pos(ref, a, b)] += P       # S = ... - sum: leaving a product out adds it back
    got["val"][_pos(ref, b, a)] += P.T


def test_mutation_drop_median_product_of_a_long_list(awkward):
    p, ref = awkward
    off = ref.row != ref.col
    a, b = None, None
    for q in np.flatnonzero(off & (ref.row < ref.col)):
        prods = _products(p, ref, ref.row[q], ref.col[q])
        if len(prods) > 1000:
            a, b = ref.row[q], ref.col[q]
            break
    assert a is not None
    mag = np.abs(prods).max(axis=(1, 2))
    got = _export(ref)
    _drop(ref, got, a, b, prods[np.argsort(mag)[len(mag) // 2]])
    assert R.compare_blocks(ref, got)["S"] > 100
    assert R.worst_block(ref, got)[:2] in ((a, b), (b, a))


def test_mutation_drop_one_of_two_products(awkward):
    p, ref = awkward
    for q in np.flatnonzero(ref.row < ref.col):
        prods = _products(p, ref, ref.row[q], ref.col[q])
        if len(prods) == 2:
            break
    assert len(prods) == 2
    got = _export(ref)
    _drop(ref, got, ref.row[q], ref.col[q], prods[0])
    assert R.compare_blocks(ref, got)["S"] > 100


def test_mutation_negate_and_transpose_an_off_diagonal_block(awkward):
    p, ref = awkward
    a = int(np.flatnonzero(p.fixed == 0)[100])
    q = ref.rowptr[a] + 1 if ref.col[ref.rowptr[a]] == a else ref.rowptr[a]   # the first neighbour of a
    assert ref.row[q] != ref.col[q]
    got = _export(ref)
    got["val"][q] = -got["val"][q]
    assert R.compare_blocks(ref, got)["S"] > 100
    got = _export(ref)
    got["val"][q] = got["val"][q].T.copy()
    assert R.compare_blocks(ref, got)["S"] > 100


def test_mutation_neighbouring_landmark_in_b_schur(awkward):
    p, ref = awkward
    act = (p.edge_flags & 1) == 0
    e = ref.sel[ref.sel_active][len(ref.sel) // 2]
    assert act[e]
    l = p.obs_mp[e]
    got = _export(ref)
    got["bschur"][p.obs_kf[e]] += ref.Z[e] @ ref.g[l] - ref.Z[e] @ ref.g[l + 1]
    assert R.compare_blocks(ref, got)["bschur"] > 100

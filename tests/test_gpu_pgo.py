"""The Sim3 essential graph on the device, step by step (ccm_pgo_solve, csrc/pgo.cu): the Sim3 arithmetic of sim3_math.cuh as nvcc
compiles it, the per-edge numeric Jacobians, the assembled 7x7 block system, its PCG solve on every path, and the LM run -- against the
40-digit restatement and the f64 assembly of tests/sim3_ref.py, and against the oracle, on the scenes of tests/pgo_scenes.py."""
import numpy as np
import pytest
import scipy.sparse.linalg as spla

from ccm_slam_b200 import api
from tests import pgo_scenes as ps
from tests import sim3_ref as S

pytestmark = pytest.mark.gpu
GJB = 32           # pivots per Gauss-Jordan sweep of the coarse inverse (pcg.cuh)
PCG_TOL = 1e-10    # ccm_pgo_solve's defaults
PCG_MAX = 5000
BIG, BIG_NC = 4096, 256   # from 4096 free vertices on: 256 coarse nodes, piecewise-linear prolongation (pgo.cu)
SCENES = ("two_agent_merge", "ragged", "tiny2", "tiny3", "far", "large6k", "large12k")


@pytest.fixture(scope="module", autouse=True)
def _dev():
    assert api.device_count() > 0, "no CUDA device: the product path has no CPU fallback"
    api.init(0)


_cache = {}


def _scene(name, fix_scale):
    key = (name, fix_scale)
    if key not in _cache:
        if len(_cache) > 4:
            _cache.clear()
        _cache[key] = ps.SCENES[name](fix_scale)
    return _cache[key]


def coarse_shape(n, nc_max):
    """pcg_coarse_shape (pcg.cuh)"""
    if nc_max <= 0 or n <= 0:
        return 0, 0
    agg = max(1, -(-n // nc_max))
    return agg, -(-n // agg)


# ---- Sim3 arithmetic ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("fix_scale", [False, True])
def test_sim3_ops_inside_mp_bounds(fix_scale, capsys):
    u, a, b = ps.op_grid()
    got = api.sim3_debug_ops(u, a, b, fix_scale)
    worst = {}
    for k in range(len(u)):
        for n, (v, bd) in S.ops(u[k], a[k], b[k], fix_scale).items():
            r = S.ratio(got[n][k] - v, S.TAU * bd)
            if r > worst.get(n, (-1.0,))[0]:
                worst[n] = (r, k)
    with capsys.disabled():
        print(f"\n[sim3 ops fix_scale={fix_scale}] device error / bound: " + " ".join(f"{n} {r:.3g} (row {k})" for n, (r, k) in worst.items()))
    assert all(r <= 1.0 for r, _ in worst.values()), worst
    if fix_scale:
        assert np.array_equal(got["oplus"][:, 7], a[:, 7])     # s bit-unchanged


# ---- per-edge linearisation --------------------------------------------------------------------------------------------------
def _edge_rows():
    """(meas, si, sj, free_i, free_j): sampled scene edges (the far scene's included) with every free / fixed combination, and edges
    whose relative Sim3 sits on the branch grid"""
    rows = []
    for name, k in (("two_agent_merge", 8), ("far", 8), ("ragged", 6), ("tiny3", 3)):
        p = ps.SCENES[name](False)
        for q, e in enumerate(np.random.default_rng(len(name)).choice(len(p.edge_i), k, replace=False)):
            rows.append((p.meas[e], p.sim3[p.edge_i[e]], p.sim3[p.edge_j[e]], q % 3 != 1, q % 3 != 2))
    u, a, b = ps.op_grid()
    for k in range(0, len(a), 13):
        rows.append((b[k], a[k], b[(k + 7) % len(b)], True, True))
    return rows


@pytest.mark.parametrize("fix_scale", [False, True])
def test_edge_jacobians_inside_mp_bounds(oracle, fix_scale, capsys):
    rows = _edge_rows()
    m, si, sj = [np.array([r[c] for r in rows]) for c in range(3)]
    free = np.array([[r[3], r[4]] for r in rows], np.int32)
    got = api.pgo_debug_edges(m, si, sj, free, fix_scale)
    P = oracle.Pieces("oracle")
    w_mp = w_or = 0.0
    for k, (mk, ik, jk, fi, fj) in enumerate(rows):
        ref = S.edge_jacobians(mk, ik, jk, fi, fj, fix_scale)
        oi, oj = P.pgo_edge_jacobian(mk, ik, jk, fix_scale)
        w_mp = max(w_mp, S.ratio(got["err"][k] - ref["err"], S.TAU * ref["err_bound"]),
                   S.ratio(got["Ji"][k] - ref["Ji"], S.TAU * ref["Ji_bound"]), S.ratio(got["Jj"][k] - ref["Jj"], S.TAU * ref["Jj_bound"]))
        w_or = max(w_or, S.ratio(got["err"][k] - oracle.pgo_edge_error(mk, ik, jk), S.TAU * ref["err_bound"]))
        for J, O, B, f in ((got["Ji"][k], oi, ref["Ji_bound"], fi), (got["Jj"][k], oj, ref["Jj_bound"], fj)):
            if f:
                w_or = max(w_or, S.ratio(J - O, S.TAU * B))
            else:
                assert not J.any(), (k, "the Jacobian of a fixed side is not exactly zero")
        if fix_scale:
            assert not got["Ji"][k][:, 6].any() and not got["Jj"][k][:, 6].any(), (k, "scale column under fix_scale")
    with capsys.disabled():
        print(f"\n[edge jacobians fix_scale={fix_scale}] {len(rows)} edges: device vs exact {w_mp:.3g}, vs oracle {w_or:.3g} of the mp bound")
    assert w_mp <= 1.0 and w_or <= 1.0


# ---- the assembled system ----------------------------------------------------------------------------------------------------
def _system(oracle, p):
    return S.System(p, *S.oracle_edges(p, oracle.Pieces("oracle")))


@pytest.mark.parametrize("fix_scale", [False, True])
@pytest.mark.parametrize("name", SCENES)
def test_system_matches_restatement(oracle, name, fix_scale, capsys):
    p = _scene(name, fix_scale)
    lam = 1e-16
    d = api.pgo_debug_system(p, lam)
    ref = _system(oracle, p)
    assert d["n"] == ref.n and d["nnzb"] == ref.nnzb
    assert np.array_equal(d["vidx"], ref.vidx) and np.array_equal(d["rowptr"], ref.rowptr) and np.array_equal(d["col"], ref.col)
    rH = S.ratio(d["H"] - ref.H, S.TAU * ref.H_bound)
    rb = S.ratio(d["b"] - ref.b, S.TAU * ref.b_bound)
    rc = abs(d["chi2"] - ref.chi2) / (S.TAU * ref.chi2_bound)
    # Minv: the inverse of the device's own damped diagonal block, within a condition-scaled bound
    rp, col = d["rowptr"], d["col"]
    diag = d["H"][[rp[a] + np.searchsorted(col[rp[a]:rp[a + 1]], a) for a in range(d["n"])]]
    D = diag + lam * np.eye(7)[None]
    k = 6 if p.fix_scale else 7     # under fix_scale the scale row / column of D is lam alone: checked exactly below
    Dk = D[:, :k, :k]
    inv = np.linalg.inv(Dk)
    cond = np.abs(Dk).sum(-1).max(-1) * np.abs(inv).sum(-1).max(-1)
    tolM = S.TAU * 7 * S.U * cond * np.abs(inv).max((-1, -2))
    rM = float((np.abs(d["Minv"][:, :k, :k] - inv).max((-1, -2)) / tolM).max())
    with capsys.disabled():
        print(f"\n[system {name} fix_scale={fix_scale}] n {d['n']} nnzb {d['nnzb']} error / bound: H {rH:.3g} b {rb:.3g} chi2 {rc:.3g} Minv {rM:.3g}")
    assert rH <= 1.0 and rb <= 1.0 and rc <= 1.0 and rM <= 1.0
    if p.fix_scale:
        assert not d["H"][:, 6, :].any() and not d["H"][:, :, 6].any() and not d["b"][:, 6].any()
        assert not d["Minv"][:, 6, :6].any() and not d["Minv"][:, :6, 6].any() and np.all(d["Minv"][:, 6, 6] == 1.0 / lam)
        assert not d["x"][:, 6].any()


# ---- PCG on the exported system ----------------------------------------------------------------------------------------------
# (label, scene, CCM_PCG_NC or None, expected CTA) -- the default coarse size is 64 nodes below BIG free vertices, BIG_NC from there
PCG_CASES = [
    ("256x2-nc64", "two_agent_merge", None, 256),
    ("256x2-nc3", "two_agent_merge", "3", 256),
    ("256x2-coarse-off", "two_agent_merge", "0", 256),
    ("256x2-nc1", "tiny2", None, 256),
    ("256x2-far", "far", None, 256),
    ("256x2-ragged", "ragged", None, 256),
    ("512x1-nc64", "large6k", None, 512),
    ("512x1-12k", "large12k", None, 512),
]


def _pcg_check(p, lam, monkeypatch, nc_env):
    if nc_env is None:
        monkeypatch.delenv("CCM_PCG_NC", raising=False)
    else:
        monkeypatch.setenv("CCM_PCG_NC", nc_env)
    d = api.pgo_debug_system(p, lam)
    M = S.block_matrix(d["H"], d["rowptr"], d["col"], lam)
    bv, x = d["b"].ravel(), d["x"].ravel()
    true = np.linalg.norm(M @ x - bv) / np.linalg.norm(bv)
    xs = spla.splu(M).solve(bv)
    return d, dict(true=true, reported=d["pcg_relres"], iters=d["pcg_iters"], flag=d["pcg_flag"],
                   x_vs_splu=np.abs(x - xs).max() / np.abs(xs).max())


@pytest.mark.parametrize("lam_kind", ["1e-16", "1e-5maxdiag"])
@pytest.mark.parametrize("label,name,nc_env,cta", PCG_CASES, ids=[c[0] for c in PCG_CASES])
def test_pcg_solves_the_exported_system(label, name, nc_env, cta, lam_kind, monkeypatch, capsys):
    p = _scene(name, False)
    lam = 1e-16
    if lam_kind != "1e-16":
        d0 = api.pgo_debug_system(p, 1e-16)
        lam = 1e-5 * np.abs(np.diagonal(d0["H"], axis1=1, axis2=2)).max()
    d, r = _pcg_check(p, lam, monkeypatch, nc_env)
    paths = d["paths"]
    n = d["n"]
    agg, nc = coarse_shape(n, int(nc_env) if nc_env is not None else (BIG_NC if n >= BIG else 64))
    assert paths["pcg_block"] == cta and paths["pcg_agg"] == agg and paths["pcg_nc"] == nc, paths
    assert paths["coarse_used"] == (nc > 0) and d["pcg_nC"] == 7 * nc
    with capsys.disabled():
        print(f"\n[pgo pcg {label} lam={lam:.3g}] n {n} CTA {cta} agg {agg} nc {nc} sweeps {-(-7 * nc // GJB)} iters {r['iters']} "
              f"flag {r['flag']} true relres {r['true']:.3g} reported {r['reported']:.3g} x vs splu {r['x_vs_splu']:.3g}")
    assert r["flag"] == 0 and r["iters"] < PCG_MAX
    assert r["true"] <= PCG_TOL
    assert (r["true"] < 1e-12 and r["reported"] < 1e-12) or r["reported"] / 10 <= r["true"] <= 10 * r["reported"]
    assert r["x_vs_splu"] <= 1e-6


def test_pcg_cases_cover_the_paths():
    """the cases above reach both CTA shapes, the coarse level off, nc = 1, both parities of the Gauss-Jordan sweep count and an
    aggregate size that does not divide n"""
    n = int((S.structure(ps.two_agent_merge())[1] >= 0).sum())
    n_ragged = int((S.structure(ps.ragged())[1] >= 0).sum())
    sweeps = lambda nc: -(-7 * nc // GJB)
    # 256x2-nc64 and 256x2-ragged: the inverse ends in the second and in the first of the ping-pong buffers (coarse_inverse)
    assert sweeps(coarse_shape(n, 64)[1]) % 2 == 1 and sweeps(coarse_shape(n_ragged, 64)[1]) % 2 == 0
    assert n % coarse_shape(n, 3)[0] != 0
    assert len(ps.tiny(2).sim3) == 2 and coarse_shape(1, 64) == (1, 1)
    assert {c[3] for c in PCG_CASES} == {256, 512}


# ---- LM against the oracle ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("fix_scale", [False, True])
@pytest.mark.parametrize("name", SCENES)
def test_lm_matches_oracle(oracle, name, fix_scale, capsys):
    p = _scene(name, fix_scale)
    ref = oracle.pgo_solve(p, iterations=20)
    got = api.pgo_solve(p, iterations=20)
    with capsys.disabled():
        print(f"\n[pgo lm {name} fix_scale={fix_scale}] iters {got['iters_done']} chi2 {got['chi2_initial']:.6g} -> {got['chi2_final']:.6g} "
              f"pcg iters {got['trace'][:, 6].astype(int).tolist()} relres max {got['trace'][:, 7].max():.3g}")
    # test_gpu_frontend's rule -- same iteration count, same decision and trial count wherever |rho| is above the noise floor -- up to
    # the first iteration whose oracle step changes chi2 by less than 1e-6 relative: from there on both runs sit at the minimum, the
    # gain ratios are numeric-Jacobian noise (it grows with the translations that cancel: far, 500 m) and a graph that can be solved
    # exactly (tiny2) is at chi2 ~ 1e-31.  Both must reach that iteration and end no worse than the oracle's noise allows.
    tr = ref["trace"]
    prev = np.concatenate([[ref["chi2_initial"]], tr[:-1, 2]])
    flat = np.flatnonzero(prev - tr[:, 2] <= 1e-6 * prev)
    n_cmp = int(flat[0]) + 1 if flat.size else ref["iters_done"]
    assert ref["iters_done"] >= 1 and got["iters_done"] >= n_cmp
    if not flat.size:
        assert got["iters_done"] == ref["iters_done"]
    assert abs(got["chi2_initial"] - ref["chi2_initial"]) <= 1e-9 * ref["chi2_initial"]
    for it in range(n_cmp):
        if abs(ref["trace"][it, 3]) > 1e-9 and abs(got["trace"][it, 3]) > 1e-9:
            assert (got["trace"][it, 3] > 0) == (ref["trace"][it, 3] > 0) and got["trace"][it, 4] == ref["trace"][it, 4], it
    assert got["chi2_final"] <= ref["chi2_final"] * (1 + 1e-2) + 1e-20 * ref["chi2_initial"]
    # end state: 1e-4 of the largest entry; 1e-3 from BIG free vertices on (DESIGN.md, "Essential graph on the device")
    scale = np.abs(ref["sim3"]).max() * (1e-3 if (S.structure(p)[1] >= 0).sum() >= BIG else 1e-4)
    assert np.abs(got["sim3"] - ref["sim3"]).max() <= scale
    assert np.all(got["trace"][:, 7] <= PCG_TOL) and np.all(got["trace"][:, 6] < PCG_MAX), got["trace"][:, 6:]
    act, vidx, _, _ = S.structure(p)
    still = vidx < 0    # fixed vertices and free vertices without an edge
    assert np.array_equal(got["sim3"][still], p.sim3[still])


# ---- ABI edges ---------------------------------------------------------------------------------------------------------------
def test_abi_edges_match_oracle(oracle):
    p = ps.tiny(3)
    for kw, mod in (({"stop": np.ones(1, np.uint8)}, None), ({"iterations": 0}, None),
                    ({}, lambda q: q.__class__(**{**q.__dict__, "fixed": np.ones(len(q.sim3), np.uint8)})),
                    ({}, lambda q: q.__class__(**{**q.__dict__, "edge_i": q.edge_i[:0], "edge_j": q.edge_j[:0], "meas": q.meas[:0]}))):
        q = mod(p) if mod else p
        ref = oracle.pgo_solve(q, **kw)
        got = api.pgo_solve(q, **kw)
        assert got["iters_done"] == ref["iters_done"] and np.array_equal(got["sim3"], q.sim3), (kw, got["iters_done"], ref["iters_done"])
        if mod:
            assert got["iters_done"] == -1
    bad = p.__class__(**{**p.__dict__, "edge_j": np.array([1, 3, 0], np.int32)})
    with pytest.raises(api.CCMError):
        api.pgo_solve(bad)
    with pytest.raises(api.CCMError):
        api.pgo_debug_system(bad, 1e-16)
    ok = api.pgo_solve(p)
    assert ok["iters_done"] >= 1 and ok["chi2_final"] < ok["chi2_initial"]

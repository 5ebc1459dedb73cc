"""The coarse level of the PCG preconditioner (csrc/pcg.cuh): the Galerkin matrix P^T S P the set-up assembles and the inverse its
blocked Gauss-Jordan sweeps (GJB pivots per sweep on the f64 tensor cores) leave in the ping-pong buffers, exported through
ccm_ba_debug_coarse and checked against numpy in f64 -- at nC = 6, at sizes that are not multiples of GJB with both parities of the
sweep count, at 1536 and at the 2304 the streamed solve holds, for every CTA shape of the set-up launch, through the solves of k_pcg
and k_pcg2 that read the inverse, and in the 7x7-block pose graph."""
import numpy as np
import pytest
import scipy.sparse as sp
import scipy.sparse.linalg as spla

from ccm_slam_b200 import api, synth
from tests import pgo_scenes as ps
from tests import sim3_ref as S

pytestmark = pytest.mark.gpu
GJB = 32   # pivots per Gauss-Jordan sweep (pcg.cuh)
EPS = np.finfo(np.float64).eps


@pytest.fixture(scope="module", autouse=True)
def _dev():
    assert api.device_count() > 0, "no CUDA device: the product path has no CPU fallback"
    api.init(0)


def coarse_shape(n, nc_max):
    """pcg_coarse_shape (pcg.cuh)"""
    if nc_max <= 0 or n <= 0:
        return 0, 0
    agg = max(1, -(-n // nc_max))
    return agg, -(-n // agg)


def sweeps(nC):
    return -(-nC // GJB)


def prolongation(n, agg, nc, BS=6):
    """P of pcg.cuh coarse_parents with piecewise-linear prolongation, (BS n) x (BS nc)"""
    rows, cols, vals = [], [], []
    for a in range(n):
        if nc < 2:
            par = [(a // agg, 1.0)]
        else:
            pos = min(max((a + 0.5) / agg - 0.5, 0.0), nc - 1.0)
            lo = min(int(pos), nc - 2)
            f = min(max(pos - lo, 0.0), 1.0)
            par = [(lo, 1.0 - f), (lo + 1, f)]
        for J, w in par:
            if w != 0.0:
                for d in range(BS):
                    rows.append(a * BS + d); cols.append(J * BS + d); vals.append(w)
    return sp.csr_matrix((vals, (rows, cols)), shape=(BS * n, BS * nc))


_problems = {}


def _problem(name):
    if name not in _problems:
        _problems.clear()
        _problems[name] = {
            "small": lambda: synth.make_config("small"),
            "cfg4": lambda: synth.make_config("cfg4"),
            "cfg5_tenth": lambda: synth.make_config("cfg5", K=1000, P=100000),
            "cfg5_768": lambda: synth.make_config("cfg5", K=769, P=77000),
            "cfg5_4500": lambda: synth.make_config("cfg5", K=4500, P=60000),
        }[name]()
    return _problems[name]


# (label, problem, env, coarse nodes)
CASES = [
    ("nC6", "small", {"CCM_PCG_NC": "1"}, 1),
    ("cfg4-default", "cfg4", {}, coarse_shape(799, 128)[1]),
    ("cfg4-nc100", "cfg4", {"CCM_PCG_NC": "100"}, 100),
    ("k_pcg2-tenth", "cfg5_tenth", {"CCM_PCG_IMPL": "2"}, coarse_shape(999, 128)[1]),
    ("k_pcg2-nc100", "cfg5_tenth", {"CCM_PCG_IMPL": "2", "CCM_PCG_NC": "100"}, 100),
    ("nC1536", "cfg5_768", {"CCM_PCG_IMPL": "2", "CCM_PCG_NC": "256"}, 256),
    ("nC2304", "cfg5_768", {"CCM_PCG_IMPL": "2", "CCM_PCG_NC": "384"}, 384),
    ("setup512", "cfg5_4500", {}, coarse_shape(4499, 256)[1]),
    ("setup1024", "cfg5_4500", {"CCM_PCG_IMPL": "1", "CCM_PCG_BLOCK": "1024"}, coarse_shape(4499, 256)[1]),
]


def test_cases_cover_the_sizes():
    """nC = 6, sizes off the GJB grid with an odd and an even sweep count, 1536 and 2304"""
    nCs = {c[0]: 6 * c[3] for c in CASES}
    assert nCs["nC6"] == 6 and nCs["nC1536"] == 1536 and nCs["nC2304"] == 2304
    off = [n for n in nCs.values() if n % GJB]
    assert {sweeps(n) % 2 for n in off} == {0, 1}


@pytest.mark.parametrize("label,name,env,nc", CASES, ids=[c[0] for c in CASES])
def test_coarse_inverse(label, name, env, nc, monkeypatch, capsys):
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    p = _problem(name)
    h = api.BAHandle(p)
    try:
        paths = h.debug_paths()
        assert paths["pcg_nc"] == nc, paths
        b = h.debug_build(huber_delta=api.HUBER_GBA)
        lam = 1e-5 * max(np.abs(np.einsum("kii->ki", b["Hpp"])).max(), np.abs(np.einsum("kii->ki", b["Hll"])).max())
        got = h.debug_schur(lam, huber_delta=api.HUBER_GBA)
        blk = h.debug_schur_blocks()
        c1 = h.debug_coarse()
        c2 = h.debug_coarse()
    finally:
        h.close()
    nC = 6 * nc
    Ac, Ainv = c1["Ac"], c1["Ainv"]
    assert Ac.shape == (nC, nC)
    # the assembly against P^T S P in numpy (S from the same export, pose order = block-row order of the free poses)
    free = np.flatnonzero(p.fixed == 0)
    slot = np.full(p.K, -1); slot[free] = np.arange(free.size)
    Sm = sp.bsr_matrix((blk["val"], slot[blk["col"]], np.concatenate([[0], np.cumsum(np.diff(blk["rowptr"])[free])])),
                       shape=(6 * free.size, 6 * free.size)).tocsr()
    P = prolongation(free.size, paths["pcg_agg"], nc)
    ref_A = (P.T @ Sm @ P).toarray()
    assert np.abs(Ac - ref_A).max() <= 1e-12 * np.abs(ref_A).max()
    # the inverse against numpy's, in f64, within what the condition number allows
    ref = np.linalg.inv(Ac)
    cond = np.linalg.cond(Ac)
    err = np.abs(Ainv - ref).max() / np.abs(ref).max()
    resid = np.abs(Ac @ Ainv - np.eye(nC)).max()
    bound = nC * EPS * cond
    with capsys.disabled():
        print(f"\n[coarse {label}] CTA {paths['pcg_block']} nC {nC} sweeps {sweeps(nC)} cond {cond:.3g} inverse rel err {err:.3g} "
              f"|A X - I| {resid:.3g} bound {bound:.3g} pcg iters {got['pcg_iters']}")
    assert err <= bound and resid <= bound
    # the inversion is deterministic: the same assembled matrix gives the same bits
    # (the assembly adds with atomics, so two assemblies may differ in their last bits)
    if np.array_equal(c1["Ac"], c2["Ac"]):
        assert np.array_equal(c1["Ainv"], c2["Ainv"])
    else:
        assert np.abs(c2["Ainv"] - ref).max() / np.abs(ref).max() <= bound
    # the solve that read the inverse (k_pcg, or k_pcg2 after the set-up launch) solved the exported system
    bv = blk["bschur"][free].ravel()
    x = got["dx_pose"][free].ravel()
    assert np.linalg.norm(Sm @ x - bv) / np.linalg.norm(bv) <= 1e-10


def test_coarse_inverse_identical_across_handles(monkeypatch):
    """two handles built on the same problem: same assembled matrix bits -> same inverse bits"""
    p = _problem("cfg4")
    out = []
    for _ in range(2):
        h = api.BAHandle(p)
        try:
            b = h.debug_build(huber_delta=api.HUBER_GBA)
            lam = 1e-5 * max(np.abs(np.einsum("kii->ki", b["Hpp"])).max(), np.abs(np.einsum("kii->ki", b["Hll"])).max())
            h.debug_schur(lam, huber_delta=api.HUBER_GBA)
            out.append(h.debug_coarse())
        finally:
            h.close()
    if np.array_equal(out[0]["Ac"], out[1]["Ac"]):
        assert np.array_equal(out[0]["Ainv"], out[1]["Ainv"])
    else:
        ref = np.linalg.inv(out[0]["Ac"])
        bound = out[0]["Ac"].shape[0] * EPS * np.linalg.cond(out[0]["Ac"])
        assert np.abs(out[1]["Ainv"] - ref).max() / np.abs(ref).max() <= bound


# ---- the 7x7-block pose graph (pgo.cu): the same set-up on BS = 7, checked through the solve that uses the inverse ----------
def _pgo_n():
    return int((S.structure(ps.two_agent_merge())[1] >= 0).sum())


PGO_NC = ("5", "9", "64")


def test_pgo_cases_cover_both_parities():
    n = _pgo_n()
    nCs = [7 * coarse_shape(n, int(v))[1] for v in PGO_NC]
    assert any(c % GJB for c in nCs)
    assert {sweeps(c) % 2 for c in nCs} == {0, 1}


@pytest.mark.parametrize("nc_env", PGO_NC)
def test_pgo_coarse_solve(nc_env, monkeypatch, capsys):
    monkeypatch.setenv("CCM_PCG_NC", nc_env)
    p = ps.SCENES["two_agent_merge"](False)
    d0 = api.pgo_debug_system(p, 1e-16)
    lam = 1e-5 * np.abs(np.diagonal(d0["H"], axis1=1, axis2=2)).max()
    d = api.pgo_debug_system(p, lam)
    M = S.block_matrix(d["H"], d["rowptr"], d["col"], lam)
    bv, x = d["b"].ravel(), d["x"].ravel()
    nc = coarse_shape(d["n"], int(nc_env))[1]
    assert d["paths"]["coarse_used"] == 1 and d["pcg_nC"] == 7 * nc
    true = np.linalg.norm(M @ x - bv) / np.linalg.norm(bv)
    xs = spla.splu(M).solve(bv)
    with capsys.disabled():
        print(f"\n[pgo coarse nc {nc}] nC {7 * nc} sweeps {sweeps(7 * nc)} iters {d['pcg_iters']} true relres {true:.3g}")
    assert d["pcg_flag"] == 0 and true <= 1e-10
    assert np.abs(x - xs).max() / np.abs(xs).max() <= 1e-6

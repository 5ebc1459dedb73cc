"""CPU self-test of tests/sim3_ref.py, the restatement the device's Sim3 arithmetic, edge Jacobians and pose-graph system are checked
against (tests/test_gpu_pgo.py): the oracle stays inside its bounds over the branch grid and on sampled edges, the f64 assembly
reproduces the oracle's first LM step, and every deliberate defect of the restatement leaves its bound by at least 1e3."""
import numpy as np
import pytest
import scipy.sparse.linalg as spla

from tests import pgo_scenes as ps
from tests import sim3_ref as S
from ccm_slam_b200 import synth

OPS = ("exp", "log", "mul", "inv", "oplus")


def _oracle_ops(O, u, a, b, fix_scale):
    uu = np.array(u, np.float64)
    if fix_scale:
        uu[6] = 0.0
    return dict(exp=O.sim3_exp(u), log=O.sim3_log(a), mul=O.sim3_mul(a, b), inv=O.sim3_inv(a), oplus=O.sim3_mul(O.sim3_exp(uu), a))


def _ops_ratio(O, rows, fix_scale):
    u, a, b = ps.op_grid()
    worst = dict.fromkeys(OPS, 0.0)
    for k in rows:
        ref = S.ops(u[k], a[k], b[k], fix_scale)
        got = _oracle_ops(O, u[k], a[k], b[k], fix_scale)
        for n in OPS:
            worst[n] = max(worst[n], S.ratio(got[n] - ref[n][0], S.TAU * ref[n][1]))
    return worst


@pytest.mark.parametrize("fix_scale", [False, True])
def test_oracle_ops_inside_bounds(oracle, fix_scale, capsys):
    w = _ops_ratio(oracle, range(len(ps.op_grid()[0])), fix_scale)
    with capsys.disabled():
        print(f"\n[sim3 ops, fix_scale={fix_scale}] oracle error / bound: " + " ".join(f"{k} {v:.3g}" for k, v in w.items()))
    assert max(w.values()) <= 1.0, w


def _edge_sample():
    """(meas, si, sj, from a scene) rows: sampled edges of the scenes, and edges whose relative Sim3 sits on the branch grid"""
    out = []
    for name, k in (("two_agent_merge", 4), ("far", 4), ("ragged", 3), ("tiny3", 2)):
        p = ps.SCENES[name](False)
        for e in np.random.default_rng(len(name)).choice(len(p.edge_i), k, replace=False):
            out.append((p.meas[e], p.sim3[p.edge_i[e]], p.sim3[p.edge_j[e]], True))
    u, a, b = ps.op_grid()
    for k in range(0, len(a), 19):
        out.append((b[k], a[k], b[(k + 7) % len(b)], False))
    return out


def test_oracle_edges_inside_bounds(oracle, capsys):
    P = oracle.Pieces("oracle")
    worst = dict(err=0.0, J=0.0, closed=0.0)
    for fix_scale in (False, True):
        for m, si, sj, scene in _edge_sample():
            r = S.edge_jacobians(m, si, sj, fix_scale=fix_scale)
            Ji, Jj = P.pgo_edge_jacobian(m, si, sj, fix_scale)
            worst["J"] = max(worst["J"], S.ratio(Ji - r["Ji"], S.TAU * r["Ji_bound"]), S.ratio(Jj - r["Jj"], S.TAU * r["Jj_bound"]))
            worst["err"] = max(worst["err"], S.ratio(oracle.pgo_edge_error(m, si, sj) - r["err"], S.TAU * r["err_bound"]))
            ce = oracle.pgo_edge_error(m, si, sj)[None]
            ci, cj = S.jacobian_bound(m[None], si[None], sj[None], ce, [True], [True], fix_scale)
            if scene:   # the closed form is for essential-graph edges (small relative rotations, scales near 1), not the grid's extremes
                worst["closed"] = max(worst["closed"], S.ratio(Ji - r["Ji"], S.TAU * ci[0]), S.ratio(Jj - r["Jj"], S.TAU * cj[0]),
                                      S.ratio(ce[0] - r["err"], S.TAU * S.error_bound(m[None], si[None], sj[None], ce)[0]))
            if fix_scale:
                assert not Ji[:, 6].any() and not Jj[:, 6].any() and not r["Ji"][:, 6].any()
    with capsys.disabled():
        print(f"\n[edge jacobians] oracle error / bound: err {worst['err']:.3g} J {worst['J']:.3g}; "
              f"against the closed-form bound of the assembly {worst['closed']:.3g}")
    assert worst["err"] <= 1.0 and worst["J"] <= 1.0
    assert worst["closed"] <= 1.0   # the closed form the f64 assembly uses covers the oracle's rounding


def _system(oracle, p):
    return S.System(p, *S.oracle_edges(p, oracle.Pieces("oracle")))


def _step(oracle, p, sysm, lam=1e-16):
    x = spla.splu(sysm.sparse(lam=lam)).solve(sysm.b.ravel()).reshape(-1, 7)
    out = np.array(p.sim3, np.float64)
    for k in np.flatnonzero(sysm.vidx >= 0):
        u = x[sysm.vidx[k]].copy()
        if p.fix_scale:
            u[6] = 0.0
        out[k] = oracle.sim3_mul(oracle.sim3_exp(u), p.sim3[k])
    return out


@pytest.mark.parametrize("name,fix_scale", [("make_pgo60", False), ("make_pgo60", True), ("ragged", False), ("two_agent_merge", True)])
def test_assembly_reproduces_oracle_step(oracle, name, fix_scale):
    p = synth.make_pgo(K=60, fix_scale=fix_scale) if name == "make_pgo60" else ps.SCENES[name](fix_scale)
    ref = oracle.pgo_solve(p, iterations=1)
    assert ref["iters_done"] == 1 and ref["trace"][0, 3] > 0 and ref["trace"][0, 4] == 1   # the first trial is accepted
    sysm = _system(oracle, p)
    assert abs(sysm.chi2 - ref["chi2_initial"]) <= S.TAU * sysm.chi2_bound
    got = _step(oracle, p, sysm)
    assert np.abs(got - ref["sim3"]).max() <= 1e-9 * max(1.0, np.abs(ref["sim3"]).max())
    if fix_scale:
        assert not sysm.H[:, 6, :].any() and not sysm.H[:, :, 6].any() and not sysm.b[:, 6].any()


def test_structure_of_ragged():
    p = ps.ragged()
    act, vidx, rowptr, col = S.structure(p)
    fixed = p.fixed != 0
    assert not np.any(fixed[p.edge_i[act]] & fixed[p.edge_j[act]]) and len(act) == len(p.edge_i) - 3
    assert vidx[25] == vidx[33] == -1 and (vidx[fixed] == -1).all() and vidx[39] >= 0
    assert rowptr[vidx[39] + 1] - rowptr[vidx[39]] == 1                      # only its diagonal block
    for a in range(len(rowptr) - 1):
        c = col[rowptr[a]:rowptr[a + 1]]
        assert (np.diff(c) > 0).all() and a in c


# ---- mutations -------------------------------------------------------------------------------------------------------------
# exp_half shows in exp only just below theta = 1e-5: w moves by theta^2 / 8 = 1.25e-11, about 1e3 TAU-bounds of w
@pytest.mark.parametrize("mut,ops", [("abc_swap", ("exp", "log")), ("exp_half", ("exp",))])
def test_op_mutations_exceed_bounds(oracle, monkeypatch, mut, ops):
    monkeypatch.setitem(S.MUT, mut, True)
    w = _ops_ratio(oracle, range(len(ps.op_grid()[0])), False)
    assert min(w[o] for o in ops) >= 1e3, w


def test_no_fix_scale_mutation_exceeds_bounds(oracle, monkeypatch):
    monkeypatch.setitem(S.MUT, "no_fix_scale", True)
    P = oracle.Pieces("oracle")
    p = ps.two_agent_merge(True)
    m, si, sj = p.meas[3], p.sim3[p.edge_i[3]], p.sim3[p.edge_j[3]]
    r = S.edge_jacobians(m, si, sj, fix_scale=True)
    Ji, _ = P.pgo_edge_jacobian(m, si, sj, True)
    assert S.ratio(Ji - r["Ji"], S.TAU * r["Ji_bound"]) >= 1e3
    u, a, b = ps.op_grid()
    k = int(np.argmax(np.abs(u[:, 6])))
    ref = S.ops(u[k], a[k], b[k], True)["oplus"]
    assert S.ratio(_oracle_ops(oracle, u[k], a[k], b[k], True)["oplus"] - ref[0], S.TAU * ref[1]) >= 1e3


@pytest.mark.parametrize("mut,name", [("swap_jac", "two_agent_merge"), ("mirror_no_transpose", "two_agent_merge"),
                                      ("fixed_side", "ragged")])
def test_assembly_mutations_exceed_bounds(oracle, monkeypatch, mut, name):
    p = ps.SCENES[name](False)
    edges = S.oracle_edges(p, oracle.Pieces("oracle"))
    good = S.System(p, *edges)
    monkeypatch.setitem(S.MUT, mut, True)
    bad = S.System(p, *edges)
    r = max(S.ratio(bad.H - good.H, S.TAU * good.H_bound), S.ratio(bad.b - good.b, S.TAU * good.b_bound))
    assert r >= 1e3, r
    # and the step taken from the defective system no longer reproduces the oracle's
    ref = oracle.pgo_solve(p, iterations=1)
    assert np.abs(_step(oracle, p, bad) - ref["sim3"]).max() > 1e3 * 1e-9 * np.abs(ref["sim3"]).max()

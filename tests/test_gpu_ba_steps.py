"""GPU suite: the global BA's linearisation, per-edge report, pose update, trial chi2 and initial lambda, step by step against the
restatement of tests/ba_ref.py on the scenes of tests/ba_scenes.py (every scene at its start, half-way along the oracle's run and at
the oracle's end state; robust on and off; both Huber deltas).  Every entry must lie within TAU times its bound; the worst ratios are
printed.  The Schur and PCG passes in between are checked by test_gpu_schur.py, test_gpu_fused_z.py and test_gpu_pcg.py."""
import numpy as np
import pytest

from ccm_slam_b200 import api
from tests import ba_ref as F
from tests import ba_scenes as B
from tests.ba_ref import TAU, ratio

pytestmark = pytest.mark.gpu

CASES = [(n, r) for n in B.SCENES for r in (True, False)]
_st = {}


@pytest.fixture(scope="module", autouse=True)
def _dev():
    assert api.device_count() > 0, "no CUDA device: the product path has no CPU fallback"
    api.init(0)


def states(oracle, name):
    if name not in _st:
        _st[name] = B.states(oracle, B.scene(name))
    return _st[name]


def _report(capsys, title, worst):
    with capsys.disabled():
        print(f"\n{title}: " + " ".join(f"{k}={v:.3g}" for k, v in worst.items()))
    for k, v in worst.items():
        assert v <= 1.0, (title, k, v)


def _upd(worst, k, v):
    worst[k] = max(worst.get(k, 0.0), v)


@pytest.mark.parametrize("name,robust", CASES)
def test_linearisation_matches_restatement(oracle, name, robust, capsys):
    """debug_build's W per edge (exact zeros for inactive edges and fixed keyframes), Hll / bl per landmark, Hpp / bp per pose and
    the robust chi2 sum; the per-edge report (plain chi2 of every active edge, depth sign)"""
    p = B.scene(name)
    worst = {}
    for st, poses, points in states(oracle, name):
        q = B.with_state(p, poses, points)
        h = api.BAHandle(q)
        try:
            for delta in B.DELTAS:
                got = h.debug_build(robust=robust, huber_delta=delta)
                L = F.Lin(q, robust=robust, delta=delta)
                _upd(worst, "W", ratio(got["W"] - L.W, TAU * L.W_b))
                _upd(worst, "Hll", ratio(got["Hll"] - L.Hll, TAU * L.Hll_b))
                _upd(worst, "bl", ratio(got["bl"] - L.bl, TAU * L.bl_b))
                _upd(worst, "Hpp", ratio(got["Hpp"] - L.Hpp, TAU * L.Hpp_b))
                _upd(worst, "bp", ratio(got["bp"] - L.bp, TAU * L.bp_b))
                _upd(worst, "chi2", ratio(got["chi2_robust_sum"] - L.chi2_sum, TAU * L.chi2_sum_b))
            rep = h.optimize(iterations=0, want_edges=True)
            act = L.act
            _upd(worst, "edge_chi2", ratio(rep["chi2"][act] - L.chi2[act], TAU * L.chi2_b[act]))
            clear = np.abs(L.depth) > L.depth_b          # the sign is decided; depth exactly 0 has bound 0 and must read as not positive
            assert np.array_equal(rep["depth_pos"][clear], (L.depth[clear] > 0).astype(np.uint8)), st
            assert (rep["depth_pos"][(L.depth == 0) & (L.depth_b == 0)] == 0).all()
        finally:
            h.close()
    _report(capsys, f"linearisation {name} robust={robust}", worst)


@pytest.mark.parametrize("name,robust", CASES)
def test_update_step_matches_restatement(oracle, name, robust, capsys):
    """debug_step with the exp-map cases: trial poses (fixed ones bit-identical), trial points = points + dx, the trial chi2
    restated at the device's own trial state, and both halves of the gain-ratio denominator"""
    p = B.scene(name)
    worst = {}
    x = F.exp_cases(p.K)
    for st, poses, points in states(oracle, name):
        q = B.with_state(p, poses, points)
        h = api.BAHandle(q)
        try:
            L = F.Lin(q, robust=robust, delta=api.HUBER_GBA)
            lam = F.lambda_init(L)[0]
            got = h.debug_step(x, lam, robust=robust, huber_delta=api.HUBER_GBA)
            want, bnd = F.update_poses(q, x)
            _upd(worst, "pose_trial", ratio(got["pose_trial"] - want, TAU * bnd))
            assert np.array_equal(got["pose_trial"][q.fixed == 1], q.poses[q.fixed == 1])
            assert np.array_equal(got["pt_trial"], q.points + got["dx_point"])
            c, cb = F.chi2_at(q, got["pose_trial"], got["pt_trial"], robust=robust, delta=api.HUBER_GBA)
            _upd(worst, "chi2_trial", ratio(got["chi2_trial"] - c, TAU * cb))
            sp, spb = F.scale_pose(L, x, lam)
            _upd(worst, "scale_pose", ratio(got["scale_pose"] - sp, TAU * spb))
            sl, slb = F.scale_point(L, got["dx_point"], lam)
            _upd(worst, "scale_point", ratio(got["scale_point"] - sl, TAU * slb))
            # the same steps from poses turned far from the identity: products that need the w < 0 flip
            h.set_estimate(B.turned(q.poses), None)
            got = h.debug_step(x, lam, robust=robust, huber_delta=api.HUBER_GBA)
            want, bnd = F.update_poses(B.with_state(q, B.turned(q.poses), q.points), x)
            _upd(worst, "pose_trial_turned", ratio(got["pose_trial"] - want, TAU * bnd))
        finally:
            h.close()
    _report(capsys, f"update {name} robust={robust}", worst)


@pytest.mark.parametrize("name", B.SCENES)
def test_initial_lambda(oracle, name, capsys):
    """1e-5 times the largest diagonal entry (in Hll on multicam, in Hpp on sizes), and the initial chi2"""
    p = B.scene(name)
    L = F.Lin(p, delta=api.HUBER_GBA)
    lam, lb = F.lambda_init(L)
    r = api.ba_solve(p, iterations=1, huber_delta=api.HUBER_GBA)
    tr = r["trace"][0]
    lam0 = tr[1] / np.prod([2.0 ** k for k in range(1, int(tr[4]))])    # undo the doublings of rejected trials (exact)
    worst = dict(lambda0=ratio(lam0 - lam, TAU * lb), chi2_initial=ratio(r["chi2_initial"] - L.chi2_sum, TAU * L.chi2_sum_b))
    _report(capsys, f"initial lambda {name} ({L.max_diag()[2]})", worst)


def _state_close(res, ref, tol):
    Tg = api.poses_to_Tcw_f32(res["poses"]).astype(np.float64)
    To = api.poses_to_Tcw_f32(ref["poses"]).astype(np.float64)
    assert np.abs(Tg - To).max() <= tol * max(1.0, np.abs(To).max())
    pg = res["points"].astype(np.float32).astype(np.float64); po = ref["points"].astype(np.float32).astype(np.float64)
    assert np.abs(pg - po).max() <= tol * max(1.0, np.abs(po).max())


@pytest.mark.parametrize("name,delta", [("multicam", api.HUBER_GBA), ("multicam", api.HUBER_LOCAL), ("sizes", api.HUBER_GBA)])
def test_lm_matches_oracle(oracle, name, delta):
    """full LM runs with test_gpu_ba.py's assertions; multicam carries the Huber band and the inactive edges at depth 0, so its
    chi2 must stay finite and its state must move as the oracle's does"""
    p = B.scene(name)
    ref = oracle.ba_solve(p, iterations=10, huber_delta=delta)
    # the near points make the reduced system ill-conditioned: solve it to 1e-13 so that the comparison with the oracle's direct
    # factorisation tests the linearisation, update and residual rather than the PCG's default stopping point
    res = api.ba_solve(p, iterations=10, huber_delta=delta, pcg_tol=1e-13, pcg_max_iter=5000)
    assert np.isfinite(res["chi2_initial"]) and np.isfinite(res["trace"][:, 2]).all()
    assert res["iters_done"] == ref["iters_done"] and res["trials_total"] == ref["trials_total"]
    n = len(ref["trace"])
    assert np.allclose(res["trace"][:n, 1], ref["trace"][:, 1], rtol=1e-6)
    assert np.allclose(res["trace"][:n, 2], ref["trace"][:, 2], rtol=1e-7)
    assert np.array_equal(res["trace"][:n, 4], ref["trace"][:, 4])
    _state_close(res, ref, 1e-4)
    assert not np.array_equal(res["poses"], p.poses)
    assert np.array_equal(res["poses"][p.fixed == 1], p.poses[p.fixed == 1])
    act, _ = F.edge_flags(p)
    assert np.allclose(res["chi2"][act], ref["chi2"][act], rtol=1e-6, atol=1e-9)
    assert np.array_equal(res["depth_pos"], ref["depth_pos"])

"""CPU suite: the restatement of the global BA's linearisation, pose update and denominator (tests/ba_ref.py) against the oracle on
the scenes of tests/ba_scenes.py, entry by entry within TAU times its bound, and every deliberate defect of ba_ref.MUT caught by at
least 100 times its bound.  The scenes are checked to really contain their edge cases."""
import numpy as np
import pytest

from ccm_slam_b200 import api, synth
from tests import ba_ref as F
from tests import ba_scenes as B
from tests.ba_ref import TAU, ratio

_states = {}


def states(oracle, name):
    if name not in _states:
        _states[name] = B.states(oracle, B.scene(name))
    return _states[name]


def mp_active(q, n=None):
    """the R-evaluated terms of the active edges of q (all of them up to ba_ref.MP_ALL edges, or the first n and the near ones)"""
    act, _ = F.edge_flags(q)
    near = getattr(q, "special", {}).get("near", ())
    idx = F.sample_edges(q, special=near) if n is None else np.union1d(np.arange(n), near).astype(np.int64)
    idx = idx[act[idx]]
    return (idx,) + F.mp_edges(q, idx)


def edge_ratios(oracle, q, robust, delta, mp):
    """worst |restated - oracle| / bound of the per-edge terms (orc_ba_linearize) of the active edges of problem q"""
    act, _ = F.edge_flags(q)
    idx, ex, bd = mp
    lin = oracle.ba_linearize(q, robust=robust, huber_delta=delta)
    L = F.Lin(q, robust=robust, delta=delta)
    out = dict(err=ratio(ex["err"] - lin["err"][idx], TAU * bd["err"]),
               Jp=ratio(ex["Jp"] - lin["Jpose"][idx], TAU * bd["Jp"]),
               Jl=ratio(ex["Jl"] - lin["Jpoint"][idx], TAU * bd["Jl"]),
               chi2=ratio(ex["chi2"] - lin["chi2"][idx], TAU * bd["chi2"]),
               rho1=ratio(L.rho1[act] - lin["rho1"][act], TAU * L.rho1_b[act]),
               chi2_sum=ratio(L.chi2_sum - lin["chi2_robust_sum"], TAU * L.chi2_sum_b))
    # the vectorised shadow against the exact values: within its (doubled) bound
    out["shadow"] = max(ratio(L.err[idx] - ex["err"], L.err_b[idx]), ratio(L.Jl[idx] - ex["Jl"], L.Jl_b[idx]),
                        ratio(L.Jp[idx] - ex["Jp"], L.Jp_b[idx]))
    return out


def block_ratios(oracle, q, robust, delta):
    ref = oracle.ba_build(q, robust=robust, huber_delta=delta)
    L = F.Lin(q, robust=robust, delta=delta)
    return dict(Hpp=ratio(L.Hpp - ref["Hpp"], TAU * L.Hpp_b), bp=ratio(L.bp - ref["bp"], TAU * L.bp_b),
                Hll=ratio(L.Hll - ref["Hll"], TAU * L.Hll_b), bl=ratio(L.bl - ref["bl"], TAU * L.bl_b),
                W=ratio(L.W - ref["W"], TAU * L.W_b))


def update_ratio(oracle, q, x):
    got, bnd = F.update_poses(q, x)
    ref = np.array(q.poses, copy=True)
    for k in np.flatnonzero(q.fixed == 0):
        ref[k] = oracle.se3_mul(oracle.se3_exp(x[k]), q.poses[k])
    return ratio(got - ref, TAU * bnd)


def scale_ratio(oracle, q, robust, delta):
    """the two denominator halves at the oracle's own Schur step against numpy sums over the oracle's bp / bl"""
    ref = oracle.ba_build(q, robust=robust, huber_delta=delta)
    L = F.Lin(q, robust=robust, delta=delta)
    lam = F.lambda_init(L)[0]
    st = oracle.ba_schur_solve(q, lam, robust=robust, huber_delta=delta)
    x, xl = st["dx_pose"], st["dx_point"]
    sp, spb = F.scale_pose(L, x, lam)
    sl, slb = F.scale_point(L, xl, lam)
    free = q.fixed == 0
    rp = float((x[free] * (lam * x[free] + ref["bp"][free])).sum())
    rl = float((xl * (lam * xl + ref["bl"])).sum())
    return max(ratio(sp - rp, TAU * spb), ratio(sl - rl, TAU * slb))


def all_ratios(oracle, name="multicam"):
    p = B.scene(name)
    out = {}
    mp = mp_active(p, 300)
    for delta in B.DELTAS:
        for k, v in {**edge_ratios(oracle, p, True, delta, mp), **block_ratios(oracle, p, True, delta)}.items():
            out[k] = max(out.get(k, 0.0), v)
    x = F.exp_cases(p.K)
    out["update"] = max(update_ratio(oracle, p, x), update_ratio(oracle, B.with_state(p, B.turned(p.poses), p.points), x))
    out["scale"] = scale_ratio(oracle, p, True, api.HUBER_GBA)
    return out


@pytest.mark.parametrize("name", B.SCENES)
@pytest.mark.parametrize("robust", [True, False])
def test_restatement_matches_oracle(oracle, name, robust):
    """per-edge terms, blocks, chi2 sum, update and denominator at every state of the scene, both Huber deltas"""
    p = B.scene(name)
    worst = {}
    for st, poses, points in states(oracle, name):
        q = B.with_state(p, poses, points)
        mp = mp_active(q)
        for delta in B.DELTAS:
            r = {**edge_ratios(oracle, q, robust, delta, mp), **block_ratios(oracle, q, robust, delta)}
            for k, v in r.items():
                worst[k] = max(worst.get(k, 0.0), v)
        worst["update"] = max(worst.get("update", 0.0), update_ratio(oracle, q, F.exp_cases(q.K, seed=len(st))))
        worst["scale"] = max(worst.get("scale", 0.0), scale_ratio(oracle, q, robust, api.HUBER_GBA))
    print(name, robust, {k: f"{v:.3g}" for k, v in worst.items()})
    for k, v in worst.items():
        assert v <= 1.0, (k, v)


@pytest.mark.parametrize("mut,keys", [("dsqr_double", ("rho1",)), ("small_half", ("update",)), ("intr_kf0", ("err", "Jp", "Hpp")),
                                      ("jl_col2_sign", ("Jl", "Hll", "W")), ("w_fixed", ("W",)), ("bl_sign", ("bl",)),
                                      ("no_point_scale", ("scale",))])
def test_every_mutation_fails(oracle, mut, keys):
    if "base" not in _states:
        _states["base"] = all_ratios(oracle)
    base = _states["base"]
    F.MUT[mut] = True
    try:
        bad = all_ratios(oracle)
    finally:
        F.MUT[mut] = False
    assert all(v <= 1.0 for v in base.values()), base
    assert max(bad[k] for k in keys) >= 100.0, (mut, bad)


def test_scenes_contain_their_edge_cases(oracle):
    for name in B.SCENES:
        p = B.scene(name)
        act, rob = F.edge_flags(p)
        cams = {tuple(r) for r in p.intr}
        assert len(cams) >= 4 and all(np.float32(v) == v for v in p.intr.ravel())
        octaves = (1.0 / synth.SCALE_FACTOR ** (2 * np.arange(8))).astype(np.float32)
        assert set(octaves.tolist()) <= set(p.obs_w[act].tolist())                           # invSigma2 of all 8 octaves
        flags = np.asarray(p.edge_flags)
        assert {0, 1, 2, 3} <= set(flags.tolist())
        fixed = np.flatnonzero(p.fixed)
        assert ((fixed > 0) & (fixed < p.K - 1)).any()                                       # fixed among free keyframes
        j = p.special["only_fixed_point"]
        assert (p.fixed[p.obs_kf[p.obs_mp == j]] == 1).all() and act[p.obs_mp == j].any()
    for name in B.SCENES:
        p = B.scene(name)
        L = F.Lin(p, delta=api.HUBER_GBA)
        act, _ = F.edge_flags(p)
        d = L.depth
        assert (d[p.special["far"]] > 1e3).all()
        assert (d[p.special["behind"]] < 0).all() and act[p.special["behind"]].all()
        d0 = p.special["depth0"]
        assert (~act[d0]).all() and set(d[d0].tolist()) == {0.0, 1e-300}
        assert set(p.obs_kf[d0].tolist()) == {0, B.DEPTH0_FREE_KF} and p.fixed[0] == 1 and p.fixed[B.DEPTH0_FREE_KF] == 0
        hd = np.abs(np.diagonal(L.Hll, axis1=1, axis2=2))
        far_lm = np.unique(p.obs_mp[p.special["far"]])
        assert hd[far_lm].max() < 1e-6 * L.max_diag()[0]
        # the Huber band, confirmed edge by edge, for both deltas and every target
        for delta in B.DELTAS:
            for lo, hi in B.band_targets(delta):
                assert sum(1 for _, dd, a, b in p.band if dd == delta and (a, b) == (lo, hi)) >= 2, (name, delta, lo, hi)
    p = B.scene("multicam")
    d = F.Lin(p, delta=api.HUBER_GBA).depth
    assert np.abs(d[p.special["near"]] - 0.05).max() < 1e-6
    assert F.Lin(p, delta=api.HUBER_GBA).max_diag()[2] == "Hll" and F.Lin(B.scene("sizes"), delta=api.HUBER_GBA).max_diag()[2] == "Hpp"
    # on sizes the depth-0 landmark and the band edges span more than one 128-observation chunk of k_linearize
    q = B.scene("sizes")
    n = np.bincount(q.obs_mp)
    assert n[q.special["depth0_landmark"]] > 128 and all(n[q.obs_mp[i]] > 128 for i, *_ in q.band)
    # landmark sizes around the chunks of k_linearize
    assert set(B.SPECIAL) <= set(np.bincount(B.scene("sizes").obs_mp).tolist())
    # the exp-map cases: every angle, every R_to_quat branch, and a product that needs the w < 0 flip
    x = F.exp_cases(p.K)
    th = np.linalg.norm(x[:, :3], axis=1)
    assert {float(t) for t in np.round(th, 17)} >= {float(np.round(t, 17)) for t in F.EXP_THETAS}
    branches, flips = set(), 0
    for k in range(p.K):
        for T in (p.poses[k], B.turned(p.poses)[k]):
            _, _, br, fl = F.se3_exp_times(x[k], T)
            branches.add(br); flips += fl
    assert branches == {-1, 0, 1, 2} and flips > 0


def test_sampled_edges_on_a_large_scene(oracle):
    """above ba_ref.MP_ALL edges the mpmath pass runs on a fixed sample plus the given edges; the vectorised terms of every edge
    and the sampled exact terms agree with the oracle (cfg3: 400 keyframes, two agents)"""
    q = synth.make_config("cfg3")
    assert q.E > F.MP_ALL
    special = np.arange(10)
    idx = F.sample_edges(q, special=special)
    assert len(idx) <= F.SAMPLE + len(special) and set(special) <= set(idx.tolist())
    ex, bd = F.mp_edges(q, idx)
    lin = oracle.ba_linearize(q, huber_delta=api.HUBER_GBA)
    L = F.Lin(q, delta=api.HUBER_GBA)
    r = dict(err=ratio(ex["err"] - lin["err"][idx], TAU * bd["err"]), Jp=ratio(ex["Jp"] - lin["Jpose"][idx], TAU * bd["Jp"]),
             Jl=ratio(ex["Jl"] - lin["Jpoint"][idx], TAU * bd["Jl"]), chi2=ratio(ex["chi2"] - lin["chi2"][idx], TAU * bd["chi2"]),
             chi2_all=ratio(L.chi2 - lin["chi2"], TAU * L.chi2_b),
             rho1=ratio(L.rho1 - lin["rho1"], TAU * L.rho1_b), Jp_all=ratio(L.Jp - lin["Jpose"], TAU * L.Jp_b),
             shadow=ratio(L.Jl[idx] - ex["Jl"], L.Jl_b[idx]))
    assert all(v <= 1.0 for v in r.values()), r

"""The single-vertex optimisations on the device, step by step (ccm_pose_optimize / ccm_sim3_optimize, csrc/single.cu): the per-edge
errors and Jacobians, the assembled 6x6 / 7x7 normal equation and its damped Cholesky solve against the 40-digit restatement of
tests/single_ref.py, and g2o's Levenberg protocol (lambda, trials, decisions, how every optimize() call ended, the cached errors
the classification reads) against the oracle's trace, on the scenes of tests/single_scenes.py."""
import numpy as np
import pytest

from ccm_slam_b200 import api
from tests import single_ref as SR
from tests import single_scenes as SS

pytestmark = pytest.mark.gpu
KINDS = ("pose", "sim3")
D_OF = {"pose": 6, "sim3": 7}
STATE = {"pose": "Tcw0", "sim3": "S12_0"}
# LM trace tolerances, relative, from measured values (printed by test_trace_matches_oracle): the pose problem follows the oracle
# to f64 rounding; the Sim3 problem's numeric Jacobians (delta 1e-9) carry ~1e-7 relative noise into H, b and every step.
# On an H100, 52 of the 62 pose calls and 26 of the 30 Sim3 calls reach the noise floor (chi2 gain < 1e-6) before they end; from
# there on a call is held to its iteration limit, its classification (rejected count) and a converged ending, not to the oracle's
# exact ending and iteration count.
TRACE_TOL = {"pose": 1e-9, "sim3": 1e-5}
RHO_FLOOR = 1e-9      # test_gpu_frontend / test_gpu_pgo: decisions are compared where |rho| is above this on both sides


@pytest.fixture(scope="module", autouse=True)
def _dev():
    assert api.device_count() > 0, "no CUDA device: the product path has no CPU fallback"
    api.init(0)


_SC = {}


def scenes(kind):
    if kind not in _SC:
        _SC[kind] = SS.pose_scenes() if kind == "pose" else SS.sim3_scenes()
    return _SC[kind]


def n_edges(kind, d):
    return len(d["Xw"]) if kind == "pose" else 2 * len(d["P1c"])


def oracle_run(oracle, kind, d):
    if kind == "pose":
        return oracle.pose_opt_trace(d["Tcw0"], d["Xw"], d["uv"], d["inv_sigma2"], d["intr"])
    return oracle.sim3_opt_trace(d["S12_0"], d["P1c"], d["P2c"], d["uv1"], d["uv2"], d["w1"], d["w2"], d["K1"], d["K2"], d["th2"],
                                 d["fix_scale"])


def restate(kind, d, state, active, robust, delta):
    return (SR.pose_system if kind == "pose" else SR.sim3_system)(d, state, active, robust, delta)


# ---- per-edge linearisation, H, b, chi2 and the damped solve --------------------------------------------------------------------
# far-measurement scenes (pose_stale, sim3_stale) exist for the protocol: a 1e25 px error has no use in a bound check
SYS_SKIP = ("pose_n0", "pose_n1", "pose_n2", "pose_depth_zero", "pose_weightless", "pose_n5000", "pose_stale", "sim3_n0", "sim3_n600",
            "sim3_stale")


def midway(kind, a, b):
    """the state halfway between a and b: rotation by normalised quaternion mean (same hemisphere), translation / scale averaged"""
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    qb = b[:4] if np.dot(a[:4], b[:4]) >= 0 else -b[:4]
    q = (a[:4] + qb) / np.linalg.norm(a[:4] + qb)
    return np.concatenate([q, (a[4:] + b[4:]) / 2])


@pytest.mark.parametrize("kind", KINDS)
def test_system_matches_restatement(oracle, kind, capsys):
    """every scene at its start, at a mid-run state (halfway to the oracle's end state) and at the oracle's end state; robust on,
    robust off, and a partial active mask with mixed robust flags; lambda = 1e-5 max diag H"""
    worst = dict(err=0.0, J=0.0, H=0.0, b=0.0, chi2=0.0, x=0.0)
    fs_checked = 0
    cases = []
    for d in scenes(kind):
        if d["name"] in SYS_SKIP:
            continue
        E = n_edges(kind, d)
        end = oracle_run(oracle, kind, d)[0]
        rng = np.random.default_rng(E)
        part = rng.random(E) < 0.7
        part[0] = True
        start = np.asarray(d[STATE[kind]], np.float64)
        for state in (start, midway(kind, start, end), end):
            for act, rob in ((np.ones(E, bool), np.ones(E, bool)), (np.ones(E, bool), np.zeros(E, bool)), (part, rng.random(E) < 0.5)):
                cases.append((d, state, act, rob))
    delta = lambda d: SR.POSE_DELTA if kind == "pose" else SR.sim3_delta(d)
    refs = [restate(kind, d, s, a, r, delta(d)) for d, s, a, r in cases]
    lams = [1e-5 * np.abs(np.diag(sy.H)).max() for _, sy in refs]
    got = api.single_debug_system(kind, [c[0] for c in cases], [c[1] for c in cases], [c[2] for c in cases], [c[3] for c in cases],
                                  [delta(c[0]) for c in cases], lams)
    for (d, state, act, rob), ((err, eb, J, Jb), sy), lam, g in zip(cases, refs, lams, got):
        worst["err"] = max(worst["err"], SR.ratio(g["err"] - err, SR.TAU * eb))
        worst["J"] = max(worst["J"], SR.ratio(g["J"] - J, SR.TAU * Jb))
        worst["H"] = max(worst["H"], SR.ratio(g["H"] - sy.H, SR.TAU * sy.H_bound))
        worst["b"] = max(worst["b"], SR.ratio(g["b"] - sy.b, SR.TAU * sy.b_bound))
        worst["chi2"] = max(worst["chi2"], abs(g["chi2"] - sy.chi2) / (SR.TAU * sy.chi2_bound))
        assert g["solved"], d["name"]
        xs, tol = SR.solve_bound(g["H"], g["b"], lam, g["x"])
        worst["x"] = max(worst["x"], np.abs(g["x"] - xs).max() / tol)
        if kind == "sim3" and d["fix_scale"]:
            fs_checked += 1
            assert not g["J"][:, :, 6].any(), (d["name"], "J column 6 under fix_scale")
            assert not g["H"][6, :].any() and not g["H"][:, 6].any() and g["b"][6] == 0 and g["x"][6] == 0, d["name"]
    with capsys.disabled():
        print(f"\n[single {kind} system] {len(cases)} cases, device error / bound: " + " ".join(f"{k} {v:.3g}" for k, v in worst.items()))
    assert all(v <= 1.0 for v in worst.values()), worst
    assert kind == "pose" or fs_checked > 0


@pytest.mark.parametrize("kind", KINDS)
def test_solve_refuses_an_indefinite_system(oracle, kind):
    """lambda below -min eig(H) makes H + lambda I indefinite: not solved and x = 0, as orc_chol_solve refuses it"""
    d = SS.by_name(scenes(kind))["pose_n11" if kind == "pose" else "sim3_two_cams"]
    E = n_edges(kind, d)
    st = np.asarray(d[STATE[kind]], np.float64)
    delta = SR.POSE_DELTA if kind == "pose" else SR.sim3_delta(d)
    g0 = api.single_debug_system(kind, [d], [st], [np.ones(E, bool)], [np.ones(E, bool)], [delta], [0.0])[0]
    D = D_OF[kind]
    ev = np.linalg.eigvalsh(g0["H"][:6, :6] if kind == "sim3" and d["fix_scale"] else g0["H"])
    lam = -0.5 * (ev[0] + ev[-1])
    g = api.single_debug_system(kind, [d], [st], [np.ones(E, bool)], [np.ones(E, bool)], [delta], [lam])[0]
    A = np.ascontiguousarray(g["H"] + lam * np.eye(D)); b = np.ascontiguousarray(g["b"]); x = np.zeros(D)
    rc = oracle.lib().orc_chol_solve(D, oracle._p(A), oracle._p(b), oracle._p(x))
    assert rc == 1 and not g["solved"] and not g["x"].any()


def test_depth_zero_system_is_nan_and_unsolved():
    """the point at camera depth 0: infinite error, NaN H and b, the factorisation fails and x = 0"""
    d = SS.pose_depth_zero()
    n = len(d["Xw"])
    g = api.single_debug_system("pose", [d], [d["Tcw0"]], [np.ones(n, bool)], [np.ones(n, bool)], [SR.POSE_DELTA], [1.0])[0]
    assert np.isinf(g["err"][0]).any() and np.isnan(g["H"]).all() and np.isinf(g["chi2"])
    assert not g["solved"] and not g["x"].any()
    assert np.isfinite(g["err"][1:]).all()


# ---- the Levenberg protocol against the oracle's trace ----------------------------------------------------------------------
def _close(a, b, tol):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    same_nan = np.isnan(a) == np.isnan(b)
    fin = ~np.isnan(a) & ~np.isnan(b)
    with np.errstate(invalid="ignore"):
        ok = np.where(fin, (a == b) | (np.abs(a - b) <= tol * np.maximum(np.abs(b), 1e-300)), True)
    return bool(same_nan.all() and ok.all())


def _device(kind, probs, trace=True):
    return (api.pose_optimize if kind == "pose" else api.sim3_optimize)(probs, trace=trace)


_RUNS = {}


def runs(oracle, kind):
    if kind not in _RUNS:
        sc = scenes(kind)
        _RUNS[kind] = (sc, _device(kind, sc), [oracle_run(oracle, kind, d) for d in sc])
    return _RUNS[kind]


@pytest.mark.parametrize("kind", KINDS)
def test_trace_matches_oracle(oracle, kind, capsys):
    sc, got, ref = runs(oracle, kind)
    tol = TRACE_TOL[kind]
    worst = dict(lam=0.0, chi=0.0, cached=0.0)
    n_calls = n_flat = n_stale = 0
    for d, g, r in zip(sc, got, ref):
        gc, rc = SR.parse_trace(g[3]), SR.parse_trace(r[3])
        assert [c is None for c in gc] == [c is None for c in rc], d["name"]
        for k, (a, b) in enumerate(zip(gc, rc)):
            if b is None:
                continue
            where = (d["name"], "call", k)
            n_calls += 1
            # the call's iteration limit (10; Sim3: 5, then 10 after a rejected pair and 5 without) and what the classification after
            # it rejects are exact.  A call whose first trial is rejected with rho == 0 (pose_stale, sim3_stale: a full step) leaves
            # every edge the step moved with the errors of that step: the number of stale edges is exact there, and a device that
            # classified from fresh errors would report none.  (At the noise floor a last rejected step is tiny: not compared.)
            assert a["limit"] == b["limit"] and a["rejected"] == b["rejected"], (where, a["limit"], b["limit"], a["rejected"], b["rejected"])
            if b["end"] == 2 and b["iters"] == 1:
                assert (a["end"], a["iters"], a["stale"]) == (2, 1, b["stale"]), (where, "stale cached errors", a, b["stale"])
                n_stale += b["stale"] > 0
            if b["end"] == -1:
                assert a["end"] == -1 and a["iters"] == -1, where
                continue
            # test_gpu_pgo's rule: iterations are compared up to the first one whose oracle step changes chi2 by less than 1e-6
            # relative.  From there on both runs sit at the minimum (an exactly determined frame reaches chi2 ~ 1e-25), the gain
            # ratios are rounding noise, and the call may end there by ten rejections, rho == 0 or three strikes on either side.
            # A call with fewer residuals than unknowns (one Sim3 pair; a frame left with one or two edges) has a singular H that
            # lambda alone regularises; its steps follow rounding noise, so it is held to the endings from its first iteration on.
            under = k >= d.get("underdetermined_from", 99)
            with np.errstate(invalid="ignore"):
                gain = b["rows"][:, 0] - b["rows"][:, 4]
                flat = np.flatnonzero((gain <= 1e-6 * b["rows"][:, 0] + 1e-12 * abs(b["rows"][0, 0])) | under)
            if flat.size:
                n_cmp = int(flat[0]) + 1
                n_flat += 1
                assert n_cmp <= a["iters"] <= a["limit"] and a["end"] in (0, 1, 2, 3), (where, a["end"], a["iters"], n_cmp)
            else:
                n_cmp = b["iters"]
                assert a["end"] == b["end"] and a["iters"] == b["iters"], (where, a["end"], b["end"], a["iters"], b["iters"])
            floor = 1e-12 * abs(b["rows"][0, 0]) if np.isfinite(b["rows"][0, 0]) else 0.0
            near = lambda x, y: _close(x, y, tol) or (np.isfinite(x) and np.isfinite(y) and abs(x - y) <= tol * abs(y) + floor)
            for it in range(n_cmp):
                ra, rb = a["rows"][it], b["rows"][it]
                if abs(ra[3]) > RHO_FLOOR and abs(rb[3]) > RHO_FLOOR:
                    assert ra[2] == rb[2] and ra[5] == rb[5], (where, it, ra, rb)
                if it < n_cmp - 1 or not flat.size:
                    assert ra[6] == rb[6], (where, it, "failed factorisations", ra[6], rb[6])
                    assert near(ra[4], rb[4]), (where, it, "currentChi", ra[4], rb[4])
                    worst["chi"] = max(worst["chi"], _rel(ra[4], rb[4]))
                assert _close(ra[1], rb[1], tol), (where, it, "lambda", ra[1], rb[1])
                assert near(ra[0], rb[0]), (where, it, "iniChi", ra[0], rb[0])
                worst["lam"] = max(worst["lam"], _rel(ra[1], rb[1]))
                worst["chi"] = max(worst["chi"], _rel(ra[0], rb[0]))
            assert near(a["cached"], b["cached"]), (where, "cached chi2", a["cached"], b["cached"])
            worst["cached"] = max(worst["cached"], _rel(a["cached"], b["cached"]))
    with capsys.disabled():
        print(f"\n[single {kind} trace] {len(sc)} scenes, {n_calls} calls ({n_flat} reach the noise floor, {n_stale} end with stale "
              "errors), largest relative difference to the oracle: " + " ".join(f"{k} {v:.3g}" for k, v in worst.items()))
    assert n_stale >= 1


def _rel(a, b):
    if a == b or (np.isnan(a) and np.isnan(b)):
        return 0.0
    return abs(a - b) / max(abs(b), 1e-300)


@pytest.mark.parametrize("kind", KINDS)
def test_outputs_match_oracle(oracle, kind):
    """flags and counts exact; estimates within 1e-8 (pose) / 1e-4 (Sim3) of the largest entry, untouched where the reference
    leaves them; the traced and the product kernels give the same bits"""
    sc, got, ref = runs(oracle, kind)
    plain = _device(kind, sc, trace=False)
    bar = 1e-8 if kind == "pose" else 1e-4
    for d, g, p, r in zip(sc, got, plain, ref):
        assert g[2] == r[2] and np.array_equal(g[1], r[1]), d["name"]
        assert np.abs(g[0] - r[0]).max() <= bar * max(1.0, np.abs(r[0]).max()), (d["name"], g[0], r[0])
        assert np.array_equal(g[0], p[0]) and np.array_equal(g[1], p[1]) and g[2] == p[2], d["name"]
        if kind == "sim3" and d["fix_scale"]:
            assert g[0][7] == d["S12_0"][7]
        if r[2] == 0 and (kind == "sim3" or len(d["Xw"]) < 3):
            assert np.array_equal(g[0], d[STATE[kind]]), d["name"]


def test_trace_covers_the_endings(oracle):
    """every way an optimize() call can end is reached on the device by the pose problem (a pose round with no active edge
    included) and by the Sim3 problem except ten rejections; a Cholesky factorisation fails; and in both problems a classification
    reads stale errors on nearly every edge, on the device as on the oracle"""
    for kind in KINDS:
        ends, fails, stale = set(), 0, []
        sc, got, ref = runs(oracle, kind)
        for d, g, r in zip(sc, got, ref):
            for c, rc in zip(SR.parse_trace(g[3]), SR.parse_trace(r[3])):
                if c is None:
                    continue
                ends.add(c["end"])
                fails += int(np.nansum(c["rows"][:, 6])) if len(c["rows"]) else 0
                if rc["stale"] >= 0.9 * n_edges(kind, d):
                    stale.append((d["name"], rc["stale"], c["stale"]))
        want = set(SR.ENDS) if kind == "pose" else set(SR.ENDS) - {1}
        assert ends >= want, (kind, {SR.ENDS[e] for e in want - ends})
        assert stale and all(a == b for _, a, b in stale), (kind, stale)
        assert kind == "sim3" or fails > 0


def test_lambda_init_keeps_nan(oracle):
    """std::max(fabs(H_ii), maxd) keeps a NaN diagonal: on the depth-0 frame lambda is NaN on the device as on the oracle"""
    d = SS.pose_depth_zero()
    g = SR.parse_trace(api.pose_optimize([d], trace=True)[0][3])[0]
    r = SR.parse_trace(oracle_run(oracle, "pose", d)[3])[0]
    assert np.isnan(r["rows"][0, 1]) and np.isnan(g["rows"][0, 1])
    assert np.all(g["rows"][:, 6] == 1) and g["end"] == 0 and g["iters"] == 10


# ---- batches --------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", KINDS)
def test_batch_independent_of_neighbours(kind):
    """about 300 problems (more CTAs than SMs) holding every scene: each result is bit-identical alone, inside the batch and in
    the reversed batch"""
    sc = scenes(kind)
    extra = [SS.pose_size(n, seed=5000 + k) for k, n in enumerate(np.random.default_rng(1).integers(3, 400, 300 - len(sc)))] \
        if kind == "pose" else \
        [SS._sim3(f"x{k}", n=int(n), seed=7000 + k) for k, n in enumerate(np.random.default_rng(2).integers(5, 200, 300 - len(sc)))]
    batch = sc + extra
    fwd = _device(kind, batch, trace=False)
    rev = _device(kind, batch[::-1], trace=False)[::-1]
    same = lambda a, b: np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1]) and a[2] == b[2]
    for k, d in enumerate(batch):
        assert same(fwd[k], rev[k]), (d["name"], "reversed batch")
    for k, d in enumerate(sc):      # every scene alone (a batch of one; Sim3 included)
        assert same(fwd[k], _device(kind, [d], trace=False)[0]), (d["name"], "alone")
    assert _device(kind, [], trace=False) == [] and _device(kind, [], trace=True) == []
    assert api.single_debug_system(kind, [], [], [], [], [], []) == []


# ---- ABI ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", KINDS)
def test_abi_refuses_bad_arguments(kind):
    d = SS.by_name(scenes(kind))["pose_n11" if kind == "pose" else "sim3_n10"]
    L = api.lib()
    for mod in ("n", "null"):
        probs, res, keep = (api._pose_probs if kind == "pose" else api._sim3_probs)([d])
        if mod == "n":
            probs[0].n = -1
        elif kind == "pose":
            probs[0].Xw = None
        else:
            probs[0].P2c = None
        for f in ((L.ccm_pose_optimize if kind == "pose" else L.ccm_sim3_optimize),):
            with pytest.raises(api.CCMError):
                api._chk(f(probs, 1, res))
        tr = np.empty((1, api.SINGLE_TRACE_CALLS[kind], api.SINGLE_TRACE_CALL))
        with pytest.raises(api.CCMError):
            api._chk((L.ccm_pose_optimize_traced if kind == "pose" else L.ccm_sim3_optimize_traced)(probs, 1, res, api._p(tr)))
        dl = np.array([[1.0, 1.0]])
        with pytest.raises(api.CCMError):
            api._chk((L.ccm_pose_debug_system if kind == "pose" else L.ccm_sim3_debug_system)(probs, 1, None, None, api._p(dl), None, None,
                                                                                                  None, None))
    with pytest.raises(api.CCMError):
        api._chk((L.ccm_pose_optimize if kind == "pose" else L.ccm_sim3_optimize)(None, 1, None))
    probs, res, keep = (api._pose_probs if kind == "pose" else api._sim3_probs)([d])
    with pytest.raises(api.CCMError):       # a traced run without a trace buffer
        api._chk((L.ccm_pose_optimize_traced if kind == "pose" else L.ccm_sim3_optimize_traced)(probs, 1, res, None))
    ok = _device(kind, [d], trace=False)[0]          # still usable
    assert ok[2] > 0

"""The restatement of tests/single_ref.py against the oracle (orc_pose_opt_build / orc_sim3_opt_build: H, b and the per-edge
errors) on every scene of tests/single_scenes.py, and every deliberate defect of single_ref.MUT pushed far outside its bound.
Also: the oracle's LM trace only observes (the traced protocol gives the results of the plain one) and reaches every ending."""
import numpy as np
import pytest

from tests import single_ref as SR
from tests import single_scenes as SS

# the far-measurement scenes exist for the protocol (their 1e25 px error has no use in a bound check)
SKIP = ("pose_n0", "pose_n1", "pose_n2", "pose_depth_zero", "pose_n5000", "pose_stale", "sim3_n0", "sim3_n600", "sim3_stale")


def _oracle_build(P, kind, d, state, robust, delta):
    if kind == "pose":
        return P.pose_opt_build(state, d["Xw"], d["uv"], d["inv_sigma2"], d["intr"], robust, delta)
    return P.sim3_opt_build(state, d["P1c"], d["P2c"], d["uv1"], d["uv2"], d["w1"], d["w2"], d["K1"], d["K2"], d["fix_scale"], robust, delta)


def _worst(oracle, kind, names=None):
    P = oracle.Pieces("oracle")
    sc = SS.pose_scenes() if kind == "pose" else SS.sim3_scenes()
    worst = dict(err=0.0, H=0.0, b=0.0)
    for d in sc:
        if d["name"] in SKIP or (names and d["name"] not in names):
            continue
        st = np.asarray(d["Tcw0"] if kind == "pose" else d["S12_0"], np.float64)
        delta = SR.POSE_DELTA if kind == "pose" else SR.sim3_delta(d)
        for robust in (True, False):
            E = len(d["Xw"]) if kind == "pose" else 2 * len(d["P1c"])
            (err, eb, J, Jb), sy = (SR.pose_system if kind == "pose" else SR.sim3_system)(d, st, np.ones(E, bool), np.full(E, robust), delta)
            H, b, oerr = _oracle_build(P, kind, d, st, robust, delta)
            worst["err"] = max(worst["err"], SR.ratio(oerr - err, SR.TAU * eb))
            worst["H"] = max(worst["H"], SR.ratio(H - sy.H, SR.TAU * sy.H_bound))
            worst["b"] = max(worst["b"], SR.ratio(b - sy.b, SR.TAU * sy.b_bound))
            if kind == "sim3" and d["fix_scale"]:
                assert not H[6].any() and not H[:, 6].any() and b[6] == 0
    return worst


@pytest.mark.parametrize("kind", ["pose", "sim3"])
def test_oracle_inside_restated_bounds(oracle, kind, capsys):
    w = _worst(oracle, kind)
    with capsys.disabled():
        print(f"\n[single_ref {kind}] oracle error / bound: " + " ".join(f"{k} {v:.3g}" for k, v in w.items()))
    assert all(v <= 1.0 for v in w.values()), w


# (switch, kind, scenes): each defect is seen on scenes that exercise it -- two cameras, outliers beyond the Huber threshold, fix_scale
MUTATIONS = [("k_swap", "sim3", ("sim3_two_cams",)), ("huber_b", "pose", ("pose_n11", "pose_bad_start")),
             ("huber_b", "sim3", ("sim3_two_cams",)), ("jac_sign", "pose", ("pose_n11",)), ("jac_sign", "sim3", ("sim3_n10",)),
             ("no_fix_scale", "sim3", ("sim3_two_cams_fix",))]


@pytest.mark.parametrize("switch,kind,names", MUTATIONS, ids=[f"{m[0]}-{m[1]}" for m in MUTATIONS])
def test_mutation_leaves_the_bound(oracle, monkeypatch, switch, kind, names):
    monkeypatch.setitem(SR.MUT, switch, True)
    w = _worst(oracle, kind, names)
    assert max(w.values()) > 1e3, (switch, w)


def _stale_round_disagreement(oracle):
    """how far the restated round-1 classification of pose_stale is from the oracle's trace: |stale diff| + |rejected diff|"""
    d = SS.pose_stale()
    c = SR.parse_trace(oracle.pose_opt_trace(d["Tcw0"], d["Xw"], d["uv"], d["inv_sigma2"], d["intr"])[3])[0]
    assert c["end"] == 2 and c["iters"] == 1      # one rejected full step, rho == 0: the cached errors are that step's
    stale, rejected = SR.pose_first_round_classification(d, oracle)
    return abs(stale - c["stale"]) + abs(rejected - c["rejected"]), c


def test_classification_reads_cached_errors(oracle):
    """round 1 of pose_stale ends on a rejected full step: the oracle's classification reads that step's errors (nearly every edge
    stale) and rejects exactly the edges the restatement rejects from them"""
    diff, c = _stale_round_disagreement(oracle)
    assert diff == 0 and c["stale"] >= 0.9 * len(SS.pose_stale()["Xw"]), c


def test_mutation_fresh_errors_disagrees(oracle, monkeypatch):
    monkeypatch.setitem(SR.MUT, "fresh_errors", True)
    diff, c = _stale_round_disagreement(oracle)
    assert diff >= 50, (diff, c)


def test_mutations_cover_the_switches():
    assert {m[0] for m in MUTATIONS} | {"fresh_errors"} == set(SR.MUT)


@pytest.mark.parametrize("kind", ["pose", "sim3"])
def test_oracle_trace_only_observes(oracle, kind):
    """the traced protocol returns exactly what the plain one returns, and its calls reach every ending"""
    ends, fails = set(), 0
    for d in (SS.pose_scenes() if kind == "pose" else SS.sim3_scenes()):
        if kind == "pose":
            a = oracle.pose_optimize(d["Tcw0"], d["Xw"], d["uv"], d["inv_sigma2"], d["intr"])
            b = oracle.pose_opt_trace(d["Tcw0"], d["Xw"], d["uv"], d["inv_sigma2"], d["intr"])
        else:
            args = (d["S12_0"], d["P1c"], d["P2c"], d["uv1"], d["uv2"], d["w1"], d["w2"], d["K1"], d["K2"], d["th2"], d["fix_scale"])
            a, b = oracle.sim3_optimize(*args), oracle.sim3_opt_trace(*args)
        assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1]) and a[2] == b[2], d["name"]
        for c in SR.parse_trace(b[3]):
            if c is not None:
                ends.add(c["end"])
                fails += int(c["rows"][:, 6].sum()) if len(c["rows"]) else 0
                assert len(c["rows"]) == max(c["iters"], 0)
    if kind == "pose":
        assert ends == set(SR.ENDS) and fails > 0, ends

"""A high-precision restatement of the single-vertex optimisations' edges and normal equation (test infrastructure).

* EdgeSE3ProjectXYZOnlyPose (types_six_dof_expmap.h:153-157, .cpp:266-288): the error and the analytic Jacobian, evaluated with
  sim3_ref's `R` (exact value in mpmath at 40 digits, f64 shadow, first-order rounding bound) on the exact values of the f64 / f32
  inputs.
* EdgeSim3ProjectXYZ / EdgeInverseSim3ProjectXYZ (types_seven_dof_expmap.h:130-172): the error, and the central difference at
  delta = 1e-9 (base_binary_edge.hpp:131-205) over the 14 states displaced by +-delta along each coordinate through sim3_ref's
  s3_oplus (so the displaced states carry their own rounding bound).  The Jacobian's bound is (e(e+) + e(e-)) / (2 delta).
  Edge 2i is the forward edge of pair i, 2i+1 the inverse edge, as in the device's Sim3M.
* The normal equation in f64 from those edges: H = sum wo J^T J, b = -sum wr w J^T e, the robust chi2, with the Huber weights as
  g2o applies them (dsqr kept in a float) and a bound for every entry that covers the rounding of the edges, of the weights and of
  any order of the f64 summation -- both the device's binary grouping of b and the oracle's BaseUnaryEdge grouping.

A comparison passes when |got - exact| <= TAU * bound entry by entry (sim3_ref.ratio).
"""
from __future__ import annotations

import numpy as np

from tests import sim3_ref as S
from tests.sim3_ref import R, U, TAU, DELTA, ratio   # noqa: F401  (re-exported for the tests)

# Deliberate defects for the mutation tests (tests/test_single_ref.py): each must push the restatement far outside its bound
# against the oracle, or make the restated classification disagree with the oracle's.  All False in normal use.
MUT = dict(k_swap=False, huber_b=False, jac_sign=False, no_fix_scale=False, fresh_errors=False)


def _r(x):
    return R(float(x))


def _vals(xs):
    return np.array([float(x.v) for x in xs])


def _bnds(xs):
    return np.array([x.e for x in xs])


# ---- pose edge -----------------------------------------------------------------------------------------------------------------
def pose_edge(T, X, uv, intr):
    """exact error (2,), J (2,6) of EdgeSE3ProjectXYZOnlyPose at the pose row T (qx qy qz qw tx ty tz) and their bounds"""
    q = [_r(v) for v in T[:4]]
    xc = S.quat_rotate(q, [_r(v) for v in X])
    x, y, z = [xc[k] + _r(T[4 + k]) for k in range(3)]
    fx, fy, cx, cy = [_r(v) for v in intr]
    e = [_r(uv[0]) - (x / z * fx + cx), _r(uv[1]) - (y / z * fy + cy)]
    invz = 1.0 / z
    invz_2 = invz * invz
    zero = R(0.0)
    J = [x * y * invz_2 * fx, -(1 + (x * x * invz_2)) * fx, y * invz * fx, -invz * fx, zero, x * invz_2 * fx,
         (1 + y * y * invz_2) * fy, -x * y * invz_2 * fy, -x * invz * fy, zero, -invz * fy, y * invz_2 * fy]
    Jv, Jb = _vals(J).reshape(2, 6), _bnds(J).reshape(2, 6)
    if MUT["jac_sign"]:
        Jv[1] = -Jv[1]
    return _vals(e), _bnds(e), Jv, Jb


def pose_edges(d, T, edges=None):
    """restated errors and Jacobians of the edges of pose problem d at T: err (E,2), err_bound, J (E,2,6), J_bound"""
    idx = range(len(d["Xw"])) if edges is None else edges
    out = [pose_edge(T, d["Xw"][e], d["uv"][e], d["intr"]) for e in idx]
    if not out:
        return np.zeros((0, 2)), np.zeros((0, 2)), np.zeros((0, 2, 6)), np.zeros((0, 2, 6))
    return tuple(np.array([o[k] for o in out]) for k in range(4))


# ---- Sim3 edges ----------------------------------------------------------------------------------------------------------------
def _proj_err(Sst, P, uv, K):
    p = S.quat_rotate(Sst[:4], [_r(v) for v in P])
    x, y, z = [Sst[7] * p[k] + Sst[4 + k] for k in range(3)]
    fx, fy, cx, cy = [_r(v) for v in K]
    return [_r(uv[0]) - (x / z * fx + cx), _r(uv[1]) - (y / z * fy + cy)]


def sim3_edges(d, S12, pairs=None):
    """restated errors and central-difference Jacobians of the edges of Sim3 problem d at S12 (row qx qy qz qw tx ty tz s):
    err (E,2), err_bound, J (E,2,7), J_bound with E = 2 * len(pairs), edge 2k the forward and 2k+1 the inverse edge of pairs[k]"""
    fs = bool(d["fix_scale"]) and not MUT["no_fix_scale"]
    st = S.s3(S12)
    pert = []
    for k in range(7):
        for sg in (1.0, -1.0):
            u = [R(0.0)] * 7
            u[k] = R(sg * DELTA)
            pert.append(S.s3_oplus(st, u, fs))
    inv = [S.s3_inv(p) for p in [st] + pert]
    K1, K2 = d["K1"], d["K2"]
    if MUT["k_swap"]:
        K2 = K1
    scalar = R(1.0 / (2 * DELTA))
    idx = range(len(d["P1c"])) if pairs is None else pairs
    err, eb, J, Jb = [], [], [], []
    for i in idx:
        for fwd in (True, False):
            f = (lambda s: _proj_err(s, d["P2c"][i], d["uv1"][i], K1)) if fwd else (lambda s: _proj_err(s, d["P1c"][i], d["uv2"][i], K2))
            states = [st] + pert if fwd else inv
            e0 = f(states[0])
            Jv, Jbd = np.zeros((2, 7)), np.zeros((2, 7))
            for k in range(7):
                if k == 6 and fs:
                    continue    # oplus zeroes u[6]: e+ and e- are the same f64 computation, their difference is exactly zero
                ep, em = f(states[1 + 2 * k]), f(states[2 + 2 * k])
                for r in range(2):
                    j = scalar * (ep[r] - em[r])
                    Jv[r, k], Jbd[r, k] = float(j.v), j.e
            if MUT["jac_sign"]:
                Jv[1] = -Jv[1]
            err.append(_vals(e0)); eb.append(_bnds(e0)); J.append(Jv); Jb.append(Jbd)
    if not err:
        return np.zeros((0, 2)), np.zeros((0, 2)), np.zeros((0, 2, 7)), np.zeros((0, 2, 7))
    return np.array(err), np.array(eb), np.array(J), np.array(Jb)


def edge_weights(d, kind):
    if kind == "pose":
        return np.asarray(d["inv_sigma2"], np.float32).astype(np.float64)
    w = np.empty(2 * len(d["w1"]))
    w[0::2] = np.asarray(d["w1"], np.float32); w[1::2] = np.asarray(d["w2"], np.float32)
    return w


# ---- the normal equation -------------------------------------------------------------------------------------------------------
class System:
    """H (D x D, without lambda), b (D) and the robust chi2 over the active edges, assembled in f64 from restated edges, with a bound
    per entry.  err, eb (E,2), J, Jb (E,2,D), w (E,), active / robust (E,) bool, delta the Huber delta (g2o keeps delta^2 in a
    float)."""

    def __init__(self, err, eb, J, Jb, w, active, robust, delta):
        a = np.asarray(active, bool)
        e, de, J, dJ, w = err[a], eb[a], J[a], Jb[a], np.asarray(w, np.float64)[a]
        rob = np.asarray(robust, bool)[a]
        D = J.shape[-1]
        n = len(e)
        c = w * (e * e).sum(1)
        dc = w * (2 * (np.abs(e) * de).sum(1) + de.sum(1) ** 2) + 4 * U * c
        dsqr = float(np.float32(delta * delta))
        out = rob & (c > dsqr)
        sq = np.sqrt(np.where(out, c, 1.0))
        rho0 = np.where(out, 2 * sq * delta - dsqr, c)
        drho0 = np.where(out, delta * dc / sq + 4 * U * (2 * sq * delta + dsqr), dc)
        rho1 = np.where(out, delta / sq, 1.0)
        drho1 = np.where(out, rho1 * (0.5 * dc / np.where(out, c, 1.0) + 4 * U), 0.0)
        wo, dwo = rho1 * w, drho1 * w + U * rho1 * w
        wb = w if MUT["huber_b"] else wo                       # the weight of b: rho1 * w, or w alone in the mutation
        A = np.abs(J)
        outer = lambda X, Y: np.einsum("eki,ekj->eij", X, Y)
        self.H = np.einsum("e,eij->ij", wo, outer(J, J))
        self.H_bound = (np.einsum("e,eij->ij", wo, outer(A, dJ) + outer(dJ, A) + outer(dJ, dJ)) + np.einsum("e,eij->ij", dwo, outer(A, A))
                        + (8 + n) * U * np.einsum("e,eij->ij", wo, outer(A, A)))
        self.b = -np.einsum("e,eki,ek->i", wb, J, e)
        ae = np.abs(e)
        self.b_bound = (np.einsum("e,eki,ek->i", wo, A, de) + np.einsum("e,eki,ek->i", wo, dJ, ae) + np.einsum("e,eki,ek->i", dwo, A, ae)
                        + (8 + n) * U * np.einsum("e,eki,ek->i", wo, A, ae))
        self.chi2 = float(rho0.sum())
        self.chi2_bound = float(drho0.sum() + (2 + n) * U * np.abs(rho0).sum())
        self.D = D


def pose_system(d, T, active=None, robust=None, delta=None):
    n = len(d["Xw"])
    err, eb, J, Jb = pose_edges(d, T)
    act = np.ones(n, bool) if active is None else active
    rob = np.ones(n, bool) if robust is None else robust
    return (err, eb, J, Jb), System(err, eb, J, Jb, edge_weights(d, "pose"), act, rob, POSE_DELTA if delta is None else delta)


def sim3_system(d, S12, active=None, robust=None, delta=None):
    E = 2 * len(d["P1c"])
    err, eb, J, Jb = sim3_edges(d, S12)
    act = np.ones(E, bool) if active is None else active
    rob = np.ones(E, bool) if robust is None else robust
    return (err, eb, J, Jb), System(err, eb, J, Jb, edge_weights(d, "sim3"), act, rob, sim3_delta(d) if delta is None else delta)


POSE_DELTA = float(np.float32(np.sqrt(5.991)))        # const float deltaMono = sqrt(5.991)


def sim3_delta(d):
    return float(np.sqrt(np.float32(d["th2"]), dtype=np.float32))   # const float deltaHuber = sqrt(th2)


def solve_bound(H, b, lam, x):
    """|x - solve(H + lam I, b)| tolerance for an f64 Cholesky solve: TAU * D u cond(H + lam I) |x|_max (infinity norm)"""
    A = H + lam * np.eye(len(b))
    Ai = np.linalg.inv(A)
    cond = np.abs(A).sum(1).max() * np.abs(Ai).sum(1).max()
    xs = np.linalg.solve(A, b)
    return xs, TAU * len(b) * U * cond * max(np.abs(xs).max(), 1e-300)


# ---- the LM protocol's classification -----------------------------------------------------------------------------------------
TRACE_HEAD, TRACE_ITERS, TRACE_COLS = 7, 10, 7
TRACE_ROW = ("iniChi", "lambda", "trials", "rho", "currentChi", "accepted", "chol_fail")
ENDS = {0: "iteration limit", 1: "ten rejections", 2: "rho == 0", 3: "three strikes", -1: "no active edge"}


def parse_trace(tr):
    """one problem's raw trace (calls, 77) -> list of calls dict(end, iters, limit, cached, fresh, stale, rejected, rows (iters, 7));
    None for a call that did not happen"""
    out = []
    for c in np.asarray(tr):
        if np.isnan(c[0]):
            out.append(None)
            continue
        it = int(c[1])
        rows = c[TRACE_HEAD:].reshape(TRACE_ITERS, TRACE_COLS)[:max(it, 0)]
        out.append(dict(end=int(c[0]), iters=it, limit=int(c[2]), cached=c[3], fresh=c[4], stale=int(c[5]), rejected=int(c[6]), rows=rows))
    return out



# ---- the first round of PoseOptimizationClient on a frame whose first trial is rejected with rho == 0 -------------------------
def pose_first_round_classification(d, oracle):
    """(stale, rejected) of round 1 of PoseOptimizationClient on a frame whose first call ends after one rejected trial
    (single_scenes.pose_stale: tempChi == currentChi).  The trial state is exp(x) * T0 with x = (H + lambda0 I)^-1 b from the
    restated system at T0 (every edge active and robust, lambda0 = 1e-5 max diag H; exp and product are the oracle's SE3Quat).
    g2o's classification reads the errors cached at that trial state: `stale` counts the edges whose trial-state error differs
    from the error at T0, `rejected` the edges whose float chi2 exceeds 5.991.  MUT["fresh_errors"] classifies from errors
    recomputed at the estimate, T0, instead."""
    T0 = np.asarray(d["Tcw0"], np.float64)
    (err0, _, _, _), sy = pose_system(d, T0)
    lam = 1e-5 * np.abs(np.diag(sy.H)).max()
    x = np.linalg.solve(sy.H + lam * np.eye(6), sy.b)
    T1 = oracle.se3_mul(oracle.se3_exp(x), T0)
    err1 = pose_edges(d, T1)[0]
    cached = err0 if MUT["fresh_errors"] else err1
    w = edge_weights(d, "pose")
    with np.errstate(over="ignore"):      # the far edge's chi2 is infinite as a float, as in g2o's (float) e->chi2()
        chi2 = (cached[:, 0] * (w * cached[:, 0]) + cached[:, 1] * (w * cached[:, 1])).astype(np.float32)
    stale = int(np.count_nonzero((cached != err0).any(1)))
    return stale, int(np.count_nonzero(chi2 > np.float32(5.991)))

"""A high-precision restatement of g2o's Sim3 (G/types/sim3.h) and of the essential graph's linear system (test infrastructure).

Two layers:

* Sim3 exp / log / product / inverse / oplus and the EdgeSim3 error log(C * Si * Sj^-1), evaluated in mpmath at 40 digits on the
  exact values of f64 inputs, with g2o's quirks kept: R = I + Omega + Omega^2 for theta < 1e-5, both branches of the A, B, C
  coefficients, the log's (B Omega) Omega, W.lu().solve(t) with partial pivoting.  Every number is an `R`: the exact value of the
  formula (`v`), the f64 value the same operations give in order (`f`: every branch is taken on it, as the f64 code decides), and a
  first-order bound on the rounding of any f64 evaluation of the formula (`e`: each operation adds u (|a| + |b|) or u |result|,
  libm / libdevice functions 4 u, and propagates its inputs' bounds through its derivative).  The numeric Jacobian is the central
  difference at delta = 1e-9 of that restated error, so its exact value is the exact value of the formula the device evaluates and
  its bound is (e(e+) + e(e-)) / (2 delta): the rounding of the magnitudes that cancel inside C * Si * Sj^-1, over delta.

* The f64 assembly of H, b and chi2 in free-vertex block CSR from per-edge Jacobians (numpy; the oracle's pgo_edge_jacobian, which
  the suite pins bit for bit to the reference's g2o, supplies them), with a bound for every entry.  A Jacobian entry's bound is
  EDGE_OPS u M_e / delta with M_e = 1 + |t_C| + s_C |t_i| + s_C s_i |t_j| / s_j (the translations that cancel in the edge error;
  edge_magnitude adds the log's large-angle conditioning) -- zero for a
  fixed side and, under fix_scale, for the scale column, which any implementation must return as exact zeros.  H and b take it
  through |J|^T dJ + dJ^T |J| (+ dJ^T dJ) summed over the edges of the block, plus the f64 summation of the products.

A comparison passes when |got - exact| <= TAU * bound entry by entry (`ratio`); an entry whose bound is zero must be exactly zero.
"""
from __future__ import annotations

import math

import mpmath as mp
import numpy as np

mp.mp.dps = 40
U = 2.0 ** -53          # unit roundoff of f64
UF = 4 * U              # one libm / libdevice call (sin, cos, acos, log, exp, sqrt): correctly rounded to within 2 ulp
TAU = 16.0
DELTA = 1e-9
# The closed-form per-edge bound is EDGE_OPS u M_e (/ delta for a Jacobian).  The oracle's error and Jacobians stay within 2.3 u M_e
# (/ delta) of the exact values on the sampled scene edges; tests/test_sim3_ref.py checks that they stay within TAU times the bound.
# (The running bound of the restatement is a worst case over every rounding and runs ~100x wider: too wide to see a mirrored block.)
EDGE_OPS = 4.0
EPS_BRANCH = 0.00001    # the 1e-5 of every g2o Sim3 branch
LOG_SMALL_ANGLE = math.acos(1 - EPS_BRANCH)   # the log's d > 1 - 1e-5 in terms of the angle

# Deliberate defects for the mutation tests (tests/test_sim3_ref.py): each must make the restatement disagree with the oracle by far
# more than its bound.  All False in normal use.
MUT = dict(abc_swap=False, exp_half=False, no_fix_scale=False, swap_jac=False, mirror_no_transpose=False, fixed_side=False)


class R:
    """exact value v (mpf), f64 shadow f (float), rounding bound e (float)"""
    __slots__ = ("v", "f", "e")

    def __init__(self, v, f=None, e=0.0):
        if isinstance(v, R):
            self.v, self.f, self.e = v.v, v.f, v.e
            return
        self.v = mp.mpf(v)
        self.f = float(v) if f is None else f
        self.e = e

    @staticmethod
    def _c(x):
        return x if isinstance(x, R) else R(x)

    def __add__(self, o):
        o = R._c(o)
        return R(self.v + o.v, self.f + o.f, self.e + o.e + U * (abs(self.f) + abs(o.f)))
    __radd__ = __add__

    def __sub__(self, o):
        o = R._c(o)
        return R(self.v - o.v, self.f - o.f, self.e + o.e + U * (abs(self.f) + abs(o.f)))

    def __rsub__(self, o):
        return R._c(o) - self

    def __neg__(self):
        return R(-self.v, -self.f, self.e)

    def __mul__(self, o):
        o = R._c(o)
        r = self.v * o.v
        return R(r, self.f * o.f, abs(self.f) * o.e + abs(o.f) * self.e + self.e * o.e + U * abs(float(r)))
    __rmul__ = __mul__

    def __truediv__(self, o):
        o = R._c(o)
        r = self.v / o.v
        den = max(abs(o.f) - o.e, abs(o.f) * 0.5)
        return R(r, self.f / o.f, (self.e + abs(float(r)) * o.e) / den + U * abs(float(r)))

    def __rtruediv__(self, o):
        return R._c(o) / self

    def __abs__(self):
        return R(abs(self.v), abs(self.f), self.e)


def _fn(x, fv, f64, deriv):
    r = fv(x.v)
    return R(r, f64(x.f), abs(deriv) * x.e + UF * abs(float(r)))


def sqrt(x):
    r = mp.sqrt(x.v)
    rf = float(r)
    return R(r, math.sqrt(x.f), (x.e / (2 * rf) if rf > 0 and x.e < x.f else math.sqrt(x.e)) + UF * rf)


def sin(x): return _fn(x, mp.sin, math.sin, 1.0)
def cos(x): return _fn(x, mp.cos, math.cos, 1.0)
def exp(x): return _fn(x, mp.exp, math.exp, math.exp(x.f))
def log(x): return _fn(x, mp.log, math.log, 1.0 / abs(x.f))


def acos(x):
    r = mp.acos(x.v)
    return R(r, math.acos(x.f), x.e / math.sqrt(max(1.0 - x.f * x.f, 1e-300)) + UF * abs(float(r)))


# ---- Sim3 (rows: qx qy qz qw tx ty tz s) -----------------------------------------------------------------------------------
def s3(row):
    return [R(float(v)) for v in row]


def values(xs):
    return np.array([float(x.v) for x in xs])


def bounds(xs):
    return np.array([x.e for x in xs])


def quat_rotate(q, v):
    qx, qy, qz, qw = q
    vx, vy, vz = v
    ux, uy, uz = qy * vz - qz * vy, qz * vx - qx * vz, qx * vy - qy * vx
    ux, uy, uz = ux + ux, uy + uy, uz + uz
    return [vx + qw * ux + (qy * uz - qz * uy), vy + qw * uy + (qz * ux - qx * uz), vz + qw * uz + (qx * uy - qy * ux)]


def s3_mul(a, b):                                   # sim3.h:266-272
    ax, ay, az, aw = a[:4]
    bx, by, bz, bw = b[:4]
    qw = aw * bw - ax * bx - ay * by - az * bz
    qx = aw * bx + ax * bw + ay * bz - az * by
    qy = aw * by + ay * bw + az * bx - ax * bz
    qz = aw * bz + az * bw + ax * by - ay * bx
    r = quat_rotate(a[:4], b[4:7])
    return [qx, qy, qz, qw] + [a[7] * r[k] + a[4 + k] for k in range(3)] + [a[7] * b[7]]


def s3_inv(a):                                      # sim3.h:233-236
    q = [-a[0], -a[1], -a[2], a[3]]
    k = -1.0 / a[7]
    return q + quat_rotate(q, [k * a[4], k * a[5], k * a[6]]) + [1.0 / a[7]]


def quat_to_R(q):
    x, y, z, w = q
    tx, ty, tz = 2 * x, 2 * y, 2 * z
    twx, twy, twz = tx * w, ty * w, tz * w
    txx, txy, txz = tx * x, ty * x, tz * x
    tyy, tyz, tzz = ty * y, tz * y, tz * z
    return [1 - (tyy + tzz), txy - twz, txz + twy, txy + twz, 1 - (txx + tzz), tyz - twx, txz - twy, tyz + twx, 1 - (txx + tyy)]


def R_to_quat(Rm):                                  # Eigen's Quaterniond(Matrix3d) branches
    t = Rm[0] + Rm[4] + Rm[8]
    if t.f > 0:
        t = sqrt(t + 1.0)
        w = 0.5 * t
        t = 0.5 / t
        return [(Rm[7] - Rm[5]) * t, (Rm[2] - Rm[6]) * t, (Rm[3] - Rm[1]) * t, w]
    if Rm[0].f >= Rm[4].f and Rm[0].f >= Rm[8].f:
        t = sqrt(Rm[0] - Rm[4] - Rm[8] + 1.0)
        x = 0.5 * t; t = 0.5 / t
        return [x, (Rm[3] + Rm[1]) * t, (Rm[6] + Rm[2]) * t, (Rm[7] - Rm[5]) * t]
    if Rm[4].f > Rm[0].f and Rm[4].f >= Rm[8].f:
        t = sqrt(Rm[4] - Rm[8] - Rm[0] + 1.0)
        y = 0.5 * t; t = 0.5 / t
        return [(Rm[1] + Rm[3]) * t, y, (Rm[7] + Rm[5]) * t, (Rm[2] - Rm[6]) * t]
    t = sqrt(Rm[8] - Rm[0] - Rm[4] + 1.0)
    z = 0.5 * t; t = 0.5 / t
    return [(Rm[2] + Rm[6]) * t, (Rm[5] + Rm[7]) * t, z, (Rm[3] - Rm[1]) * t]


def _skew(o):
    z = R(0.0)
    return [z, -o[2], o[1], o[2], z, -o[0], -o[1], o[0], z]


def _matmul3(A, B):
    return [A[3 * i] * B[j] + A[3 * i + 1] * B[3 + j] + A[3 * i + 2] * B[6 + j] for i in range(3) for j in range(3)]


def s3_abc(sigma, s, theta, small_theta):          # sim3.h:88-135, 166-208
    if abs(sigma.f) < EPS_BRANCH:
        C = R(1.0)
        if small_theta:
            A, B = R(0.5), R(1.0 / 6.0)
        else:
            theta2 = theta * theta
            A = (1 - cos(theta)) / theta2
            B = (theta - sin(theta)) / (theta2 * theta)
    else:
        C = (s - 1) / sigma
        if small_theta:
            sigma2 = sigma * sigma
            A = ((sigma - 1) * s + 1) / sigma2
            B = ((0.5 * sigma2 - sigma + 1) * s) / (sigma2 * sigma)
        else:
            a, b = s * sin(theta), s * cos(theta)
            theta2, sigma2 = theta * theta, sigma * sigma
            c = theta2 + sigma2
            A = (a * sigma + (1 - b) * theta) / (theta * c)
            B = (C - ((b - 1) * sigma + a * theta) / c) * (1.0 / theta2)
    if MUT["abc_swap"]:
        A, B = B, A
    return A, B, C


def s3_exp(u):                                      # Sim3(Vector7d), sim3.h:70-142
    om = u[:3]
    sigma = u[6]
    theta = sqrt(om[0] * om[0] + om[1] * om[1] + om[2] * om[2])
    small = theta.f < EPS_BRANCH
    s = exp(sigma)
    A, B, C = s3_abc(sigma, s, theta, small)
    Om = _skew(om)
    O2 = _matmul3(Om, Om)
    I = [R(1.0 if k in (0, 4, 8) else 0.0) for k in range(9)]
    if small:
        rb = R(0.5) if MUT["exp_half"] else R(1.0)
        Rm = [I[k] + Om[k] + rb * O2[k] for k in range(9)]
    else:
        ra, rb = sin(theta) / theta, (1 - cos(theta)) / (theta * theta)
        Rm = [I[k] + ra * Om[k] + rb * O2[k] for k in range(9)]
    W = [A * Om[k] + B * O2[k] + C * I[k] for k in range(9)]
    t = [W[3 * i] * u[3] + W[3 * i + 1] * u[4] + W[3 * i + 2] * u[5] for i in range(3)]
    return R_to_quat(Rm) + t + [s]


def s3_log(S):                                      # Sim3::log, sim3.h:148-230
    sigma = log(S[7])
    Rm = quat_to_R(S[:4])
    d = 0.5 * (Rm[0] + Rm[4] + Rm[8] - 1)
    small = d.f > 1 - EPS_BRANCH
    dR = [Rm[7] - Rm[5], Rm[2] - Rm[6], Rm[3] - Rm[1]]
    if small:
        om = [0.5 * x for x in dR]
        theta = R(0.0)
    else:
        theta = acos(d)
        f = theta / (2 * sqrt(1 - d * d))
        om = [f * x for x in dR]
    A, B, C = s3_abc(sigma, S[7], theta, small)
    Om = _skew(om)
    BOm = [B * x for x in Om]
    BO2 = _matmul3(BOm, Om)                         # (B * Omega) * Omega
    W = [A * Om[k] + BO2[k] + C * R(1.0 if k in (0, 4, 8) else 0.0) for k in range(9)]
    y = list(S[4:7])
    for k in range(3):                              # W.lu().solve(t): partial pivoting
        piv = max(range(k, 3), key=lambda i: abs(W[3 * i + k].f))
        if abs(W[3 * piv + k].f) <= abs(W[3 * k + k].f):
            piv = k
        if piv != k:
            for j in range(3):
                W[3 * k + j], W[3 * piv + j] = W[3 * piv + j], W[3 * k + j]
            y[k], y[piv] = y[piv], y[k]
        for i in range(k + 1, 3):
            f = W[3 * i + k] / W[3 * k + k]
            for j in range(k + 1, 3):
                W[3 * i + j] = W[3 * i + j] - f * W[3 * k + j]
            y[i] = y[i] - f * y[k]
    u2 = y[2] / W[8]
    u1 = (y[1] - W[5] * u2) / W[4]
    u0 = (y[0] - W[1] * u1 - W[2] * u2) / W[0]
    return om + [u0, u1, u2, sigma]


def s3_oplus(v, u, fix_scale):                      # VertexSim3Expmap::oplusImpl, types_seven_dof_expmap.h:60-69
    u = list(u)
    if fix_scale and not MUT["no_fix_scale"]:
        u[6] = R(0.0)
    return s3_mul(s3_exp(u), v)


def edge_error(C, vi, vj):                          # EdgeSim3::computeError, types_seven_dof_expmap.h:105-114
    return s3_log(s3_mul(s3_mul(C, vi), s3_inv(vj)))


def edge_jacobians(meas, si, sj, free_i=True, free_j=True, fix_scale=False):
    """exact error (7,), Ji, Jj (7,7) of the central-difference formula and their rounding bounds, for f64 rows meas, si, sj"""
    C, vi, vj = s3(meas), s3(si), s3(sj)
    e = edge_error(C, vi, vj)
    scalar = R(1.0 / (2 * DELTA))
    out = []
    for side, free in ((0, free_i), (1, free_j)):
        J = np.zeros((7, 7)); B = np.zeros((7, 7))
        if free:
            for d in range(7):
                if d == 6 and fix_scale and not MUT["no_fix_scale"]:
                    continue    # oplus zeroes u[6]: e+ and e- are the same f64 computation, their difference is exactly zero
                cols = []
                for sgn in (1.0, -1.0):
                    add = [R(0.0)] * 7
                    add[d] = R(sgn * DELTA)
                    cols.append(edge_error(C, vi, s3_oplus(vj, add, fix_scale)) if side else
                                edge_error(C, s3_oplus(vi, add, fix_scale), vj))
                for r in range(7):
                    jr = scalar * (cols[0][r] - cols[1][r])
                    J[r, d] = float(jr.v); B[r, d] = jr.e
        out.append((J, B))
    (Ji, Bi), (Jj, Bj) = out
    if MUT["swap_jac"]:
        Ji, Jj = Jj, Ji
    return dict(err=values(e), err_bound=bounds(e), Ji=Ji, Ji_bound=Bi, Jj=Jj, Jj_bound=Bj)


def ops(u, a, b, fix_scale=False):
    """exact values and bounds of exp(u), log(a), a*b, a^-1, oplus(a, u) for one row"""
    U_, A_, B_ = [R(float(x)) for x in u], s3(a), s3(b)
    res = dict(exp=s3_exp(U_), log=s3_log(A_), mul=s3_mul(A_, B_), inv=s3_inv(A_), oplus=s3_oplus(A_, U_, fix_scale))
    return {k: (values(v), bounds(v)) for k, v in res.items()}


def ratio(err, tol):
    """max of |err| / tol over the entries; an entry with zero tolerance must be exactly zero"""
    err = np.abs(np.asarray(err, np.float64)); tol = np.asarray(tol, np.float64)
    if ((tol == 0) & (err != 0)).any():
        return float("inf")
    r = np.divide(err, tol, out=np.zeros_like(err), where=tol > 0)
    return float(r.max()) if r.size else 0.0


# ---- the essential graph's linear system in f64 ------------------------------------------------------------------------------
def structure(p):
    """(active edges, vidx, rowptr, col) as ccm_pgo_solve builds them: edges with at least one free end, free vertices that have an
    edge numbered in row order, the full symmetric block pattern with ascending columns"""
    fixed = np.asarray(p.fixed) != 0
    ei, ej = np.asarray(p.edge_i, np.int64), np.asarray(p.edge_j, np.int64)
    act = np.flatnonzero(~(fixed[ei] & fixed[ej]))
    has = np.zeros(len(fixed), bool)
    has[ei[act]] = True; has[ej[act]] = True
    free = has & ~fixed
    vidx = np.full(len(fixed), -1, np.int64)
    vidx[free] = np.arange(free.sum())
    n = int(free.sum())
    a, b = vidx[ei[act]], vidx[ej[act]]
    both = (a >= 0) & (b >= 0) & (a != b)
    keys = np.unique(np.concatenate([np.arange(n) * (n + 1), a[both] * n + b[both], b[both] * n + a[both]]))
    rows, cols = keys // n, keys % n
    rowptr = np.searchsorted(rows, np.arange(n + 1)).astype(np.int32)
    return act, vidx.astype(np.int32), rowptr, cols.astype(np.int32)


def edge_magnitude(meas, si, sj, err):
    """M_e = (1 + |t_C| + s_C |t_i| + s_C s_i |t_j| / s_j) k_e per edge: the translation magnitudes that cancel in log(C Si Sj^-1),
    times k_e = 1 + 1 / theta_e when the error's rotation angle theta_e takes the log's large-angle branch, where (1 - cos) / theta^2
    loses u / theta^2 of A and W^-1 t gains u |t| / theta"""
    n3 = lambda x: np.linalg.norm(x[:, 4:7], axis=1)
    th = np.linalg.norm(np.asarray(err)[:, :3], axis=1)
    k = np.where(th > 0.9 * LOG_SMALL_ANGLE, 1.0 + 1.0 / np.maximum(th, 1e-300), 1.0)
    return (1.0 + n3(meas) + meas[:, 7] * n3(si) + meas[:, 7] * si[:, 7] * n3(sj) / sj[:, 7]) * k


def jacobian_bound(meas, si, sj, err, free_i, free_j, fix_scale):
    """per-edge bound of every Jacobian entry, (E,7,7) for each side: EDGE_OPS u M_e / delta, zero on a fixed side and in the scale
    column under fix_scale"""
    M = edge_magnitude(meas, si, sj, err) * EDGE_OPS * U / DELTA
    out = []
    for free in (free_i, free_j):
        B = np.broadcast_to(M[:, None, None], (len(M), 7, 7)).copy()
        B[~np.asarray(free, bool)] = 0.0
        if fix_scale:
            B[:, :, 6] = 0.0
        out.append(B)
    return out


def error_bound(meas, si, sj, err):
    return edge_magnitude(meas, si, sj, err) * EDGE_OPS * U


class System:
    """H (without lambda), b and chi2 of problem p at p.sim3, assembled in f64 from per-edge errors and Jacobians, in the pattern of
    `structure`, with a bound for every entry.  err (E,7), Ji, Jj (E,7,7) are given for every edge of p (only active ones are used)."""

    def __init__(self, p, err, Ji, Jj):
        act, vidx, rowptr, col = structure(p)
        self.act, self.vidx, self.rowptr, self.col = act, vidx, rowptr, col
        n = len(rowptr) - 1
        self.n, self.nnzb = n, len(col)
        sim3, meas = np.asarray(p.sim3, np.float64), np.asarray(p.meas, np.float64)
        ei, ej = np.asarray(p.edge_i, np.int64)[act], np.asarray(p.edge_j, np.int64)[act]
        m, si, sj = meas[act], sim3[ei], sim3[ej]
        a, b = vidx[ei].astype(np.int64), vidx[ej].astype(np.int64)
        e, Ji, Jj = np.asarray(err)[act], np.asarray(Ji)[act].copy(), np.asarray(Jj)[act].copy()
        if MUT["swap_jac"]:
            Ji, Jj = Jj, Ji
        dJi, dJj = jacobian_bound(m, si, sj, e, a >= 0, b >= 0, p.fix_scale)
        de = error_bound(m, si, sj, e)
        if not MUT["fixed_side"]:
            Ji[a < 0] = 0.0; Jj[b < 0] = 0.0
        row_of = np.repeat(np.arange(n), np.diff(rowptr))
        blk = lambda r, c: np.searchsorted(row_of * n + col, r * n + c)
        H = np.zeros((self.nnzb, 7, 7)); HB = np.zeros((self.nnzb, 7, 7)); Ha = np.zeros((self.nnzb, 7, 7))
        cnt = np.zeros(self.nnzb)
        bv = np.zeros((n, 7)); bB = np.zeros((n, 7)); ba = np.zeros((n, 7)); bc = np.zeros(n)
        T = lambda X: np.swapaxes(X, -1, -2)
        dot = lambda X, Y: np.einsum("ekr,ekc->erc", X, Y)

        def scatter(idx, val, bnd, absval):
            for q in range(0, len(idx), 1 << 16):
                s = slice(q, q + (1 << 16))
                np.add.at(H, idx[s], val[s]); np.add.at(HB, idx[s], bnd[s]); np.add.at(Ha, idx[s], absval[s])
                np.add.at(cnt, idx[s], 1)

        for J, dJ, v in ((Ji, dJi, a), (Jj, dJj, b)):
            # MUT["fixed_side"]: a fixed side's (nonzero) Jacobian is scattered through its unset slot, block 0 / row 0
            on = v >= 0 if not MUT["fixed_side"] else np.ones(len(v), bool)
            vv = np.maximum(v, 0)[on]
            Jo, dJo, Ao = J[on], dJ[on], np.abs(J[on])
            scatter(blk(vv, vv), dot(Jo, Jo), dot(Ao, dJo) + dot(dJo, Ao) + dot(dJo, dJo), dot(Ao, Ao))
            eo, deo = e[on], de[on]
            np.add.at(bv, vv, -np.einsum("ekr,ek->er", Jo, eo))
            np.add.at(bB, vv, np.einsum("ekr,ek->er", Ao, np.broadcast_to(deo[:, None], eo.shape)) + np.einsum("ekr,ek->er", dJo, np.abs(eo)))
            np.add.at(ba, vv, np.einsum("ekr,ek->er", Ao, np.abs(eo)))
            np.add.at(bc, vv, 1)
        both = (a >= 0) & (b >= 0) & (a != b)
        Xi, Xj, dXi, dXj = Ji[both], Jj[both], dJi[both], dJj[both]
        cross = dot(Xi, Xj)
        cb = dot(np.abs(Xi), dXj) + dot(dXi, np.abs(Xj)) + dot(dXi, dXj)
        ca = dot(np.abs(Xi), np.abs(Xj))
        scatter(blk(a[both], b[both]), cross, cb, ca)
        mirror = cross if MUT["mirror_no_transpose"] else T(cross)
        scatter(blk(b[both], a[both]), mirror, T(cb), T(ca))
        # f64 summation: 7 products per entry, then one red.add per contributing edge
        self.H = H
        self.H_bound = HB + (7 + cnt[:, None, None]) * U * Ha
        self.b = bv
        self.b_bound = bB + (7 + bc[:, None]) * U * ba
        ee = np.einsum("ek,ek->e", e, e)
        self.chi2 = float(ee.sum())
        self.chi2_bound = float(2 * (np.abs(e).sum(1) * de).sum() + (7 + len(ee)) * U * ee.sum())
        self.row = row_of

    def dense(self, lam=0.0):
        n = self.n
        D = np.zeros((7 * n, 7 * n))
        for q in range(self.nnzb):
            r, c = self.row[q], self.col[q]
            D[7 * r:7 * r + 7, 7 * c:7 * c + 7] = self.H[q]
        return D + lam * np.eye(7 * n)

    def sparse(self, lam=0.0):
        return block_matrix(self.H, self.rowptr, self.col, lam)


def block_matrix(H, rowptr, col, lam=0.0):
    """H + lam I as a scipy CSC matrix from 7x7 block CSR (rowptr, col, H (nnzb,7,7))"""
    import scipy.sparse as sp
    n = len(rowptr) - 1
    return (sp.bsr_matrix((H, col, rowptr), shape=(7 * n, 7 * n)) + lam * sp.identity(7 * n)).tocsc()


def oracle_edges(p, pieces):
    """f64 per-edge error and Jacobians of every edge of p from the oracle (Jacobians of both sides; System zeroes a fixed side)"""
    from oracle import pyoracle
    sim3, meas = np.asarray(p.sim3, np.float64), np.asarray(p.meas, np.float64)
    ei, ej = np.asarray(p.edge_i), np.asarray(p.edge_j)
    E = len(ei)
    err = np.empty((E, 7)); Ji = np.empty((E, 7, 7)); Jj = np.empty((E, 7, 7))
    for k in range(E):
        err[k] = pyoracle.pgo_edge_error(meas[k], sim3[ei[k]], sim3[ej[k]])
        Ji[k], Jj[k] = pieces.pgo_edge_jacobian(meas[k], sim3[ei[k]], sim3[ej[k]], p.fix_scale)
    return err, Ji, Jj

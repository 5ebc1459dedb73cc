"""A high-precision restatement of the global BA's linearisation, pose update and trial chi2 (test infrastructure).

* Per edge, EdgeSE3ProjectXYZ (G/types/types_six_dof_expmap.cpp:103-139) with each keyframe's own intrinsics: the error z - proj,
  the Jacobians Jp (2x6, d e / d (omega, upsilon)) and Jl (2x3), and chi2 = w |e|^2.  Written once over an abstract number type and
  evaluated two ways:
    - with sim3_ref's `R` (mpmath at 40 digits on the exact values of the f64 / f32 inputs, an f64 shadow and a first-order bound on
      the rounding of any f64 evaluation of the formula) on every edge of a small scene, or on a fixed sample plus the edge-case
      edges of a large one;
    - with `V`, the same bound arithmetic on numpy arrays of f64 shadows, on every edge.  The shadow is one f64 evaluation of the
      formula, so it is within the bound of the exact value and any other f64 evaluation is within twice the bound of it; the
      comparisons use that doubled bound.  The R pass checks that the shadow really sits inside its bound.
* RobustKernelHuber (G/core/robust_kernel_impl.cpp:77-91) with delta^2 rounded to a float (robust_kernel_impl.h:84), and the per-edge
  blocks of constructQuadraticForm (G/core/base_binary_edge.hpp:75-113): W = wz rho' w Jp^T Jl, wz = 0 for a fixed keyframe, and the
  landmark terms rho' w Jl^T Jl and -rho' w Jl^T e.
* Assembled per landmark (Hll, bl), per free pose (Hpp, bp) and over the active edges (the robust chi2), each entry with a bound
  that covers the rounding of its terms and any order of the f64 summation: (n + 1) u sum |term|.
* VertexSE3Expmap::oplusImpl = exp(x) * T (G/types/types_six_dof_expmap.h:73-76, G/types/se3quat.h:223-257) in R, with g2o's
  theta < 1e-5 branch R = I + W + W^2, Eigen's four branches of Quaterniond(Matrix3d) and normalisation with w >= 0, and the two
  halves of the gain-ratio denominator, sum x (lambda x + bp) and sum xl (lambda xl + bl).

Only active edges contribute (flag bit 0 clear); flag bit 1, or a negative weight in the device's packed form, means no kernel.
A comparison passes when |got - restated| <= TAU * bound entry by entry (`ratio`); an entry whose bound is zero must be exactly zero.
"""
from __future__ import annotations

import numpy as np

from tests import sim3_ref as S
from tests.sim3_ref import R, U, UF, TAU, ratio   # noqa: F401  (re-exported for the tests)

# Deliberate defects for the mutation tests (tests/test_ba_ref.py, tests/test_ba_math_host.py): each must push the restatement far
# outside its bound against the oracle.  All False in normal use.
MUT = dict(dsqr_double=False, small_half=False, intr_kf0=False, jl_col2_sign=False, w_fixed=False, bl_sign=False, no_point_scale=False)

EPS_THETA = 0.00001       # g2o's small-angle threshold of SE3Quat::exp
SAMPLE = 2000             # mpmath edges of a scene above MP_ALL edges
MP_ALL = 20000


class V:
    """f64 shadow f (numpy array) and rounding bound e of every element: sim3_ref.R's arithmetic without the exact value"""
    __slots__ = ("f", "e")

    def __init__(self, f, e=None):
        self.f = np.asarray(f, np.float64)
        self.e = np.zeros_like(self.f) if e is None else e

    @staticmethod
    def _c(x):
        return x if isinstance(x, V) else V(x)

    def __add__(self, o):
        o = V._c(o)
        return V(self.f + o.f, self.e + o.e + U * (np.abs(self.f) + np.abs(o.f)))
    __radd__ = __add__

    def __sub__(self, o):
        o = V._c(o)
        return V(self.f - o.f, self.e + o.e + U * (np.abs(self.f) + np.abs(o.f)))

    def __rsub__(self, o):
        return V._c(o) - self

    def __neg__(self):
        return V(-self.f, self.e)

    def __mul__(self, o):
        o = V._c(o)
        r = self.f * o.f
        return V(r, np.abs(self.f) * o.e + np.abs(o.f) * self.e + self.e * o.e + U * np.abs(r))
    __rmul__ = __mul__

    def __truediv__(self, o):
        o = V._c(o)
        r = self.f / o.f
        den = np.maximum(np.abs(o.f) - o.e, np.abs(o.f) * 0.5)
        return V(r, (self.e + np.abs(r) * o.e) / den + U * np.abs(r))

    def __rtruediv__(self, o):
        return V._c(o) / self


def _sqrt(x):
    if isinstance(x, R):
        return S.sqrt(x)
    r = np.sqrt(x.f)
    return V(r, np.where((r > 0) & (x.e < x.f), x.e / (2 * np.where(r > 0, r, 1.0)), np.sqrt(x.e)) + UF * r)


# ---- one edge --------------------------------------------------------------------------------------------------------------
def edge_terms(T, X, uv, intr, w, mk):
    """error (2), Jp (12, row-major 2x6), Jl (6, row-major 2x3), Xc (3) and chi2 of EdgeSE3ProjectXYZ at pose row T (qx qy qz qw
    tx ty tz), point X, measurement uv, intrinsics (fx fy cx cy) and information weight w; mk turns an input into the number type"""
    q = [mk(T[k]) for k in range(4)]
    xc = S.quat_rotate(q, [mk(X[k]) for k in range(3)])
    x, y, z = [xc[k] + mk(T[4 + k]) for k in range(3)]
    fx, fy, cx, cy = [mk(intr[k]) for k in range(4)]
    iz = 1.0 / z
    e = [mk(uv[0]) - (x * iz * fx + cx), mk(uv[1]) - (y * iz * fy + cy)]
    chi2 = mk(w) * (e[0] * e[0] + e[1] * e[1])
    Rm = S.quat_to_R(q)
    iz2 = iz * iz
    a0, a2 = -fx * iz, x * iz2 * fx                    # Jl = -1/z [[fx, 0, -x/z fx], [0, fy, -y/z fy]] R
    b1, b2 = -fy * iz, y * iz2 * fy
    Jl = [a0 * Rm[j] + a2 * Rm[6 + j] for j in range(3)] + [b1 * Rm[3 + j] + b2 * Rm[6 + j] for j in range(3)]
    if MUT["jl_col2_sign"]:
        Jl[2], Jl[5] = -Jl[2], -Jl[5]
    zero = x * 0.0                                     # an exact zero of the operand's shape
    Jp = [x * y * iz2 * fx, -(1 + (x * x * iz2)) * fx, y * iz * fx, -iz * fx, zero, x * iz2 * fx,
          (1 + y * y * iz2) * fy, -x * y * iz2 * fy, -x * iz * fy, zero, -iz * fy, y * iz2 * fy]
    return e, Jp, Jl, [x, y, z], chi2


def dsqr_of(delta):
    return delta * delta if MUT["dsqr_double"] else float(np.float32(delta * delta))


def huber_r(c, delta):
    """rho(c), rho'(c) in R for one chi2 c"""
    d2 = dsqr_of(delta)
    if c.f <= d2:
        return c, R(1.0)
    sq = S.sqrt(c)
    return 2 * sq * delta - d2, delta / sq


def huber_v(c, delta, rob):
    """rho, rho' in V; rob (bool array) selects the edges with a kernel"""
    d2 = dsqr_of(delta)
    out = rob & (c.f > d2)
    sq = _sqrt(V(np.where(out, c.f, 1.0), np.where(out, c.e, 0.0)))
    r0o, r1o = 2 * sq * delta - d2, delta / sq
    rho0 = V(np.where(out, r0o.f, c.f), np.where(out, r0o.e, c.e))
    rho1 = V(np.where(out, r1o.f, 1.0), np.where(out, r1o.e, 0.0))
    return rho0, rho1, out


def _intr(p):
    return np.broadcast_to(p.intr[0], p.intr.shape) if MUT["intr_kf0"] else p.intr


def edge_flags(p):
    f = np.zeros(p.E, np.uint8) if p.edge_flags is None else np.asarray(p.edge_flags, np.uint8)
    return (f & 1) == 0, (f & 2) == 0


def mp_edges(p, idx, poses=None, points=None):
    """R-evaluated err (n,2), Jp (n,2,6), Jl (n,2,3), chi2 (n) with their exact values and bounds for the edges idx"""
    poses = p.poses if poses is None else poses
    points = p.points if points is None else points
    intr = _intr(p)
    out = {k: [] for k in ("err", "Jp", "Jl", "chi2")}
    bnd = {k: [] for k in out}
    for i in idx:
        kf, mp = int(p.obs_kf[i]), int(p.obs_mp[i])
        e, Jp, Jl, _, c = edge_terms(poses[kf], points[mp], p.obs_uv[i].astype(np.float64), intr[kf], float(p.obs_w[i]), R)
        for k, v in (("err", e), ("Jp", Jp), ("Jl", Jl), ("chi2", [c])):
            out[k].append([float(x.v) for x in v]); bnd[k].append([x.e for x in v])
        # the f64 shadow must sit within its bound of the exact value (this is what V relies on)
        for v in e + Jp + Jl + [c]:
            assert abs(v.f - float(v.v)) <= v.e * 1.0000001 + 1e-300, (i, v.f, float(v.v), v.e)
    shp = dict(err=(2,), Jp=(2, 6), Jl=(2, 3), chi2=())
    return ({k: np.array(out[k]).reshape((-1,) + shp[k]) for k in out}, {k: np.array(bnd[k]).reshape((-1,) + shp[k]) for k in out})


def sample_edges(p, special=(), seed=0):
    """every edge of a scene up to MP_ALL edges; above, a fixed sample of SAMPLE edges plus the given edge-case edges"""
    if p.E <= MP_ALL:
        return np.arange(p.E)
    rng = np.random.default_rng(seed)
    return np.union1d(rng.choice(p.E, SAMPLE, replace=False), np.asarray(special, np.int64))


class Lin:
    """the restated linearisation of problem p at (poses, points): per edge (V over all edges) and the assembled blocks"""

    def __init__(self, p, poses=None, points=None, robust=True, delta=None):
        poses = np.asarray(p.poses if poses is None else poses, np.float64)
        points = np.asarray(p.points if points is None else points, np.float64)
        kf, mp = np.asarray(p.obs_kf, np.int64), np.asarray(p.obs_mp, np.int64)
        act, rob = edge_flags(p)
        rob = rob & bool(robust)
        w = np.asarray(p.obs_w, np.float32).astype(np.float64)
        intr = _intr(p)
        with np.errstate(all="ignore"):
            e, Jp, Jl, Xc, c = edge_terms(poses[kf].T, points[mp].T, p.obs_uv.astype(np.float64).T, intr[kf].T, w, V)
            rho0, rho1, out = huber_v(c, delta, rob)
            wo = rho1 * V(w)
            fixed = np.asarray(p.fixed) != 0
            zf = fixed[kf] & (not MUT["w_fixed"])
            wz = V(np.where(zf, 0.0, wo.f), np.where(zf, 0.0, wo.e))
            Wt = [[(wz * Jp[r]) * Jl[cc] + (wz * Jp[6 + r]) * Jl[3 + cc] for cc in range(3)] for r in range(6)]
            r0, r1 = -wo * e[0], -wo * e[1]
            hl = [wo * (Jl[i] * Jl[j] + Jl[3 + i] * Jl[3 + j]) for i in range(3) for j in range(3)]
            bl = [Jl[i] * r0 + Jl[3 + i] * r1 for i in range(3)]
            hp = [wo * (Jp[i] * Jp[j] + Jp[6 + i] * Jp[6 + j]) for i in range(6) for j in range(6)]
            bp = [Jp[i] * r0 + Jp[6 + i] * r1 for i in range(6)]
        self.p, self.act, self.rob, self.out = p, act, rob, out
        self.delta = delta
        self.dsqr = dsqr_of(delta)
        self.err = np.stack([x.f for x in e], 1); self.err_b = 2 * np.stack([x.e for x in e], 1)
        self.Jp = np.stack([x.f for x in Jp], 1).reshape(-1, 2, 6); self.Jp_b = 2 * np.stack([x.e for x in Jp], 1).reshape(-1, 2, 6)
        self.Jl = np.stack([x.f for x in Jl], 1).reshape(-1, 2, 3); self.Jl_b = 2 * np.stack([x.e for x in Jl], 1).reshape(-1, 2, 3)
        self.chi2, self.chi2_b = c.f, 2 * c.e
        self.rho1, self.rho1_b = rho1.f, 2 * rho1.e
        self.depth, self.depth_b = Xc[2].f, 2 * Xc[2].e
        # per edge W (E,6,3): zero for inactive edges and fixed keyframes
        Wv = np.stack([np.stack([x.f for x in row], 1) for row in Wt], 1)
        Wb = 2 * np.stack([np.stack([x.e for x in row], 1) for row in Wt], 1)
        self.W = np.where(act[:, None, None], Wv, 0.0); self.W_b = np.where(act[:, None, None], Wb, 0.0)
        a = act
        self.Hll, self.Hll_b = _assemble(mp[a], p.P, [x for x in hl], a)
        self.Hll, self.Hll_b = self.Hll.reshape(-1, 3, 3), self.Hll_b.reshape(-1, 3, 3)
        sgn = -1.0 if MUT["bl_sign"] else 1.0
        self.bl, self.bl_b = _assemble(mp[a], p.P, bl, a)
        self.bl = sgn * self.bl
        free = ~fixed
        pa = a & free[kf]
        self.Hpp, self.Hpp_b = _assemble(kf[pa], p.K, hp, pa)
        self.Hpp, self.Hpp_b = self.Hpp.reshape(-1, 6, 6), self.Hpp_b.reshape(-1, 6, 6)
        self.bp, self.bp_b = _assemble(kf[pa], p.K, bp, pa)
        r = rho0.f[a]
        self.chi2_sum = float(r.sum())
        self.chi2_sum_b = float(2 * rho0.e[a].sum() + (a.sum() + 1) * U * np.abs(r).sum())

    def max_diag(self):
        """the largest diagonal entry of Hpp (free poses) and Hll, its bound, and where it is ('Hpp' / 'Hll')"""
        dp = np.diagonal(self.Hpp, axis1=1, axis2=2); dl = np.diagonal(self.Hll, axis1=1, axis2=2)
        bp = np.diagonal(self.Hpp_b, axis1=1, axis2=2); bl = np.diagonal(self.Hll_b, axis1=1, axis2=2)
        ip, il = np.unravel_index(np.argmax(dp), dp.shape), np.unravel_index(np.argmax(dl), dl.shape)
        if dp[ip] >= dl[il]:
            return float(dp[ip]), float(max(bp.max(), bl.max())), "Hpp"
        return float(dl[il]), float(max(bp.max(), bl.max())), "Hll"


def _assemble(owner, n, terms, sel):
    """sum over the selected edges of each term (V over all edges) per owner index, with a bound for any summation order"""
    f = np.stack([t.f[sel] for t in terms], 1)
    e = np.stack([t.e[sel] for t in terms], 1)
    cnt = np.bincount(owner, minlength=n).astype(np.float64)
    val = np.zeros((n, f.shape[1])); bd = np.zeros((n, f.shape[1])); ab = np.zeros((n, f.shape[1]))
    np.add.at(val, owner, f); np.add.at(bd, owner, 2 * e); np.add.at(ab, owner, np.abs(f))
    return val, bd + (cnt[:, None] + 1) * U * ab


def chi2_at(p, poses, points, robust=True, delta=None):
    """the robust chi2 over the active edges at (poses, points) and its bound"""
    kf, mp = np.asarray(p.obs_kf, np.int64), np.asarray(p.obs_mp, np.int64)
    act, rob = edge_flags(p)
    rob = rob & bool(robust)
    w = np.asarray(p.obs_w, np.float32).astype(np.float64)
    poses, points = np.asarray(poses, np.float64), np.asarray(points, np.float64)
    with np.errstate(all="ignore"):
        _, _, _, _, c = edge_terms(poses[kf].T, points[mp].T, p.obs_uv.astype(np.float64).T, _intr(p)[kf].T, w, V)
        rho0, _, _ = huber_v(c, delta, rob)
    r = rho0.f[act]
    return float(r.sum()), float(2 * rho0.e[act].sum() + (act.sum() + 1) * U * np.abs(r).sum())


# ---- the update step -------------------------------------------------------------------------------------------------------
def quat_normalize_pos_w(q):
    x, y, z, w = q
    if w.f < 0:
        x, y, z, w = -x, -y, -z, -w
    n = S.sqrt(x * x + y * y + z * z + w * w)
    return [x / n, y / n, z / n, w / n]


def se3_exp_times(u, T):
    """exp(u) * T in R for u = (omega, upsilon) and a pose row T (qx qy qz qw tx ty tz): values (7), bounds (7), and which branch
    of R_to_quat the exponential took (-1 for the trace branch, 0 / 1 / 2 for the diagonal ones) and whether the product needed
    the w < 0 flip"""
    u = [R(float(v)) for v in u]
    T = [R(float(v)) for v in T]
    ox, oy, oz = u[:3]
    theta2 = ox * ox + oy * oy + oz * oz
    theta = S.sqrt(theta2)
    if theta.f < EPS_THETA:
        a = va = R(1.0)
        b = vb = R(0.5) if MUT["small_half"] else R(1.0)     # the mutation: the textbook I + W + W^2 / 2, and V = R as in g2o
    else:
        s, c = S.sin(theta), S.cos(theta)
        a = s / theta
        b = (1 - c) / theta2
        va = b
        vb = (theta - s) / (theta2 * theta)
    W2 = [ox * ox - theta2, ox * oy, ox * oz, ox * oy, oy * oy - theta2, oy * oz, ox * oz, oy * oz, oz * oz - theta2]
    z = R(0.0)
    Wm = [z, -oz, oy, oz, z, -ox, -oy, ox, z]
    Rm, Vm = [], []
    for i in range(9):
        idn = R(1.0 if i in (0, 4, 8) else 0.0)
        Rm.append(idn + a * Wm[i] + b * W2[i])
        Vm.append(idn + va * Wm[i] + vb * W2[i])
    tr = (Rm[0] + Rm[4] + Rm[8]).f
    branch = -1 if tr > 0 else (0 if Rm[0].f >= Rm[4].f and Rm[0].f >= Rm[8].f else (1 if Rm[4].f > Rm[0].f and Rm[4].f >= Rm[8].f else 2))
    ex, ey, ez, ew = quat_normalize_pos_w(S.R_to_quat(Rm))
    et = [Vm[3 * i] * u[3] + Vm[3 * i + 1] * u[4] + Vm[3 * i + 2] * u[5] for i in range(3)]
    r = S.quat_rotate([ex, ey, ez, ew], T[4:7])
    tx, ty, tz = [et[k] + r[k] for k in range(3)]
    qx, qy, qz, qw = T[:4]
    ow = ew * qw - ex * qx - ey * qy - ez * qz
    ox_ = ew * qx + ex * qw + ey * qz - ez * qy
    oy_ = ew * qy + ey * qw + ez * qx - ex * qz
    oz_ = ew * qz + ez * qw + ex * qy - ey * qx
    flip = ow.f < 0
    q = quat_normalize_pos_w([ox_, oy_, oz_, ow])
    res = q + [tx, ty, tz]
    return np.array([float(x.v) for x in res]), np.array([x.e for x in res]), branch, flip


def update_poses(p, x):
    """restated trial poses for the pose step x (K,6): free poses exp(x) * T, fixed poses unchanged (bound 0: bit-identical)"""
    vals = np.array(p.poses, np.float64, copy=True); bnds = np.zeros_like(vals)
    for k in np.flatnonzero(np.asarray(p.fixed) == 0):
        vals[k], bnds[k], _, _ = se3_exp_times(x[k], p.poses[k])
    return vals, bnds


def scale_pose(lin, x, lam):
    """sum over free poses of x (lambda x + bp) and its bound, bp restated"""
    free = np.asarray(lin.p.fixed) == 0
    xv = np.asarray(x, np.float64)[free]
    t = xv * (lam * xv + lin.bp[free])
    b = np.abs(xv) * lin.bp_b[free] + 2 * U * np.abs(xv) * (lam * np.abs(xv) + np.abs(lin.bp[free]))
    return float(t.sum()), float(b.sum() + (t.size + 1) * U * np.abs(t).sum())


def scale_point(lin, xl, lam):
    """sum over landmarks of xl (lambda xl + bl) for the landmark step xl (P,3) and its bound, bl restated"""
    if MUT["no_point_scale"]:
        return 0.0, 0.0
    xl = np.asarray(xl, np.float64)
    t = xl * (lam * xl + lin.bl)
    b = np.abs(xl) * lin.bl_b + 2 * U * np.abs(xl) * (lam * np.abs(xl) + np.abs(lin.bl))
    return float(t.sum()), float(b.sum() + (t.size + 1) * U * np.abs(t).sum())


def lambda_init(lin):
    """g2o's initial lambda, 1e-5 * max diag (G/core/optimization_algorithm_levenberg.cpp:185-199), and its bound"""
    m, mb, _ = lin.max_diag()
    return 1e-5 * m, 1e-5 * mb + 2 * U * 1e-5 * m


EXP_THETAS = (0.0, 1e-12, 0.99999e-5, 1.00001e-5, 0.3, 2.2, 3.1)


def exp_cases(K, seed=0):
    """pose steps (K,6) whose rotation angles cycle through EXP_THETAS about axes that send R_to_quat down each of its branches
    (near pi the largest diagonal entry of R picks x, y or z), with translations of a few decimetres"""
    rng = np.random.default_rng(seed)
    axes = [np.array(a, np.float64) for a in ((1, 0.2, 0.1), (0.1, 1, 0.3), (0.2, 0.1, 1), (0.6, -0.5, 0.62))]
    x = np.zeros((K, 6))
    for k in range(K):
        th = EXP_THETAS[k % len(EXP_THETAS)]
        ax = axes[(k // len(EXP_THETAS)) % len(axes)]
        x[k, :3] = ax / np.linalg.norm(ax) * th
        x[k, 3:] = rng.normal(0, 0.3, 3)
    return x

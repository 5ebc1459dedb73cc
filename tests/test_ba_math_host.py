"""CPU suite: the arithmetic of the BA kernels (csrc/ba_math.cuh: linearize_obs, huber, se3_exp_times) built with g++ and held to
the restatement of tests/ba_ref.py at the edge cases of tests/ba_scenes.py: four cameras, far, near and behind-the-camera points,
the Huber band of both deltas, and the exp-map angles around g2o's 1e-5 branch with every R_to_quat branch and the w < 0 flip.
What this cannot show is the kernels' own use of these functions (gathers, weights, sums, the zeros of inactive edges, which
linearize_obs evaluates like any other edge): tests/test_gpu_ba_steps.py."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from tests import ba_ref as F
from tests import ba_scenes as B
from tests.ba_ref import TAU, ratio

HERE = os.path.dirname(os.path.abspath(__file__))


@pytest.fixture(scope="module")
def bm(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("bm") / "libba_math_host.so")
    cxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
    subprocess.check_call([cxx, "-O2", "-std=c++17", "-fPIC", "-shared", "-fno-fast-math", "-ffp-contract=off", "-o", so,
                           os.path.join(HERE, "host", "ba_math_host.cpp")])
    return C.CDLL(so)


def _d(a):
    a = np.ascontiguousarray(a, np.float64)
    return a, a.ctypes.data_as(C.c_void_p)


def linearize(bm, p, i):
    kf, mp = int(p.obs_kf[i]), int(p.obs_mp[i])
    keep = [_d(p.poses[kf]), _d(p.intr[kf]), _d(p.points[mp]), _d(p.obs_uv[i].astype(np.float64))]
    out = np.empty(24)
    bm.bm_linearize(*[k[1] for k in keep], C.c_double(float(p.obs_w[i])), out.ctypes.data_as(C.c_void_p))
    return out


def huber(bm, c, delta):
    out = np.empty(2)
    bm.bm_huber(C.c_double(c), C.c_double(delta), out.ctypes.data_as(C.c_void_p))
    return out


def exp_times(bm, x, T):
    a, pa = _d(x); b, pb = _d(T)
    out = np.empty(7)
    bm.bm_exp_times(pa, pb, out.ctypes.data_as(C.c_void_p))
    return out


def edge_case_edges(p):
    s = p.special
    band = [i for i, *_ in p.band]
    rng = np.random.default_rng(1)
    return np.unique(np.concatenate([s["far"], s["near"], s["behind"], band, rng.choice(p.E, 300, replace=False)]))


def worst_linearize(bm, p):
    act, _ = F.edge_flags(p)
    idx = edge_case_edges(p)
    idx = idx[act[idx]]
    ex, bd = F.mp_edges(p, idx)
    got = np.array([linearize(bm, p, i) for i in idx])
    return max(ratio(got[:, :2] - ex["err"], TAU * bd["err"]), ratio(got[:, 2] - ex["chi2"], TAU * bd["chi2"]),
               ratio(got[:, 6:12] - ex["Jl"].reshape(-1, 6), TAU * bd["Jl"].reshape(-1, 6)),
               ratio(got[:, 12:] - ex["Jp"].reshape(-1, 12), TAU * bd["Jp"].reshape(-1, 12)))


def worst_huber(bm, p):
    """rho and rho' of every band edge's restated chi2 through the product's huber, against the restated Huber of the same chi2"""
    w = 0.0
    for i, delta, _, _ in p.band:
        kf, mp = int(p.obs_kf[i]), int(p.obs_mp[i])
        c = F.edge_terms(p.poses[kf], p.points[mp], p.obs_uv[i].astype(np.float64), p.intr[kf], float(p.obs_w[i]), F.R)[4]
        r0, r1 = F.huber_r(F.R(c.f), delta)
        got = huber(bm, c.f, delta)
        w = max(w, ratio(got[0] - float(r0.v), TAU * r0.e), ratio(got[1] - float(r1.v), TAU * r1.e))
    return w


def worst_exp(bm, p):
    x = F.exp_cases(p.K)
    w = 0.0
    for poses in (p.poses, B.turned(p.poses)):
        for k in range(p.K):
            v, b, _, _ = F.se3_exp_times(x[k], poses[k])
            w = max(w, ratio(exp_times(bm, x[k], poses[k]) - v, TAU * b))
    return w


def test_linearize_obs_within_bounds(bm):
    assert worst_linearize(bm, B.scene("multicam")) <= 1.0


def test_huber_in_the_band(bm):
    p = B.scene("multicam")
    assert len(p.band) >= 12
    assert worst_huber(bm, p) <= 1.0
    # inside the band the product's inlier test uses float(delta^2): rho' is exactly 1 below it and below 1 above it
    for i, delta, lo, hi in p.band:
        kf, mp = int(p.obs_kf[i]), int(p.obs_mp[i])
        c = F.edge_terms(p.poses[kf], p.points[mp], p.obs_uv[i].astype(np.float64), p.intr[kf], float(p.obs_w[i]), F.R)[4]
        assert (huber(bm, c.f, delta)[1] == 1.0) == (c.f <= float(np.float32(delta * delta)))


def test_se3_exp_times_within_bounds(bm):
    assert worst_exp(bm, B.scene("multicam")) <= 1.0


@pytest.mark.parametrize("mut,fn", [("small_half", worst_exp), ("dsqr_double", worst_huber), ("jl_col2_sign", worst_linearize),
                                    ("intr_kf0", worst_linearize)])
def test_mutations_fail_against_the_product(bm, mut, fn):
    F.MUT[mut] = True
    try:
        r = fn(bm, B.scene("multicam"))
    finally:
        F.MUT[mut] = False
    assert r >= 100.0, (mut, r)


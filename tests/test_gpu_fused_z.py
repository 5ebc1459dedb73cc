"""The landmark-aligned linearisation (k_linearize forms Hll / bl per landmark inside one CTA, and Z = W U^-1 in the same pass) and
the landmark-aligned back-substitution, on a problem built around their schedule: landmarks of 1, 2, 32 and 33 observations (either
side of the size that still shares a CTA), 97, 127, 128 and 129 (a chunk of 128 observations and either side of it) and 300
(several chunks, summed in a first pass and recomputed in a second), placed between ordinary landmarks of 3-8 observations.

Checked: the reduced camera system and the landmark step against the f64 restatement of tests/schur_ref.py, the LM solve against
the oracle (the problem has a rejected trial, so the Z-only recompute at a larger lambda is on the compared path), and that the
per-landmark sums are deterministic."""
import numpy as np
import pytest

from ccm_slam_b200 import api, synth
from tests import schur_ref as R

pytestmark = pytest.mark.gpu

TILE = 128   # LIN_TILE of ba_kernels.cuh
SPECIAL = [1, 2, 32, 33, 97, TILE - 1, TILE, TILE + 1, 300]


@pytest.fixture(scope="module", autouse=True)
def _dev():
    assert api.device_count() > 0, "no CUDA device: the product path has no CPU fallback"
    api.init(0)


def make_problem(seed=5, K=320, n_base=1500):
    """K cameras on a 3 m baseline facing one field of points 6-10 m away, so that any subset of them sees any point"""
    rng = np.random.default_rng(seed)
    C = np.stack([np.linspace(-1.5, 1.5, K), rng.uniform(-0.1, 0.1, K), rng.uniform(-0.1, 0.1, K)], 1)
    sizes = [int(s) for s in rng.integers(3, 9, n_base)]
    at = np.sort(rng.choice(n_base, len(SPECIAL), replace=False))
    for i, s in sorted(zip(at, SPECIAL), reverse=True):
        sizes.insert(int(i), s)
    P = len(sizes)
    X = np.stack([rng.uniform(-1, 1, P), rng.uniform(-0.6, 0.6, P), rng.uniform(6, 10, P)], 1)
    kf = np.concatenate([np.sort(rng.choice(K, s, replace=False)) for s in sizes]).astype(np.int32)
    mp = np.repeat(np.arange(P), sizes).astype(np.int32)
    fx, fy, cx, cy = synth.EUROC_INTR
    Xc = X[mp] - C[kf]
    sigma = synth.SCALE_FACTOR ** rng.integers(0, 4, kf.size)
    uv = np.stack([fx * Xc[:, 0] / Xc[:, 2] + cx, fy * Xc[:, 1] / Xc[:, 2] + cy], 1) + rng.normal(size=(kf.size, 2)) * sigma[:, None]
    q_gt = np.tile([0.0, 0.0, 0.0, 1.0], (K, 1)); t_gt = -C
    drot = synth._rotvec_to_quat(rng.normal(size=(K, 3)) * 0.01)
    q0 = synth._quat_mul(drot, q_gt)
    t0 = synth._quat_rot(drot, t_gt) + rng.normal(size=(K, 3)) * 0.03
    fixed = np.zeros(K, np.uint8); fixed[:2] = 1
    q0[:2] = q_gt[:2]; t0[:2] = t_gt[:2]
    q0 /= np.linalg.norm(q0, axis=-1, keepdims=True)
    pts0 = (X + rng.normal(size=(P, 3)) * 0.05).astype(np.float32).astype(np.float64)
    intr = np.tile(np.array(synth.EUROC_INTR, np.float32).astype(np.float64), (K, 1))
    return synth.BAProblem(poses=np.ascontiguousarray(np.concatenate([q0, t0.astype(np.float32).astype(np.float64)], -1)), intr=intr,
                           fixed=fixed, points=pts0, obs_kf=kf, obs_mp=mp, obs_uv=uv.astype(np.float32),
                           obs_w=(1.0 / sigma ** 2).astype(np.float32), name="landmark-sizes")


_p = {}


def problem():
    if "p" not in _p:
        _p["p"] = make_problem()
        assert set(SPECIAL) <= set(np.bincount(_p["p"].obs_mp).tolist())
    return _p["p"]


@pytest.mark.parametrize("lam_kind", ["lm_start", "heavy"])
def test_schur_system_and_step_match_the_restatement(lam_kind):
    p = problem()
    h = api.BAHandle(p)
    try:
        b = h.debug_build(huber_delta=api.HUBER_GBA)
        md = max(np.abs(np.einsum("kii->ki", b["Hpp"])).max(), np.abs(np.einsum("kii->ki", b["Hll"])).max())
        lam = (1e-5 if lam_kind == "lm_start" else 1e-1) * md
        ref = R.schur_reference(p, b, lam)
        got = h.debug_schur(lam, huber_delta=api.HUBER_GBA)
        r = R.compare_blocks(ref, h.debug_schur_blocks())
        d, dt = ref.dx_point(got["dx_pose"])
        r["dx_point"] = R.ratio(got["dx_point"] - d, dt)
    finally:
        h.close()
    assert max(r.values()) <= 1.0, r


def test_linear_system_matches_oracle(oracle):
    p = problem()
    ref = oracle.ba_build(p, huber_delta=api.HUBER_GBA)
    h = api.BAHandle(p)
    got = h.debug_build(huber_delta=api.HUBER_GBA)
    h.close()
    for k in ("Hpp", "bp", "Hll", "bl", "W"):
        assert np.abs(got[k] - ref[k]).max() <= 1e-9 * np.abs(ref[k]).max(), k


def test_per_landmark_sums_are_deterministic():
    h = api.BAHandle(problem())
    a = h.debug_build(huber_delta=api.HUBER_GBA)
    b = h.debug_build(huber_delta=api.HUBER_GBA)
    h.close()
    for k in ("Hll", "bl", "W", "Hpp", "bp"):
        assert np.array_equal(a[k], b[k]), k
    assert a["chi2_robust_sum"] == b["chi2_robust_sum"]


def test_lm_with_rejected_trials_matches_oracle(oracle):
    """started with far too little damping, the first iteration rejects trials (six here) and recomputes Z at each larger lambda"""
    p = problem()
    ref = oracle.ba_solve(p, iterations=10, huber_delta=api.HUBER_GBA, lambda_init=1e-9)
    assert ref["trials_total"] > ref["iters_done"], "the problem must reject a trial: the Z-only pass is under test"
    res = api.ba_solve(p, iterations=10, huber_delta=api.HUBER_GBA, lambda_init=1e-9)
    assert res["iters_done"] == ref["iters_done"]
    assert res["trials_total"] == ref["trials_total"]
    assert res["pcg_not_converged"] == 0
    n = len(ref["trace"])
    assert np.allclose(res["trace"][:n, 2], ref["trace"][:, 2], rtol=1e-7)
    assert np.array_equal(res["trace"][:n, 4], ref["trace"][:, 4])
    Tg = api.poses_to_Tcw_f32(res["poses"]).astype(np.float64); To = api.poses_to_Tcw_f32(ref["poses"]).astype(np.float64)
    assert np.abs(Tg - To).max() <= 1e-4 * max(1.0, np.abs(To).max())
    pg = res["points"].astype(np.float32).astype(np.float64); po = ref["points"].astype(np.float32).astype(np.float64)
    assert np.abs(pg - po).max() <= 1e-4 * max(1.0, np.abs(po).max())

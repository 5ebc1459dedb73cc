"""The reduced camera system on the GPU, block by block: the Schur product kernel (k_schur_mma) against the f64 restatement of
tests/schur_ref.py, fed with the device's own linear system (ccm_ba_debug_build) so that only the Z pass, the Schur kernel,
k_finalize_S, k_block_jacobi, the solve and k_backsub_points are under test.  Every entry of S and b_schur, and every landmark
step, is held to its own bound (TAU = 1e-12 times the absolute sum of its terms); a failure names the case and the worst block."""
import numpy as np
import pytest

from ccm_slam_b200 import api, synth
from tests import schur_ref as R

pytestmark = pytest.mark.gpu

SHAPES = {
    "tiny": lambda: synth.make_config("tiny"),
    "small": lambda: synth.make_config("small"),
    "cfg2": lambda: synth.make_config("cfg2"),
    "cfg4": lambda: synth.make_config("cfg4"),
    "cfg5_tenth": lambda: synth.make_config("cfg5", K=1000, P=100000),
    "awkward": synth.make_awkward_ba,
}


@pytest.fixture(scope="module", autouse=True)
def _dev():
    assert api.device_count() > 0, "no CUDA device: the product path has no CPU fallback"
    api.init(0)


_cache = {}


def _case(name, robust):
    """problem, the device's own linear system, and the max diagonal (lambda scale): once per (shape, robust)"""
    key = (name, robust)
    if key not in _cache:
        p = SHAPES[name]()
        h = api.BAHandle(p)
        b = h.debug_build(robust=robust, huber_delta=api.HUBER_GBA)
        h.close()
        md = max(np.abs(np.einsum("kii->ki", b["Hpp"])).max(), np.abs(np.einsum("kii->ki", b["Hll"])).max())
        _cache.clear()
        _cache[key] = (p, b, md)
    return _cache[key]


def _run(h, lam, robust):
    got = h.debug_schur(lam, robust=robust, huber_delta=api.HUBER_GBA)
    blk = h.debug_schur_blocks()
    return got, blk


def _check(ref, got, blk, label):
    r = R.compare_blocks(ref, blk)
    d, dt = ref.dx_point(got["dx_pose"])
    r["dx_point"] = R.ratio(got["dx_point"] - d, dt)
    worst = R.worst_block(ref, blk)
    return r, f"{label}: err/tol {r}, worst block (row {worst[0]}, col {worst[1]}) at {worst[2]:.3g}"


@pytest.mark.parametrize("robust", [True, False], ids=["robust", "plain"])
@pytest.mark.parametrize("lam_kind", ["lm_start", "heavy"])
@pytest.mark.parametrize("name", list(SHAPES))
def test_schur_kernel_matches_the_restatement(name, lam_kind, robust, capsys):
    p, b, md = _case(name, robust)
    lam = (1e-5 if lam_kind == "lm_start" else 1e-1) * md
    ref = R.schur_reference(p, b, lam)
    label = f"{name} {lam_kind} {'robust' if robust else 'plain'}"
    h = api.BAHandle(p)
    try:
        got, blk = _run(h, lam, robust)
    finally:
        h.close()
    r, msg = _check(ref, got, blk, label)
    with capsys.disabled():
        print(f"\n[schur {label}] err/tol S {r['S']:.3g} b {r['bschur']:.3g} dx {r['dx_point']:.3g}")
    assert max(r.values()) <= 1.0, msg


@pytest.mark.parametrize("name", ["tiny", "small"])
def test_schur_system_and_step_match_oracle(oracle, name):
    """The step against the oracle's exact factorisation (S itself is checked block by block above)."""
    p = synth.make_config(name)
    lam = 1e-5 * max(np.abs(np.einsum("kii->ki", oracle.ba_build(p, huber_delta=api.HUBER_GBA)["Hpp"])).max(), 1.0)
    ref = oracle.ba_schur_solve(p, lam, huber_delta=api.HUBER_GBA, dense=True)
    h = api.BAHandle(p)
    got = h.debug_schur(lam, huber_delta=api.HUBER_GBA, dense=True)
    rel = lambda a, b: np.abs(a - b).max() / max(np.abs(b).max(), 1e-300)
    assert rel(got["S"], ref["S"]) < 1e-9
    assert rel(got["bschur"], ref["bschur"]) < 1e-9
    assert got["pcg_relres"] < 1e-12
    assert rel(got["dx_pose"], ref["dx_pose"]) < 1e-6
    assert rel(got["dx_point"], ref["dx_point"]) < 1e-6
    h.close()

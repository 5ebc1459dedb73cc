"""The default coarse space of the PCG preconditioner steps from 256 to 320 nodes at Kf = 8192 free poses (cfg5 has 9999): the
size rule on both sides of the step, and the solve at the larger default checked on the exported system against a float64
direct solve, with the same bounds as test_gpu_pcg.py."""
import numpy as np
import pytest
import scipy.sparse as sp
import scipy.sparse.linalg as spla

from ccm_slam_b200 import api, synth

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module", autouse=True)
def _dev():
    assert api.device_count() > 0, "no CUDA device: the product path has no CPU fallback"
    api.init(0)


def coarse_shape(n, nc_max):
    """pcg_coarse_shape (pcg.cuh): aggregate size and node count for n block rows and at most nc_max nodes"""
    if nc_max <= 0 or n <= 0:
        return 0, 0
    agg = max(1, -(-n // nc_max))
    return agg, -(-n // agg)


def _problem(K):
    return synth.make_config("cfg5", K=K, P=8 * K)


@pytest.mark.parametrize("K,nc_max", [(8192, 256), (8193, 320)])
def test_default_coarse_size_steps_at_8192_free_poses(K, nc_max, monkeypatch):
    for k in ("CCM_PCG_NC", "CCM_PCG_IMPL", "CCM_PCG_PROLONG"):
        monkeypatch.delenv(k, raising=False)
    p = _problem(K)
    Kf = int((p.fixed == 0).sum())
    h = api.BAHandle(p)
    try:
        paths = h.debug_paths()
    finally:
        h.close()
    assert (Kf >= 8192) == (nc_max == 320)
    agg, nc = coarse_shape(Kf, nc_max)
    assert paths["pcg_impl"] == 2 and paths["pcg_agg"] == agg and paths["pcg_nc"] == nc, paths


def test_solve_at_the_larger_default(monkeypatch, capsys):
    for k in ("CCM_PCG_NC", "CCM_PCG_IMPL", "CCM_PCG_PROLONG"):
        monkeypatch.delenv(k, raising=False)
    p = _problem(8193)
    h = api.BAHandle(p)
    try:
        paths = h.debug_paths()
        b = h.debug_build(huber_delta=api.HUBER_GBA)
        lam = 1e-5 * max(np.abs(np.einsum("kii->ki", b["Hpp"])).max(), np.abs(np.einsum("kii->ki", b["Hll"])).max())
        got = h.debug_schur(lam, huber_delta=api.HUBER_GBA)
        blk = h.debug_schur_blocks()
    finally:
        h.close()
    free = np.flatnonzero(p.fixed == 0)
    slot = np.full(p.K, -1); slot[free] = np.arange(free.size)
    S = sp.bsr_matrix((blk["val"], slot[blk["col"]], np.concatenate([[0], np.cumsum(np.diff(blk["rowptr"])[free])])),
                      shape=(6 * free.size, 6 * free.size)).tocsc()
    bv = blk["bschur"][free].ravel()
    x = got["dx_pose"][free].ravel()
    true = np.linalg.norm(S @ x - bv) / np.linalg.norm(bv)
    xs = spla.splu(S).solve(bv)
    xrel = np.abs(x - xs).max() / np.abs(xs).max()
    with capsys.disabled():
        print(f"\n[pcg default coarse] Kf {free.size} nc {paths['pcg_nc']} iters {got['pcg_iters']} true relres {true:.3g} "
              f"reported {got['pcg_relres']:.3g} x vs splu {xrel:.3g}")
    assert paths["pcg_nc"] == coarse_shape(free.size, 320)[1]
    assert true <= 1e-10
    rep = got["pcg_relres"]
    assert (true < 1e-12 and rep < 1e-12) or rep / 10 <= true <= 10 * rep
    assert xrel <= 1e-6

"""k_pcg2's mirrored stream: inside a CTA's own rows each upper block is applied twice from one copy and its mirror is not streamed.
The items the device plans are compared block for block with the numpy restatement of tools/pcg2_bytes.py, and the solve of the
exported system with splu: on cfg5 at 1/10 length (CTA cuts inside the band) with the coarse level on and off, on the loop-closure
scene, and with four CTAs, where the warps' slabs overflow and the fallback to the full stream runs."""
import os
import sys

import numpy as np
import pytest
import scipy.sparse as sp
import scipy.sparse.linalg as spla

from ccm_slam_b200 import api, synth
from tests import schur_setup_scenes as SC

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools"))
import pcg2_bytes as PB  # noqa: E402

pytestmark = pytest.mark.gpu

_cache = {}


def _problem(name):
    if name not in _cache:
        _cache.clear()
        _cache[name] = synth.make_config("cfg5", K=1000, P=100000) if name == "cfg5_tenth" else SC.SCENES[name]()
    return _cache[name]


@pytest.fixture(scope="module", autouse=True)
def _dev():
    assert api.device_count() > 0, "no CUDA device: the product path has no CPU fallback"
    api.init(0)


def _solve(p, monkeypatch, env):
    monkeypatch.setenv("CCM_PCG_IMPL", "2")
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    h = api.BAHandle(p)
    try:
        plan = h.debug_pcg2()
        b = h.debug_build(huber_delta=api.HUBER_GBA)
        lam = 1e-5 * max(np.abs(np.einsum("kii->ki", b["Hpp"])).max(), np.abs(np.einsum("kii->ki", b["Hll"])).max())
        got = h.debug_schur(lam, huber_delta=api.HUBER_GBA)
        blk = h.debug_schur_blocks()
    finally:
        h.close()
    return plan, got, blk


CASES = [("cfg5_tenth", {}), ("cfg5_tenth", {"CCM_PCG_NC": "0"}), ("loop_closure", {}), ("cfg5_tenth", {"CCM_PCG2_GRID": "4"})]
IDS = ["cfg5_tenth-coarse", "cfg5_tenth-nocoarse", "loop_closure", "cfg5_tenth-4ctas"]


@pytest.mark.parametrize("name,env", CASES, ids=IDS)
def test_items_and_solve(name, env, monkeypatch, capsys):
    p = _problem(name)
    plan, got, blk = _solve(p, monkeypatch, env)
    rowptr, col = PB.pattern(p)
    grid = len(plan["cta_row"]) - 1
    cut = PB.cta_cut(rowptr, sms=grid)
    assert np.array_equal(plan["cta_row"], cut)
    ref = PB.plan(rowptr, col, cut)
    assert np.array_equal(plan["cta_item"], ref["cta_item"])
    assert np.array_equal(plan["slab_lo"], ref["slab_lo"])
    assert plan["items"].shape == ref["items"].shape and np.array_equal(plan["items"], ref["items"])
    assert plan["streamed"] == ref["streamed"] < len(col)
    # the solve against splu on the exported S
    free = SC.free_poses(p)
    slot = np.full(p.K, -1); slot[free] = np.arange(free.size)
    S = sp.bsr_matrix((blk["val"], slot[blk["col"]], np.concatenate([[0], np.cumsum(np.diff(blk["rowptr"])[free])])),
                      shape=(6 * free.size, 6 * free.size)).tocsc()
    bv = blk["bschur"][free].ravel()
    x = got["dx_pose"][free].ravel()
    true = np.linalg.norm(S @ x - bv) / np.linalg.norm(bv)
    xs = spla.splu(S).solve(bv)
    xrel = np.abs(x - xs).max() / np.abs(xs).max()
    tr = int(sum(bin(int(f) >> 4).count("1") for f in plan["items"][:, 3]))
    with capsys.disabled():
        print(f"\n[pcg2 mirror {name} {env}] ctas {grid} streamed {plan['streamed']} of {len(col)} blocks, transposed {tr}, "
              f"iters {got['pcg_iters']} true relres {true:.3g} x vs splu {xrel:.3g}")
    assert true <= 1e-10 and xrel <= 1e-6


def test_two_solves_without_the_coarse_level_are_bit_identical(monkeypatch):
    p = _problem("cfg5_tenth")
    xs = [_solve(p, monkeypatch, {"CCM_PCG_NC": "0"})[1]["dx_pose"] for _ in range(2)]
    assert np.array_equal(xs[0], xs[1])

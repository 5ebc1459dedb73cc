"""The PCG solves of the reduced camera system, checked on the exported S and b_schur (ccm_ba_debug_schur_blocks) instead of the
residual the kernel reports about itself: every k_pcg CTA shape, the coarse space off and on (constant and piecewise-linear
prolongation, odd and even Gauss-Jordan sweep counts, a coarse size that is not a multiple of 8), and k_pcg2 with an odd sweep
count and with the largest coarse system its shared memory holds (6 nc = 2304).  At K = 4500 (the 512 / 1024-thread CTAs, 256
coarse nodes, refresh 4) one LM run at the default settings is also compared with the oracle."""
import os
import subprocess
import sys

import numpy as np
import pytest
import scipy.sparse as sp
import scipy.sparse.linalg as spla

from ccm_slam_b200 import api, synth

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GJB = 8   # pivots per Gauss-Jordan sweep (pcg.cuh)


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


_problems = {}


def _problem(name):
    if name not in _problems:
        _problems.clear()
        _problems[name] = {
            "small": lambda: synth.make_config("small"),
            "cfg4": lambda: synth.make_config("cfg4"),
            "cfg5_tenth": lambda: synth.make_config("cfg5", K=1000, P=100000),
            "cfg5_768": lambda: synth.make_config("cfg5", K=769, P=77000),
            "cfg5_4500": lambda: synth.make_config("cfg5", K=4500, P=60000),
        }[name]()
    return _problems[name]


def _solve_and_check(p, monkeypatch, env):
    for k, v in env.items():
        monkeypatch.setenv(k, v)
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
    rows = np.repeat(np.arange(p.K), np.diff(blk["rowptr"]))
    S = sp.bsr_matrix((blk["val"], slot[blk["col"]], np.concatenate([[0], np.cumsum(np.diff(blk["rowptr"])[free])])),
                      shape=(6 * free.size, 6 * free.size)).tocsc()
    assert np.all(slot[rows] >= 0)
    bv = blk["bschur"][free].ravel()
    x = got["dx_pose"][free].ravel()
    true = np.linalg.norm(S @ x - bv) / np.linalg.norm(bv)
    xs = spla.splu(S).solve(bv)
    xrel = np.abs(x - xs).max() / np.abs(xs).max()
    return paths, dict(true_relres=true, reported=got["pcg_relres"], iters=got["pcg_iters"], x_vs_splu=xrel)


# (label, problem, env, expected impl, CTA, coarse nodes)
CASES = [
    ("k_pcg-256x2-default", "small", {}, 1, 256, coarse_shape(39, 128)[1]),
    ("k_pcg-256x2-nocoarse", "cfg4", {"CCM_PCG_NC": "0"}, 1, 256, 0),
    ("k_pcg-256x2-prolong0", "cfg4", {"CCM_PCG_PROLONG": "0"}, 1, 256, coarse_shape(799, 128)[1]),
    ("k_pcg-256x2-prolong1", "cfg4", {"CCM_PCG_PROLONG": "1"}, 1, 256, coarse_shape(799, 128)[1]),
    ("k_pcg-odd-sweeps", "cfg4", {"CCM_PCG_NC": "100"}, 1, 256, 100),
    ("k_pcg-nC-not-8k-odd", "cfg4", {"CCM_PCG_NC": "97"}, 1, 256, coarse_shape(799, 97)[1]),
    ("k_pcg2-odd-sweeps", "cfg5_tenth", {"CCM_PCG_IMPL": "2", "CCM_PCG_NC": "100"}, 2, 256, 100),
    ("k_pcg2-even-sweeps", "cfg5_tenth", {"CCM_PCG_IMPL": "2"}, 2, 256, coarse_shape(999, 128)[1]),
    ("k_pcg2-nC2304", "cfg5_768", {"CCM_PCG_IMPL": "2", "CCM_PCG_NC": "384"}, 2, 256, 384),
    ("k_pcg-512x1", "cfg5_4500", {"CCM_PCG_IMPL": "1"}, 1, 512, coarse_shape(4499, 256)[1]),
    ("k_pcg-1024x1", "cfg5_4500", {"CCM_PCG_IMPL": "1", "CCM_PCG_BLOCK": "1024"}, 1, 1024, coarse_shape(4499, 256)[1]),
    ("k_pcg2-512-setup", "cfg5_4500", {}, 2, 512, coarse_shape(4499, 256)[1]),
]


@pytest.mark.parametrize("label,name,env,impl,cta,nc", CASES, ids=[c[0] for c in CASES])
def test_pcg_path_solves_the_exported_system(label, name, env, impl, cta, nc, monkeypatch, capsys):
    p = _problem(name)
    paths, r = _solve_and_check(p, monkeypatch, env)
    Kf = int((p.fixed == 0).sum())
    assert paths["pcg_impl"] == impl and paths["pcg_block"] == cta and paths["pcg_nc"] == nc, paths
    if nc:
        assert paths["pcg_agg"] == coarse_shape(Kf, int(env.get("CCM_PCG_NC", 0)) or (256 if Kf >= 4096 else 128))[0]
    nC = 6 * nc
    with capsys.disabled():
        print(f"\n[pcg {label}] Kf {Kf} nC {nC} sweeps {-(-nC // GJB)} iters {r['iters']} true relres {r['true_relres']:.3g} "
              f"reported {r['reported']:.3g} x vs splu {r['x_vs_splu']:.3g}")
    assert r["true_relres"] <= 1e-10
    assert (r["true_relres"] < 1e-12 and r["reported"] < 1e-12) or r["reported"] / 10 <= r["true_relres"] <= 10 * r["reported"]
    assert r["x_vs_splu"] <= 1e-6


def test_sweep_parities_are_covered():
    """the cases above reach both parities of the Gauss-Jordan sweep count on k_pcg2, a coarse size that is not a multiple of 8,
    and the 6 nc == P2_MAX_NC boundary"""
    sweeps = {c[0]: -(-6 * c[5] // GJB) for c in CASES}
    assert sweeps["k_pcg2-odd-sweeps"] % 2 == 1 and sweeps["k_pcg2-even-sweeps"] % 2 == 0
    assert sweeps["k_pcg-odd-sweeps"] % 2 == 1
    assert (6 * dict((c[0], c[5]) for c in CASES)["k_pcg-nC-not-8k-odd"]) % 8 != 0
    assert 6 * dict((c[0], c[5]) for c in CASES)["k_pcg2-nC2304"] == 2304


def test_k4500_lm_matches_oracle(oracle):
    """default settings at Kf >= 4224: k_pcg2 with the 512-thread k_pcg set-up, 256 coarse nodes and the coarse inverse reused
    across trials (refresh 4)"""
    p = _problem("cfg5_4500")
    ref = oracle.ba_solve(p, iterations=20, huber_delta=api.HUBER_GBA)
    res = api.ba_solve(p, iterations=20, huber_delta=api.HUBER_GBA, want_edges=False)
    assert res["iters_done"] == ref["iters_done"] and res["trials_total"] == ref["trials_total"]
    n = len(ref["trace"])
    assert np.allclose(res["trace"][:n, 1], ref["trace"][:, 1], rtol=1e-6)
    assert np.allclose(res["trace"][:n, 2], ref["trace"][:, 2], rtol=1e-7)
    assert np.array_equal(res["trace"][:n, 4], ref["trace"][:, 4])
    assert res["pcg_not_converged"] == 0
    Tg = api.poses_to_Tcw_f32(res["poses"]).astype(np.float64); To = api.poses_to_Tcw_f32(ref["poses"]).astype(np.float64)
    assert np.abs(Tg - To).max() <= 1e-4 * max(1.0, np.abs(To).max())
    pg = res["points"].astype(np.float32).astype(np.float64); po = ref["points"].astype(np.float32).astype(np.float64)
    assert np.abs(pg - po).max() <= 1e-4 * max(1.0, np.abs(po).max())


_LIN = """
import sys, numpy as np
sys.path.insert(0, {root!r})
from ccm_slam_b200 import api, synth
api.init(0)
h = api.BAHandle(synth.make_config("small"))
b = h.debug_build(huber_delta=api.HUBER_GBA)
np.savez({out!r}, **{{k: v for k, v in b.items()}})
"""


def test_linearize_builds_agree(tmp_path):
    """k_linearize<2> / <3> (CCM_LIN_MINB, read once per process) against the default <4>"""
    out = {}
    for minb in ("4", "2", "3"):
        f = str(tmp_path / f"lin{minb}.npz")
        env = dict(os.environ, CCM_LIN_MINB=minb)
        subprocess.run([sys.executable, "-c", _LIN.format(root=ROOT, out=f)], env=env, check=True)
        out[minb] = dict(np.load(f))
    for minb in ("2", "3"):
        for k in ("Hpp", "bp", "Hll", "bl", "W"):
            a, b = out[minb][k], out["4"][k]
            assert np.abs(a - b).max() <= 1e-12 * np.abs(b).max(), (minb, k)

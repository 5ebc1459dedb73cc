"""The reduced camera system on the GPU, block by block: every Schur kernel variant (CCM_SCHUR 0-17, sorted lists, tile edges, the
landmark-synchronous panels) against the f64 restatement of tests/schur_ref.py, fed with the device's own linear system
(ccm_ba_debug_build) so that only k_scale, the Schur kernels, k_finalize_S, k_block_jacobi, the solve and k_backsub_points are
under test.  Every entry of S and b_schur, and every landmark step, is held to its own bound (TAU = 1e-12 times the absolute
sum of its terms); a failure names the configuration and the worst block."""
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
LIST_MODES = [m for m in range(18) if m not in (9, 10, 16, 17)]   # share one handle: the mode is read at launch
BIG = "1000000"


def _configs():
    """(label, mode, env, fresh handle)"""
    c = [(f"mode{m}", m, {}, False) for m in LIST_MODES]
    c += [(f"mode{m}", m, {}, True) for m in (9, 10, 16, 17)]
    c += [(f"mode{m}+sort", m, {"CCM_SCHUR_SORT": "1"}, True) for m in list(range(1, 9)) + list(range(11, 16))]
    c += [(f"mode9+tile{t}", 9, {"CCM_SCHUR_TILE": str(t)}, True) for t in (3, 4)]
    for fac in ("default", "all"):
        env = {"CCM_SCHUR_PANEL": "1"} if fac == "default" else {"CCM_SCHUR_PANEL": "1", "CCM_SCHUR_PANEL_FACTOR": BIG}
        c += [(f"panel-{fac}+mode{m}", m, env, True) for m in range(16)]
    return c


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


def _check(ref, got, blk, label, table):
    r = R.compare_blocks(ref, blk)
    d, dt = ref.dx_point(got["dx_pose"])
    r["dx_point"] = R.ratio(got["dx_point"] - d, dt)
    table.append((label, r))
    worst = R.worst_block(ref, blk)
    return r, f"{label}: err/tol {r}, worst block (row {worst[0]}, col {worst[1]}) at {worst[2]:.3g}"


def _expect_path(label, mode, env, paths):
    assert paths["schur_mode"] == mode, (label, paths)
    if env.get("CCM_SCHUR_PANEL"):
        assert paths["panels"] > 0, (label, paths)
        if env.get("CCM_SCHUR_PANEL_FACTOR") == BIG:   # every panel on, and they own blocks
            assert paths["panels_on"] == paths["panels"] and paths["covered"] > 0, (label, paths)
    else:
        assert paths["panels"] == 0 and paths["covered"] == 0, (label, paths)


@pytest.mark.parametrize("robust", [True, False], ids=["robust", "plain"])
@pytest.mark.parametrize("lam_kind", ["lm_start", "heavy"])
@pytest.mark.parametrize("name", list(SHAPES))
def test_every_schur_variant_matches_the_restatement(name, lam_kind, robust, monkeypatch, capsys):
    p, b, md = _case(name, robust)
    lam = (1e-5 if lam_kind == "lm_start" else 1e-1) * md
    ref = R.schur_reference(p, b, lam)
    table, fails = [], []
    shared = None
    with api.schur_mode(11):
        shared = api.BAHandle(p)
    try:
        for label, mode, env, fresh in _configs():
            with monkeypatch.context() as mp:
                for k, v in env.items():
                    mp.setenv(k, v)
                with api.schur_mode(mode):
                    if mode in (16, 17) and env.get("CCM_SCHUR_PANEL"):
                        continue
                    if env.get("CCM_SCHUR_PANEL") and p.K - int(p.fixed.sum()) < 1:
                        continue
                    h = api.BAHandle(p) if fresh else shared
                    try:
                        paths = h.debug_paths()
                        if not (name == "tiny" and mode in (9, 10)):   # tiny: the row / tile schedule may be empty
                            _expect_path(label, mode, env, paths)
                        got, blk = _run(h, lam, robust)
                    finally:
                        if fresh:
                            h.close()
                r, msg = _check(ref, got, blk, label, table)
                if max(r.values()) > 1.0:
                    fails.append(msg)
    finally:
        shared.close()
    with capsys.disabled():
        worst = max(table, key=lambda t: max(t[1].values()))
        print(f"\n[schur {name} {lam_kind} {'robust' if robust else 'plain'}] {len(table)} variants, "
              f"max err/tol S {max(t[1]['S'] for t in table):.3g} b {max(t[1]['bschur'] for t in table):.3g} "
              f"dx {max(t[1]['dx_point'] for t in table):.3g} (worst: {worst[0]})")
    assert not fails, "\n".join(fails)


@pytest.mark.parametrize("mode", [16, 17])
def test_grouped_lists_with_panels_are_refused(mode, monkeypatch):
    monkeypatch.setenv("CCM_SCHUR_PANEL", "1")
    with api.schur_mode(mode):
        with pytest.raises(api.CCMError, match="alternatives"):
            api.BAHandle(synth.make_config("small"))


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

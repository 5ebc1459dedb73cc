"""GPU parity tests of the BA path: libccm_b200.so (through its C ABI) against the CPU oracle on identical inputs.

Tolerance: the north_star bar is 1e-4 relative on pose / landmark estimates after the same iteration count (compared
after the f32 round trip of the reference's write-back, S/Converter.cc:64-72); the kernel-level blocks are held to
1e-9 relative because both sides compute in f64."""
import numpy as np
import pytest

from ccm_slam_b200 import api, synth

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module", autouse=True)
def _dev():
    assert api.device_count() > 0, "no CUDA device: the product path has no CPU fallback"
    api.init(0)


def _relerr(a, b):
    return np.abs(a - b).max() / max(np.abs(b).max(), 1e-300)


def _state_close(res, ref, tol):
    Tg = api.poses_to_Tcw_f32(res["poses"]).astype(np.float64)
    To = api.poses_to_Tcw_f32(ref["poses"]).astype(np.float64)
    assert np.abs(Tg - To).max() <= tol * max(1.0, np.abs(To).max())
    pg = res["points"].astype(np.float32).astype(np.float64); po = ref["points"].astype(np.float32).astype(np.float64)
    assert np.abs(pg - po).max() <= tol * max(1.0, np.abs(po).max())


@pytest.mark.parametrize("name", ["tiny", "small", "cfg2"])
def test_linearisation_blocks_match_oracle(oracle, name):
    p = synth.make_config(name)
    ref = oracle.ba_build(p, huber_delta=api.HUBER_GBA)
    lin = oracle.ba_linearize(p, huber_delta=api.HUBER_GBA)
    h = api.BAHandle(p)
    got = h.debug_build(huber_delta=api.HUBER_GBA)
    for k in ("Hpp", "bp", "Hll", "bl", "W"):
        assert _relerr(got[k], ref[k]) < 1e-9, k
    assert abs(got["chi2_robust_sum"] - lin["chi2_robust_sum"]) <= 1e-10 * lin["chi2_robust_sum"]
    h.close()


@pytest.mark.parametrize("name,iters", [("tiny", 12), ("small", 10), ("cfg2", 15), ("cfg3", 20)])
def test_lm_matches_oracle_after_same_iteration_count(oracle, name, iters):
    p = synth.make_config(name)
    ref = oracle.ba_solve(p, iterations=iters, huber_delta=api.HUBER_GBA)
    res = api.ba_solve(p, iterations=iters, huber_delta=api.HUBER_GBA)
    assert res["iters_done"] == ref["iters_done"]
    assert res["trials_total"] == ref["trials_total"]
    assert res["pcg_not_converged"] == 0
    n = len(ref["trace"])
    assert np.allclose(res["trace"][:n, 1], ref["trace"][:, 1], rtol=1e-6)   # lambda schedule
    assert np.allclose(res["trace"][:n, 2], ref["trace"][:, 2], rtol=1e-7)   # robust chi2 per iteration
    assert np.array_equal(res["trace"][:n, 4], ref["trace"][:, 4])           # trials per iteration
    _state_close(res, ref, 1e-4)
    # per-edge outputs the LocalBA shim consumes
    assert np.allclose(res["chi2"], ref["chi2"], rtol=1e-6, atol=1e-9)
    assert np.array_equal(res["depth_pos"], ref["depth_pos"])


def test_unsorted_observations_give_the_same_answer(oracle):
    p = synth.make_config("small")
    rng = np.random.default_rng(3)
    perm = rng.permutation(p.E)
    q = p.copy()
    q.obs_kf, q.obs_mp, q.obs_uv, q.obs_w = p.obs_kf[perm], p.obs_mp[perm], p.obs_uv[perm], p.obs_w[perm]
    a = api.ba_solve(p, iterations=6)
    b = api.ba_solve(q, iterations=6)
    assert np.allclose(a["poses"], b["poses"], atol=1e-9)
    assert np.allclose(a["chi2"][perm], b["chi2"], rtol=1e-7, atol=1e-9)


def test_create_rejects_bad_observations():
    """ccm_ba_create validates the caller's arrays on the device (indices with the structure, the weights where their copy joins
    the stream) and fails loudly; grouped and ungrouped input take different paths, both must refuse."""
    p = synth.make_config("small")
    rng = np.random.default_rng(5)
    for shuffle in (False, True):
        base = p.copy()
        if shuffle:
            perm = rng.permutation(p.E)
            base.obs_kf, base.obs_mp, base.obs_uv, base.obs_w = p.obs_kf[perm], p.obs_mp[perm], p.obs_uv[perm], p.obs_w[perm]
        q = base.copy(); q.obs_w = base.obs_w.copy(); q.obs_w[p.E // 2] = -1.0
        with pytest.raises(api.CCMError, match="negative information weight"):
            api.BAHandle(q)
        q = base.copy(); q.obs_kf = base.obs_kf.copy(); q.obs_kf[7] = p.K
        with pytest.raises(api.CCMError, match="out of range"):
            api.BAHandle(q)
    h = api.BAHandle(p)   # and the library is still usable afterwards
    assert h.optimize(iterations=2)["iters_done"] >= 1
    h.close()


def test_local_ba_two_rounds_through_the_handle_api(oracle):
    """optimize(5) -> flag chi2>5.991 or depth<=0 as level 1 and drop the kernels -> optimize(10) (S/Optimizer.cpp:536-587)."""
    p = synth.make_config("cfg2")
    d = api.HUBER_LOCAL
    r1 = oracle.ba_solve(p, iterations=5, huber_delta=d)
    out_ref = (r1["chi2"] > 5.991) | (r1["depth_pos"] == 0)
    p2 = p.copy(); p2.poses = r1["poses"]; p2.points = r1["points"]; p2.edge_flags = (out_ref.astype(np.uint8) | 2)
    r2 = oracle.ba_solve(p2, iterations=10, huber_delta=d, chi2_in=r1["chi2"])

    h = api.BAHandle(p)
    g1 = h.optimize(iterations=5, huber_delta=d, want_edges=True)
    out = (g1["chi2"] > 5.991) | (g1["depth_pos"] == 0)
    assert np.array_equal(out, out_ref)
    h.set_edge_flags(out.astype(np.uint8) | 2)
    g2 = h.optimize(iterations=10, huber_delta=d, want_edges=True, chi2_in=g1["chi2"])
    assert np.array_equal(g2["chi2"][out], g1["chi2"][out])  # level-1 edges keep their round-1 chi2
    assert np.allclose(g2["trace"][:len(r2["trace"]), 2], r2["trace"][:, 2], rtol=1e-7)
    _state_close(g2, r2, 1e-4)
    erase_ref = (r2["chi2"] > 5.991) | (r2["depth_pos"] == 0)
    erase = (g2["chi2"] > 5.991) | (g2["depth_pos"] == 0)
    assert np.array_equal(erase, erase_ref)
    h.close()


def test_stop_flag_zero_iterations_reset(oracle):
    p = synth.make_config("small")
    stop = np.ones(1, np.uint8)
    r = api.ba_solve(p, iterations=20, stop=stop)
    assert r["iters_done"] == 0 and np.array_equal(r["poses"], p.poses) and np.array_equal(r["points"], p.points)
    h = api.BAHandle(p)
    a = h.optimize(iterations=4)
    h.reset()
    b = h.optimize(iterations=4)
    assert np.allclose(a["poses"], b["poses"], atol=1e-10) and a["trials_total"] == b["trials_total"]
    assert h.info()["K_free"] == p.K - 1
    h.close()


def test_set_estimate_keeps_the_structure_on_the_device(oracle):
    """A second global BA on a map that changed in value only (SURVEY.md 8(f) rank 1: the persistent mirror + a cached handle): the new
    estimate is uploaded with ccm_ba_set_estimate, structure and observations stay resident; the result equals a from-scratch solve."""
    p = synth.make_config("small")
    h = api.BAHandle(p)
    a = h.optimize(iterations=4, huber_delta=api.HUBER_GBA)
    h.set_estimate(a["poses"], a["points"])
    b = h.optimize(iterations=4, huber_delta=api.HUBER_GBA)
    q = p.copy(); q.poses = a["poses"].copy(); q.points = a["points"].copy()
    c = api.ba_solve(q, iterations=4, huber_delta=api.HUBER_GBA)
    ref = oracle.ba_solve(q, iterations=4, huber_delta=api.HUBER_GBA)
    assert b["iters_done"] == c["iters_done"] == ref["iters_done"] and b["trials_total"] == c["trials_total"] == ref["trials_total"]
    assert np.allclose(b["poses"], c["poses"], atol=1e-9) and np.allclose(b["points"], c["points"], atol=1e-9)
    _state_close(b, ref, 1e-4)
    h.set_estimate(p.poses, None)                                  # poses only: the points keep the last uploaded estimate
    d = h.optimize(iterations=1, huber_delta=api.HUBER_GBA)
    assert d["iters_done"] == 1
    h.close()


def test_degenerate_graphs_behave_like_the_oracle(oracle):
    """Empty and ragged inputs: no observations, every edge switched off, an unobserved landmark, a landmark seen once,
    a free keyframe without observations (g2o leaves vertices without active edges alone)."""
    p = synth.make_config("small")
    # (1) no observations at all: "0 vertices to optimize" -> -1, estimate untouched
    q = p.copy()
    q.obs_kf, q.obs_mp, q.obs_uv, q.obs_w = q.obs_kf[:0], q.obs_mp[:0], q.obs_uv[:0], q.obs_w[:0]
    ref = oracle.ba_solve(q, iterations=5, huber_delta=api.HUBER_GBA)
    res = api.ba_solve(q, iterations=5, huber_delta=api.HUBER_GBA)
    assert ref["iters_done"] == -1 and res["iters_done"] == -1
    assert np.array_equal(res["poses"], p.poses) and np.array_equal(res["points"], p.points)
    # (2) every edge at level 1 (flag bit 0): same
    q = p.copy()
    q.edge_flags = np.ones(p.E, np.uint8)
    ref = oracle.ba_solve(q, iterations=5, huber_delta=api.HUBER_GBA)
    res = api.ba_solve(q, iterations=5, huber_delta=api.HUBER_GBA)
    assert ref["iters_done"] == -1 and res["iters_done"] == -1
    assert np.array_equal(res["poses"], p.poses) and np.array_equal(res["points"], p.points)
    # (3) ragged: an unobserved landmark, a landmark left with one observation, a free keyframe nobody observes from
    q = p.copy()
    q.points = np.vstack([q.points, [[0.5, -0.25, 3.0]]])
    q.poses = np.vstack([q.poses, q.poses[-1:]])
    q.intr = np.vstack([q.intr, q.intr[-1:]])
    q.fixed = np.concatenate([q.fixed, np.zeros(1, np.uint8)])
    first = np.flatnonzero(q.obs_mp == q.obs_mp[0])
    keep = np.ones(q.E, bool)
    keep[first[1:]] = False  # landmark obs_mp[0] keeps a single observation
    q.obs_kf, q.obs_mp, q.obs_uv, q.obs_w = q.obs_kf[keep], q.obs_mp[keep], q.obs_uv[keep], q.obs_w[keep]
    ref = oracle.ba_solve(q, iterations=6, huber_delta=api.HUBER_GBA)
    res = api.ba_solve(q, iterations=6, huber_delta=api.HUBER_GBA)
    assert res["iters_done"] == ref["iters_done"] and res["trials_total"] == ref["trials_total"]
    _state_close(res, ref, 1e-4)
    assert np.array_equal(res["points"][-1], q.points[-1]) and np.array_equal(res["poses"][-1], q.poses[-1])


def test_cfg4_full_size_against_oracle_and_properties(oracle):
    """4-agent merged-map Global BA shape (the >=50x target shape) at full size."""
    p = synth.make_config("cfg4")
    ref = oracle.ba_solve(p, iterations=20, huber_delta=api.HUBER_GBA)
    res = api.ba_solve(p, iterations=20, huber_delta=api.HUBER_GBA)
    assert res["iters_done"] == ref["iters_done"] and res["trials_total"] == ref["trials_total"]
    assert np.allclose(res["trace"][:len(ref["trace"]), 2], ref["trace"][:, 2], rtol=1e-7)
    _state_close(res, ref, 1e-4)
    assert np.all(np.diff(res["trace"][:res["iters_done"], 2]) <= 0)       # accepted chi2 never increases
    assert np.array_equal(res["poses"][0], p.poses[0])                       # the fixed origin keyframe does not move


@pytest.mark.parametrize("impl", ["default", "streamed"])
def test_cfg5_tenth_scale_against_oracle_and_properties(oracle, impl, monkeypatch):
    """The benchmarked shape (cfg5: banded covisibility, 20 observations / landmark) at 1/10 trajectory length, K = 1000,
    P = 100 000, 2 M observations: the same stop rule as bench.py (optimize(20), ended by the three-strike rule) against the
    oracle's exact-factorisation run (about 10 s of CPU) -- iteration and trial counts, lambda schedule, chi2 trace, state --
    plus the size-independent properties."""
    if impl == "streamed":   # the kernel the full-size cfg5 takes (k_pcg2); at 1/10 length the size rule would pick the small-system one
        monkeypatch.setenv("CCM_PCG_IMPL", "2")
    p = synth.make_config("cfg5", K=1000, P=100000)
    ref = oracle.ba_solve(p, iterations=20, huber_delta=api.HUBER_GBA)
    res = api.ba_solve(p, iterations=20, huber_delta=api.HUBER_GBA, want_edges=False)
    assert res["iters_done"] == ref["iters_done"] and res["trials_total"] == ref["trials_total"]
    n = len(ref["trace"])
    assert np.allclose(res["trace"][:n, 1], ref["trace"][:, 1], rtol=1e-6)   # lambda schedule
    assert np.allclose(res["trace"][:n, 2], ref["trace"][:, 2], rtol=1e-7)   # robust chi2 per iteration
    assert np.array_equal(res["trace"][:n, 4], ref["trace"][:, 4])           # trials per iteration
    _state_close(res, ref, 1e-4)
    tr = res["trace"]
    assert res["iters_done"] == 8 and res["pcg_not_converged"] == 0
    assert np.all(np.diff(tr[:, 2]) <= 0) and tr[-1, 2] < 0.2 * res["chi2_initial"]
    assert np.array_equal(res["poses"][0], p.poses[0])
    assert np.isfinite(res["points"]).all() and np.isfinite(res["poses"]).all()
    assert np.allclose(np.linalg.norm(res["poses"][:, :4], axis=1), 1.0, atol=1e-12)

"""The reduced camera system's set-up at its edges: on scenes built to sit exactly on one boundary each (tests/schur_setup_scenes.py:
rows of ROWP_CUR and ROWP_CUR + 1 upper blocks, rows cut into one, two or three Schur tasks, Kf around 2^8 with fixed poses among the
free ones, Kf around the 32-bit words of the covisibility bitmap, free poses without observations or with a diagonal block only, a
landmark shard, a system of diagonal blocks only), every scene is checked for
  * the pattern of S against the free-pose pairs that share a landmark, plus every diagonal;
  * the product lists against the numpy pairs in landmark order, and the Schur kernel's schedule against its definition;
  * S, b_schur and the landmark step against the f64 restatement of tests/schur_ref.py, entry by entry;
  * Hpp and bp of the pose pass (which reads the diagonal product lists) against tests/ba_ref.py;
  * bit-identical lists, S, b_schur, Hpp and final state between two creates, between the observations in shuffled order and
    grouped, after set_estimate against a fresh create at that state, and after reset.
The loop-closure scene also runs LM against the oracle."""
import numpy as np
import pytest

from ccm_slam_b200 import api
from tests import ba_ref as F
from tests import schur_ref as R
from tests import schur_setup_scenes as SC
from tests.test_gpu_ba import _state_close
from tests.test_gpu_schur_order import _collect, _everything, _expected, _same, _same_as_grouped, _shuffled

pytestmark = pytest.mark.gpu

NAMES = list(SC.SCENES)
_scenes = {}


def scene(name):
    if name not in _scenes:
        _scenes[name] = SC.SCENES[name]()
    return _scenes[name]


@pytest.fixture(scope="module")
def dev():
    assert api.device_count() > 0, "no CUDA device: the product path has no CPU fallback"
    api.init(0)


def test_scenes_sit_on_the_boundaries():
    """each scene lands where its name says (numpy only)"""
    for name, edge in SC.EDGES.items():
        p = scene(name)
        free = SC.free_poses(p)
        Kf = free.size
        nu = SC.row_lengths(p)
        if "Kf" in edge:
            assert Kf == edge["Kf"], name
        for a, n in edge.get("rows", {}).items():
            assert nu[a] == n, f"{name}: row {a} has {nu[a]} upper blocks, not {n}"
        if edge.get("fixed_among_free"):
            fixed = np.flatnonzero(p.fixed)
            assert np.any((fixed > free[0]) & (fixed < free[-1])), name
            assert np.isin(fixed, p.obs_kf).all(), f"{name}: a fixed pose without observations"
        if "max_row" in edge:
            assert nu.max() == edge["max_row"], name
        for k in edge.get("no_obs", []):
            assert p.fixed[k] == 0 and not np.any(p.obs_kf == k), name
        for k in edge.get("diag_only_rows", []):
            a = int(np.searchsorted(free, k))
            ra, rb = SC.covis_pairs(p)
            assert p.fixed[k] == 0 and np.any(p.obs_kf == k) and np.sum((ra == a) | (rb == a)) == 1, name
        if edge.get("empty_rows"):
            assert np.sum(~np.isin(free, p.obs_kf)) > 100, name
        if "longest_over" in edge:
            assert nu.max() > edge["longest_over"], name
    # the radix sort's key width steps up at Kf = 2^k; the bitmap gains a word after Kf = 32 and 64
    k = SC.KF_EDGE
    assert [SC.sort_bits(SC.free_poses(scene(f"kf{(1 << k) + d}")).size) for d in (-1, 0, 1)] == [k, k + 1, k + 1]
    assert [-(-SC.free_poses(scene(f"kf{n}")).size // 32) for n in (31, 32, 33, 63, 64, 65)] == [1, 1, 2, 2, 2, 3]
    # 64 / 65 and 128 / 129 blocks across task counts
    assert [-(-n // SC.SCHUR_TASK) for n in SC.EDGES["task_cut"]["rows"].values()] == [1, 2, 2, 3]


def _pattern_msg(name, got_r, got_c, ref_r, ref_c):
    g = set(zip(got_r.tolist(), got_c.tolist())); r = set(zip(ref_r.tolist(), ref_c.tolist()))
    extra, missing = sorted(g - r)[:3], sorted(r - g)[:3]
    return f"{name}: pattern of S differs: extra blocks {extra}, missing blocks {missing}"


@pytest.mark.parametrize("name", NAMES)
def test_pattern_lists_and_schedule(dev, name):
    p = scene(name)
    h = api.BAHandle(p)
    try:
        blocks = h.debug_schur_blocks()
        lists = h.debug_products()
        sched = h.debug_schedule()
    finally:
        h.close()
    # pattern: both triangles of the free-pose covisibility, in pose indices
    free = SC.free_poses(p)
    a, b = SC.covis_pairs(p)
    rr = np.concatenate([free[a], free[b][a != b]]); cc = np.concatenate([free[b], free[a][a != b]])
    o = np.lexsort((cc, rr)); rr, cc = rr[o], cc[o]
    rowptr = np.searchsorted(rr, np.arange(p.K + 1))
    got_r = np.repeat(np.arange(p.K), np.diff(blocks["rowptr"]))
    assert np.array_equal(blocks["rowptr"], rowptr) and np.array_equal(blocks["col"], cc), \
        _pattern_msg(name, got_r, blocks["col"], rr, cc)
    # product lists
    blk, ptr, pairs = lists["blk"], lists["ptr"], lists["pairs"]
    n = np.diff(ptr)
    assert np.array_equal(blk[:, 0], free[a]) and np.array_equal(blk[:, 1], free[b]), f"{name}: upper blocks differ from the pattern"
    first = np.zeros(pairs.shape[0], bool); first[ptr[:-1][n > 0]] = True
    bad = np.flatnonzero(~((np.diff(pairs[:, 0]) > 0) | first[1:]))
    if bad.size:
        u = int(np.searchsorted(ptr, bad[0] + 1, side="right") - 1)
        pytest.fail(f"{name}: the list of block {tuple(blk[u])} is not strictly increasing in e")
    ea, eb, e, oo = _expected(p)
    assert pairs.shape[0] == e.size, f"{name}: {pairs.shape[0]} products, expected {e.size}"
    row = np.repeat(blk[:, 0], n); col = np.repeat(blk[:, 1], n)
    diff = np.flatnonzero((row != ea) | (col != eb) | (pairs[:, 0] != e) | (pairs[:, 1] != oo))
    if diff.size:
        q = diff[0]
        pytest.fail(f"{name}: lists differ from the restatement, first at block ({ea[q]}, {eb[q]}) product {q}: "
                    f"got {tuple(pairs[q])}, expected ({e[q]}, {oo[q]})")
    # schedule: per row its blocks by decreasing list length (ties by block number), cut into ceil(n / SCHUR_TASK) tasks
    Kf = free.size
    nu = np.bincount(a, minlength=Kf)
    ustart = np.concatenate([[0], np.cumsum(nu)])
    tp = [0]; exp_sched = []
    for r in range(Kf):
        ub, m = int(ustart[r]), int(nu[r])
        us = np.arange(ub, ub + m)
        exp_sched.append(us[np.lexsort((us, -n[us]))])
        parts = -(-m // SC.SCHUR_TASK)
        tp += [ub + m * k // parts for k in range(1, parts + 1)]
    assert sched["ntasks"] == len(tp) - 1, f"{name}: {sched['ntasks']} tasks, expected {len(tp) - 1}"
    assert np.array_equal(sched["task_ptr"], tp), f"{name}: task boundaries differ"
    assert np.array_equal(sched["sched"], np.concatenate(exp_sched)), f"{name}: task order differs"
    assert 1 <= sched["grid"] <= sched["ntasks"]
    if name == "diag_only":
        assert sched["ntasks"] == Kf and lists["blk"].shape[0] == Kf
    if name == "one_free_pose":
        assert sched["ntasks"] == 1 and sched["grid"] == 1


_lin = {}


def _build(name, robust):
    """the device's own linear system and the max diagonal (lambda scale): once per (scene, robust)"""
    key = (name, robust)
    if key not in _lin:
        p = scene(name)
        h = api.BAHandle(p)
        try:
            b = h.debug_build(robust=robust, huber_delta=api.HUBER_GBA)
        finally:
            h.close()
        md = max(np.abs(np.einsum("kii->ki", b["Hpp"])).max(), np.abs(np.einsum("kii->ki", b["Hll"])).max())
        _lin.clear()
        _lin[key] = (b, md)
    return _lin[key]


@pytest.mark.parametrize("robust", [True, False], ids=["robust", "plain"])
@pytest.mark.parametrize("lam_kind", ["lm_start", "heavy"])
@pytest.mark.parametrize("name", NAMES)
def test_schur_matches_the_restatement(dev, name, lam_kind, robust, capsys):
    p = scene(name)
    b, md = _build(name, robust)
    lam = (1e-5 if lam_kind == "lm_start" else 1e-1) * md
    ref = R.schur_reference(p, b, lam)
    label = f"{name} {lam_kind} {'robust' if robust else 'plain'}"
    h = api.BAHandle(p)
    try:
        got = h.debug_schur(lam, robust=robust, huber_delta=api.HUBER_GBA)
        blk = h.debug_schur_blocks()
    finally:
        h.close()
    r = R.compare_blocks(ref, blk)
    d, dt = ref.dx_point(got["dx_pose"])
    r["dx_point"] = R.ratio(got["dx_point"] - d, dt)
    worst = R.worst_block(ref, blk)
    with capsys.disabled():
        print(f"\n[schur setup {label}] err/tol S {r['S']:.3g} b {r['bschur']:.3g} dx {r['dx_point']:.3g}")
    assert max(r.values()) <= 1.0, f"{label}: err/tol {r}, worst block (row {worst[0]}, col {worst[1]}) at {worst[2]:.3g}"


@pytest.mark.parametrize("robust", [True, False], ids=["robust", "plain"])
@pytest.mark.parametrize("name", NAMES)
def test_pose_pass_matches_the_restatement(dev, name, robust, capsys):
    p = scene(name)
    b, _ = _build(name, robust)
    L = F.Lin(p, robust=robust, delta=api.HUBER_GBA)
    out = {}
    for k in ("Hpp", "bp"):
        err, tol = np.abs(b[k] - getattr(L, k)), F.TAU * getattr(L, k + "_b")
        per = np.where(tol > 0, err / np.where(tol > 0, tol, 1.0), np.where(err > 0, np.inf, 0.0)).reshape(p.K, -1).max(1)
        out[k] = (float(per.max()), int(np.argmax(per)))
    with capsys.disabled():
        print(f"\n[pose pass {name} robust={robust}] err/tol Hpp {out['Hpp'][0]:.3g} bp {out['bp'][0]:.3g}")
    for k, (v, at) in out.items():
        assert v <= 1.0, f"{name} robust={robust}: {k} of pose {at} at err/tol {v:.3g}"


@pytest.mark.parametrize("name", NAMES)
def test_setup_is_deterministic(dev, name, monkeypatch):
    """two creates, the same observations in shuffled order against them grouped, a handle moved by set_estimate against a fresh
    create at that state, and a second pass after reset: bit-identical lists, S, b_schur, Hpp and 5-iteration state"""
    monkeypatch.setenv("CCM_PCG_NC", "0")   # read by ccm_ba_create: the coarse level's set-up sums with atomics
    p = scene(name)
    first = _everything(p)
    _same(first, _everything(p), f"{name} (two creates)")
    _same_as_grouped(_shuffled(p, 11), name)
    q = p.copy()
    q.poses[:, 4:] += 1e-3
    q.points = q.points + 1e-3
    h = api.BAHandle(p)
    try:
        h.debug_schur(1e-3)
        h.set_estimate(q.poses, q.points)
        moved = _collect(h)
        h.reset()
        again = _collect(h)
    finally:
        h.close()
    _same(moved, _everything(q), f"{name} (set_estimate against a fresh create)")
    _same(moved, again, f"{name} (after reset)")


def test_loop_closure_lm_matches_oracle(dev, oracle):
    p = scene("loop_closure")
    iters = 10
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

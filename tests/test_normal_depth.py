"""CPU suite: map-point normals and depth limits (MapPoint::UpdateNormalAndDepth, cslam/src/MapPoint.cpp:779-823).

 * the pin: tests/golden/normal_depth_cv2.npz, the body evaluated with cv2 4.13 (its generator checks an independent numpy restatement
   before it writes); the oracle, the library's host entry point ccm_normal_depth_host and the literal restatement on stand-in objects
   all reproduce it bit for bit, NaN as NaN;
 * the same three agree on fresh scenes and on each edge case of the reference body;
 * shim/MapPoint_shim.cpp: the parked path (ccm_b200_prepare_normals + the member) and the host path leave identical members, and a
   stale snapshot falls back to the host path;
 * ccm_normal_depth needs a device.
The device kernel is tests/test_gpu_normal_depth.py."""
import importlib.util
import os
import subprocess

import numpy as np
import pytest

from ccm_slam_b200 import api, synth
from oracle import pynd

HERE = os.path.dirname(os.path.abspath(__file__))
KEYS = ("normal", "max_dist", "min_dist", "status")


def _golden():
    spec = importlib.util.spec_from_file_location("make_normal_depth_golden", os.path.join(HERE, "golden", "make_normal_depth_golden.py"))
    mod = importlib.util.module_from_spec(spec); spec.loader.exec_module(mod)
    return mod


def same(a, b):
    for k in KEYS:
        assert np.array_equal(a[k], b[k], equal_nan=True), k


def test_everything_reproduces_the_opencv_fixture():
    mod = _golden()
    z = np.load(os.path.join(HERE, "golden", "normal_depth_cv2.npz"))
    for c, kw in enumerate(mod.CASES):
        sc = mod.scene(kw)
        w = {k: z["case%d_%s" % (c, k)] for k in KEYS}
        same(pynd.oracle(sc), w)
        same(api.normal_depth(sc, host=True), w)
        if kw.get("map_order"):
            s = pynd.StandIn(sc)
            same(s.literal(), w)
            s.close()
        assert w["status"].sum() > 300


EDGE = dict(K=10, P=300, bad_kf_frac=0.3, bad_mp_frac=0.1, all_bad_frac=0.1, on_centre_frac=0.1, off_ref_frac=0.3, map_order=True)


@pytest.mark.parametrize("kw", [dict(seed=51, map_order=True), dict(seed=52, **EDGE), dict(seed=53, K=200, P=3000, map_order=True)],
                         ids=["random", "edges", "wide"])
def test_oracle_host_and_literal_agree(kw):
    sc = synth.make_normal_depth(**kw)
    o = pynd.oracle(sc)
    same(api.normal_depth(sc, host=True), o)
    s = pynd.StandIn(sc)
    same(s.literal(), o)
    s.close()


def test_edge_cases_of_the_reference_body():
    sc = synth.make_normal_depth(seed=54, **EDGE)
    r = api.normal_depth(sc, host=True)
    deg = np.diff(sc["obs_ptr"])
    bad = sc["kf_bad"].astype(bool)
    live = np.array([(~bad[sc["obs_kf"][sc["obs_ptr"][i]:sc["obs_ptr"][i + 1]]]).sum() for i in range(len(deg))])
    # a bad point, or one without observations, is left untouched
    assert sc["mp_bad"].sum() > 10 and (r["status"][sc["mp_bad"]] == 0).all() and (r["status"] == (deg > 0)).all()
    # every observer bad: n = 0, the normal is 0 * inf = NaN, the distances are still written
    allbad = (deg > 0) & (live == 0)
    assert allbad.sum() > 5 and np.isnan(r["normal"][allbad]).all() and np.isfinite(r["max_dist"][allbad]).all()
    # a point on an observer's centre that is not bad: r = 0, NaN
    X = sc["mp_pos"]; C = sc["kf_centre"]
    on = np.array([d > 0 and any((X[i] == C[k]).all() and not bad[k] for k in sc["obs_kf"][sc["obs_ptr"][i]:sc["obs_ptr"][i + 1]])
                   for i, d in enumerate(deg)])
    assert on.sum() > 3 and np.isnan(r["normal"][on]).all()
    # a bad reference keyframe is still used; a reference that does not observe the point takes keypoint 0's octave (the generator's
    # scale_ref) -- both through the distances, which equal the numpy statement
    ref = sc["mp_ref"]; w = deg > 0
    assert (bad[ref[w]]).sum() > 5 and (~sc["ref_observes"][w]).sum() > 5
    pc = (X[w] - C[ref[w]]).astype(np.float64)
    dist = np.sqrt((pc[:, 0] ** 2 + pc[:, 1] ** 2) + pc[:, 2] ** 2).astype(np.float32)
    assert np.array_equal(r["max_dist"][w], (dist * sc["mp_scale_ref"][w]).astype(np.float32))
    # the well-defined normals are unit-length means
    ok = w & ~np.isnan(r["normal"]).any(1) & (live == 1)
    assert np.allclose(np.linalg.norm(r["normal"][ok], axis=1), 1.0, atol=1e-6)


def test_shim_parked_and_host_paths_leave_identical_members():
    """each path on a fresh scene (members empty before the call), the parked one first; every written point took its parked value"""
    sc = synth.make_normal_depth(seed=55, K=80, P=4000, bad_kf_frac=0.1, all_bad_frac=0.01, on_centre_frac=0.01, off_ref_frac=0.05, map_order=True)
    s = pynd.StandIn(sc)
    calls, c0 = s.device_calls(), s.stats()
    parked = s.shim(prepare=True)
    assert s.device_calls() == calls + 1
    assert tuple(s.stats() - c0) == (int(parked["status"].sum()), 0, 0)
    s.close()
    s = pynd.StandIn(sc)
    c0 = s.stats()
    host = s.shim(prepare=False)
    assert s.device_calls() == calls + 1
    assert tuple(s.stats() - c0) == (0, 0, int(host["status"].sum()))
    literal = s.literal()
    s.close()
    assert parked["status"].sum() > 3000
    same(parked, host)
    same(parked, literal)
    same(parked, pynd.oracle(sc))


@pytest.mark.parametrize("kind", [1, 2, 3], ids=["observation-added", "reference-changed", "position-changed"])
def test_shim_stale_snapshot_falls_back_to_the_host_path(kind):
    sc = synth.make_normal_depth(seed=56, K=40, P=1500, map_order=True)
    # one extra keyframe that observes nothing, far from the map
    sc["kf_centre"] = np.vstack([sc["kf_centre"], np.float32([[40.0, -30.0, 25.0]])]).astype(np.float32)
    sc["kf_bad"] = np.append(sc["kf_bad"], np.uint8(0)); sc["kf_oct0"] = np.append(sc["kf_oct0"], np.int32(5))
    extra = len(sc["kf_bad"]) - 1
    s = pynd.StandIn(sc)
    before = s.literal()
    c0 = s.stats()
    r = s.stale(kind, extra, shift=0.5)
    hits, stale, host = s.stats() - c0
    n_changed = int(before["status"][::2].sum())                    # points prepared and then changed: every one found stale
    assert stale == n_changed and hits == int(before["status"].sum()) - n_changed and host == stale
    after = s.literal()                         # the scene as the members found it
    same(r, after)
    changed = np.zeros(len(sc["mp_ref"]), bool); changed[::2] = True
    w = changed & (before["status"] == 1)
    field = "normal" if kind == 1 else "max_dist"                  # what the change moves: a parked value would keep the old one
    assert not np.array_equal(before[field][w], after[field][w])
    s.close()


def test_shim_type_check_target():
    subprocess.check_call(["make", "-C", os.path.join(HERE, "..", "oracle"), "-s", "shim-check-normal_depth"])


def test_library_entry_points():
    sc = synth.make_normal_depth(seed=57, K=5, P=20)
    assert hasattr(api.lib(), "ccm_normal_depth") and hasattr(api.lib(), "ccm_normal_depth_host")
    if api.device_count() == 0:
        with pytest.raises(api.CCMError) as e:
            api.normal_depth(sc)
        assert e.value.code == -2
    bad = dict(sc); bad["obs_kf"] = sc["obs_kf"].copy(); bad["obs_kf"][0] = 99
    with pytest.raises(api.CCMError):
        api.normal_depth(bad, host=True)


def test_scaleadd_is_one_fma_and_norm_sums_in_f64():
    """the two OpenCV facts the arithmetic rests on, checked against cv2 directly where it imports"""
    cv2 = pytest.importorskip("cv2")
    from fractions import Fraction
    rng = np.random.default_rng(9)
    for _ in range(500):
        d = (rng.normal(0, 1, (3, 1)) * 10.0 ** rng.integers(-2, 3)).astype(np.float32)
        nv = rng.normal(0, 1, (3, 1)).astype(np.float32)
        r = cv2.norm(d)
        s = 0.0
        for v in d.ravel():
            s += float(v) * float(v)
        assert r == np.sqrt(s)
        a = np.float32(1.0 / r)
        want = np.array([np.float32(float(Fraction(float(d[i, 0])) * Fraction(float(a)) + Fraction(float(nv[i, 0])))) for i in range(3)],
                        np.float32).reshape(3, 1)
        assert np.array_equal(cv2.scaleAdd(d, 1.0 / r, nv), want)

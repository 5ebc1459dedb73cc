"""ccm_fuse_neighbours_host — the searches of LocalMapping::SearchInNeighbors in one call — against the flat oracle (oracle/pyfn.py):
Fuse's prelude with the host's logf and the reference-pinned window search, pair by pair.  No device needed."""
import copy
import os

import numpy as np
import pytest

from ccm_slam_b200 import api
from ccm_slam_b200 import synth_match as sm
from oracle import pyfn

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "fuse_neighbours.npz")


def _check(sc):
    fwd, bwd, settled = api.fuse_neighbours(sc, host=True)
    rf, rb = pyfn.oracle(sc)
    assert np.array_equal(fwd, rf) and np.array_equal(bwd, rb)
    return fwd, bwd, settled


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_host_equals_oracle(seed):
    sc = sm.make_fuse_scene(n_first=6, n_second=3, n=500, seed=seed)
    fwd, bwd, settled = _check(sc)
    assert (fwd >= 0).sum() > 200 and (bwd >= 0).sum() > 200
    assert settled > 0                                   # PredictScale boundary pairs were reached and settled with logf
    assert len(sc["entries"]) > len(sc["targets"])       # a second neighbour listed more than once, uploaded once


def test_predict_scale_boundary_pairs_change_results():
    """the boundary points decide matches: moving only their mfMaxDistance by one ulp moves the result of at least one of their own
    pairs, and the host entry still equals the oracle (std::log(float)) on both"""
    sc = sm.make_fuse_scene(n_first=4, n_second=2, n=400, seed=7, boundary=200)
    fwd, bwd, settled = _check(sc)
    assert settled >= 10
    rows = sc["boundary_rows"]
    sc2 = copy.deepcopy(sc)
    mx = sc2["points"]["max_d"]
    mx[rows] = np.nextafter(mx[rows], np.float32(np.inf), dtype=np.float32)
    f2, b2, _ = _check(sc2)
    at_fwd = np.isin(sc["cur_point"], rows)
    at_bwd = np.isin(sc["cand"], rows)
    assert not np.array_equal(fwd[:, at_fwd], f2[:, at_fwd]) or not np.array_equal(bwd[at_bwd], b2[at_bwd])
    assert np.array_equal(fwd[:, ~at_fwd], f2[:, ~at_fwd]) and np.array_equal(bwd[~at_bwd], b2[~at_bwd])


def test_golden_fixture():
    z = np.load(GOLDEN)
    sc = sm.fuse_scene_from_arrays(z)
    fwd, bwd, _ = _check(sc)
    assert np.array_equal(fwd, z["fwd"]) and np.array_equal(bwd, z["bwd"])


def test_one_target_and_empty():
    sc = sm.make_fuse_scene(n_first=1, n_second=0, n=300, seed=3)
    assert len(sc["targets"]) == 1
    fwd, bwd, _ = _check(sc)
    assert fwd.shape == (1, 300) and (fwd >= 0).any()
    e = copy.deepcopy(sc)
    e["targets"] = []; e["cand"] = np.zeros(0, np.int32)
    fwd, bwd, settled = _check(e)
    assert fwd.shape == (0, 300) and bwd.shape == (0,) and settled == 0
    e["cur_point"] = np.full(300, -1, np.int32)
    e["targets"] = sc["targets"]
    fwd, bwd, _ = _check(e)
    assert (fwd == -1).all()


def test_skip_flag_and_empty_slots():
    sc = sm.make_fuse_scene(n_first=3, n_second=1, n=300, seed=4)
    fwd, bwd, _ = _check(sc)
    skip = sc["points"]["skip"].astype(bool)
    cp = sc["cur_point"]
    assert skip.any()
    assert (fwd[:, (cp < 0)] == -1).all() and (fwd[:, (cp >= 0) & skip[np.maximum(cp, 0)]] == -1).all()
    assert (bwd[skip[sc["cand"]]] == -1).all()


def _err(sc):
    with pytest.raises(api.CCMError) as e:
        api.fuse_neighbours(sc, host=True)
    return str(e.value)


def test_validation_messages():
    sc = sm.make_fuse_scene(n_first=2, n_second=1, n=200, seed=5, boundary=0)
    P = len(sc["points"]["skip"])
    a = copy.deepcopy(sc); a["cur_point"][17] = P
    assert "slot 17 of the current keyframe: point row %d out of range" % P in _err(a)
    a = copy.deepcopy(sc); a["cur_point"][3] = -2
    assert "slot 3 of the current keyframe: point row -2 out of range" in _err(a)
    a = copy.deepcopy(sc); a["cand"][5] = -1
    assert "candidate 5: point row -1 out of range" in _err(a)
    a = copy.deepcopy(sc); a["targets"][1]["cols"] = 20000; a["targets"][1]["rows"] = 1
    assert "target 1: too many keypoints for the 20-bit visiting position" in _err(a)
    a = copy.deepcopy(sc); a["cur"]["cols"] = 0
    assert "current keyframe: bad grid" in _err(a)


def test_null_arrays():
    import ctypes as C
    sc = sm.make_fuse_scene(n_first=2, n_second=1, n=200, seed=6, boundary=0)
    keep = []
    cur, tg, T, pts, cp, cand = api.fuse_structs(sc, keep)
    L = api.lib()
    out = np.zeros(T * len(cp) + len(cand) + 1, np.int32)
    assert L.ccm_fuse_neighbours_host(C.byref(cur), tg, T, C.byref(pts), None, api._p(cand), len(cand), api._p(out), api._p(out), None) == -1
    assert "null cur_point" in L.ccm_last_error().decode()
    assert L.ccm_fuse_neighbours_host(C.byref(cur), tg, T, C.byref(pts), api._p(cp), api._p(cand), len(cand), None, api._p(out), None) == -1
    assert "null output array" in L.ccm_last_error().decode()
    pts.desc = None
    assert L.ccm_fuse_neighbours_host(C.byref(cur), tg, T, C.byref(pts), api._p(cp), api._p(cand), len(cand), api._p(out), api._p(out), None) == -1
    assert "null point array" in L.ccm_last_error().decode()

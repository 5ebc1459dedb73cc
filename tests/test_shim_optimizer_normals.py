"""The five write-back loops of shim/Optimizer_shim.cpp with shim/MapPoint_shim.cpp linked next to them (oracle/Makefile:
_ref/liboptimizer_nd_shim.so, device entry points doubled on the CPU; the GPU build is driven from tests/test_gpu_normal_depth.py).

For MapFusionGBA (direct and through a registered mirror), GlobalBundleAdjustemntClient, LocalBundleAdjustmentClient and both
OptimizeEssentialGraph variants: every point the loop wrote holds the members a per-point host computation gives on the state the
loop left, bit for bit; the loop wrote exactly the points it moved; and every one of those took its parked value (one hit each, no
stale entry, no host computation inside the loop)."""
import ctypes as C
import os

import numpy as np
import pytest

from ccm_slam_b200 import synth
from tests import shim_optimizer_harness as H
from tests.test_shim_optimizer import essential_scene

HERE = os.path.dirname(os.path.abspath(__file__))


def nd_lib(gpu):
    so = os.path.join(HERE, "..", "oracle", "_ref", "liboptimizer_nd_shim_gpu.so" if gpu else "liboptimizer_nd_shim.so")
    if not os.path.exists(so):
        from oracle import pyoracle
        if pyoracle.build_ref() is None:
            return None
    return C.CDLL(so) if os.path.exists(so) else None


def stats(L):
    c = (C.c_ulonglong * 3)()
    L.ndw_stats(c)
    return np.array(c[:], np.int64)


def run(L, sc, fn, *args, **kw):
    """fn: a shim_optimizer_harness runner; returns (harness output, loop members, host members, member-outcome counter deltas)"""
    P = len(sc["mp_uid"])
    loop = dict(normal=np.zeros((P, 3), np.float32), max_dist=np.zeros(P, np.float32), min_dist=np.zeros(P, np.float32), written=np.zeros(P, np.uint8))
    host = {k: v.copy() for k, v in loop.items()}
    p = lambda a: a.ctypes.data_as(C.c_void_p)
    before = stats(L)
    L.ndw_arm(C.c_int64(int(sc["mp_uid"][0])), P, p(loop["normal"]), p(loop["max_dist"]), p(loop["min_dist"]), p(loop["written"]),
              p(host["normal"]), p(host["max_dist"]), p(host["min_dist"]), p(host["written"]))
    saved = H._LIB
    H._LIB = L
    try:
        out = fn(sc, *args, **kw)
    finally:
        H._LIB = saved
        c = (C.c_ulonglong * 3)()
        L.ndw_disarm(c)
    return out, loop, host, np.array(c[:], np.int64) - before


def check(sc, out, loop, host, delta):
    moved = (out["mp_set_pos"] > 0) & (sc["mp_bad"] == 0) & (out["mp_n_obs"] > 0)
    w = loop["written"].astype(bool)
    assert moved.sum() >= 20
    assert np.array_equal(w, moved)                                 # exactly the points the loop moved
    assert host["written"][w].all()
    for k in ("normal", "max_dist", "min_dist"):
        assert np.array_equal(loop[k][w], host[k][w], equal_nan=True), k
    hits, stale, on_host = delta
    assert (hits, stale, on_host) == (int(w.sum()), 0, 0), (hits, stale, on_host, int(w.sum()))


def gba_scene(ho, name="small", bad=0.05):
    return H.scene_from_problem(synth.make_config(name), ho, seed=3, map_id=0, bad_kf=bad, bad_mp=bad)


def local_scene(ho):
    p = synth.make_config("small")
    sc = H.scene_from_problem(p, ho, seed=5, map_id=0)
    K = p.K
    rng = np.random.default_rng(6)
    center = 3
    covis = [k for k in rng.permutation(K) if k != center][:10]
    cov_ptr = np.zeros(K + 1, np.int32); cov_ptr[center + 1:] = len(covis)
    sc.update(cov_ptr=cov_ptr, cov_kf=np.array(covis, np.int32), cov_w=np.full(len(covis), 200, np.int32))
    sc["mp_bad"] = (rng.random(p.P) < 0.05).astype(np.uint8)
    return sc, center


def with_observations(sc, seed=7):
    """essential_scene's points hang off reference keyframes without observations; give each one its reference keyframe and that
    keyframe's neighbours in the chain as observers (one keypoint each, random octave), so that the member has something to compute"""
    rng = np.random.default_rng(seed)
    K, P = len(sc["kf_uid"]), len(sc["mp_uid"])
    obs = [sorted({int(r) + d for d in (-1, 0, 1) if 0 <= int(r) + d < K}) for r in sc["mp_ref"]]
    count = np.zeros(K, np.int64); okf, oidx = [], []
    for lst in obs:
        for k in lst:
            okf.append(k); oidx.append(count[k]); count[k] += 1
    kp_ptr = np.concatenate([[0], np.cumsum(count)]).astype(np.int32)
    sc = dict(sc)
    sc.update(kp_ptr=kp_ptr, kp_uv=rng.uniform(0, 400, (kp_ptr[-1], 2)).astype(np.float32), kp_octave=rng.integers(0, 8, kp_ptr[-1]).astype(np.int32),
              obs_ptr=np.concatenate([[0], np.cumsum([len(o) for o in obs])]).astype(np.int32), obs_kf=np.array(okf, np.int32),
              obs_idx=np.array(oidx, np.int32))
    assert len(sc["mp_uid"]) == P
    return sc


def write_backs(ho):
    """(id, scene, runner, args, kwargs) for the five loops"""
    ls, center = local_scene(ho)
    K = 40
    es = with_observations(essential_scene(ho, K=K, seed=1, bad=(7, 22))[0])
    conn = {K - 1: [2, 4], 2: [K - 1], 4: [K - 1], K - 2: [3]}
    near = [K - 1, K - 2, K - 3]
    eye = np.array([0.0, 0.0, 0.0, 1.0, 0.0, 0.0, 0.0, 1.0])
    corr = (near, np.stack([eye] * 3), np.stack([eye] * 3))
    return [("map_fusion_gba", gba_scene(ho), H.run_gba, (0, 6, True, (0, 0)), {}),
            ("map_fusion_gba_mirror", gba_scene(ho), H.run_gba_mirror, (6, True, (0, 0)), {}),
            ("global_ba_client", gba_scene(ho, "tiny", 0.0), H.run_gba, (1, 5, True, (0, 0)), {}),
            ("local_ba_client", ls, H.run_local_ba, (center,), {}),
            ("essential_graph_map_fusion", es, H.run_essential_graph, (2, K - 1, conn, False), {}),
            ("essential_graph_loop_closure", es, H.run_essential_graph, (2, K - 1, conn, False), dict(loop_closure=True, corr=corr))]


IDS = ["map_fusion_gba", "map_fusion_gba_mirror", "global_ba_client", "local_ba_client", "essential_graph_map_fusion",
       "essential_graph_loop_closure"]


@pytest.mark.parametrize("which", IDS)
def test_write_back_takes_every_parked_value(oracle, which):
    L = nd_lib(gpu=False)
    if L is None:
        pytest.skip("oracle/_ref/liboptimizer_nd_shim.so not available (needs the reference tree and the product library)")
    _, sc, fn, args, kw = write_backs(oracle)[IDS.index(which)]
    check(sc, *run(L, sc, fn, *args, **kw))

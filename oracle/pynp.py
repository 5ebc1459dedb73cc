"""ctypes binding of the new-map-point checker (oracle/new_points.mk).  TEST INFRASTRUCTURE, NOT PRODUCT.

  oracle(cur, neighbours, mutate=0)   oracle/libnew_points_oracle.so: the sequential loop of LocalMapping::CreateNewMapPoints over the
                                      view dicts api.new_map_points reads -> (points, best2, verdict), shaped as api.new_map_points'
  svd4_null(A)                        the stated 4x4 decomposition alone: A (4,4) f32 -> vt.row(3)
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = None


def build() -> None:
    subprocess.check_call(["make", "-C", _HERE, "-s", "-f", "new_points.mk", "ref"])


def lib():
    global _LIB
    if _LIB is None:
        so = os.path.join(_HERE, "libnew_points_oracle.so")
        if not os.path.exists(so):
            build()
        _LIB = C.CDLL(so)
    return _LIB


def oracle(cur, neighbours, mutate=0, capacity=None):
    """mutate=1 (tests only): a pair that fails a gate still claims its feature"""
    from ccm_slam_b200 import api
    keep = []
    c, nbs = api.new_points_structs(cur, neighbours, keep)
    n, B = len(cur["octave"]), len(neighbours)
    cap = n * B if capacity is None else int(capacity)
    out = np.zeros(max(cap, 1), api.NEW_POINT_DTYPE)
    best2 = np.full((B, n), -2, np.int32); verdict = np.full((B, n), 255, np.uint8)
    n_out = C.c_int32(-1)
    rc = lib().orc_new_map_points(C.byref(c), nbs, B, out.ctypes.data_as(C.c_void_p), cap, C.byref(n_out), best2.ctypes.data_as(C.c_void_p),
                                  verdict.ctypes.data_as(C.c_void_p), int(mutate))
    if rc != 0:
        raise ValueError("orc_new_map_points: capacity %d below the %d points needed" % (cap, n_out.value))
    return out[:n_out.value].copy(), best2, verdict


def svd4_null(A):
    A = np.ascontiguousarray(A, np.float32).reshape(16)
    x = np.zeros(4, np.float32)
    lib().orc_svd4_null(A.ctypes.data_as(C.c_void_p), x.ctypes.data_as(C.c_void_p))
    return x


class StandIn:
    """A current keyframe and its neighbours as stand-in KeyFrame / MapPoint / LocalMapping objects (oracle/ref_stub_np), built from the
    view dicts api.new_map_points reads; median_depth[k] is what ComputeSceneMedianDepth answers for keyframe k (0 = the current one).
    run(mode, force_at_poll): mode 0 the literal restatement of LocalMapping::CreateNewMapPoints, 1 shim/NewMapPoints_shim.cpp; over the
    CPU double of the device entry point, or the real library with gpu=True."""

    def __init__(self, cur, neighbours, median_depth=None, gpu=False):
        from ccm_slam_b200 import api
        so = os.path.join(_HERE, "_ref", "libnew_points_shim_gpu.so" if gpu else "libnew_points_shim.so")
        if not os.path.exists(so):
            build()
        self.L = C.CDLL(so)
        self.L.np_scene_create.restype = C.c_void_p
        for f in ("np_scene_destroy", "np_point_count", "np_polls"):
            getattr(self.L, f).argtypes = [C.c_void_p]
        self.L.np_run.argtypes = [C.c_void_p, C.c_int, C.c_int]
        self.keep = []
        c, nbs = api.new_points_structs(cur, neighbours, self.keep)
        self.sizes = [len(cur["octave"])] + [len(v["octave"]) for v in neighbours]
        K = len(self.sizes)
        ptrs = (C.c_void_p * K)(C.addressof(c), *[C.addressof(nbs[i].view) for i in range(K - 1)])
        self.keep += [c, nbs]
        md = np.ones(K, np.float32) if median_depth is None else np.ascontiguousarray(median_depth, np.float32)
        self.h = C.c_void_p(self.L.np_scene_create(K, ptrs, md.ctypes.data_as(C.c_void_p)))

    def close(self):
        if self.h:
            self.L.np_scene_destroy(self.h); self.h = None

    def run(self, mode, force_at_poll=-1):
        if self.L.np_run(self.h, int(mode), int(force_at_poll)) != 0:
            raise RuntimeError("the member threw")

    def members(self):
        """what the member changed: mvpMapPoints of every keyframe, the new points and the recent-points list"""
        P = self.L.np_point_count(self.h)
        o = dict(mvp=np.zeros(sum(self.sizes), np.int32), pos=np.zeros((max(P, 1), 3), np.float32), ref=np.zeros(max(P, 1), np.int32),
                 obs=np.zeros((max(P, 1), 4), np.int32), log=np.zeros((max(P, 1), 8), np.uint8), recent=np.zeros(max(P, 1), np.int32))
        nr = C.c_int32()
        p = lambda a: a.ctypes.data_as(C.c_void_p)  # noqa: E731
        assert self.L.np_members(self.h, p(o["mvp"]), p(o["pos"]), p(o["ref"]), p(o["obs"]), p(o["log"]), p(o["recent"]), C.byref(nr)) == P
        for k in ("pos", "ref", "obs", "log"):
            o[k] = o[k][:P]
        o["recent"] = o["recent"][:nr.value]
        o["polls"] = self.L.np_polls(self.h)
        return o

    def device_calls(self):
        return self.L.np_double_device_calls()

    def stats(self):
        """(library calls made by the shim member, points created, points dropped by an early return) since the process started"""
        c = (C.c_ulonglong * 3)()
        self.L.np_shim_stats(c)
        return np.array(c[:], np.int64)

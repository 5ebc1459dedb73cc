"""ctypes binding of the map-point descriptor checker (oracle/distinctive.mk).  TEST INFRASTRUCTURE, NOT PRODUCT.

  oracle(sc)             oracle/libdistinctive_oracle.so: our restatement of MapPoint::ComputeDistinctiveDescriptors over the flat arrays
  StandIn(sc, gpu=False) a scene of stand-in MapPoint / KeyFrame objects (oracle/ref_stub_dd) with .literal() (the reference body restated
                         on them), .shim(prepare) (shim/MapPointDescriptor_shim.cpp's member, with or without the batched preparation),
                         .stale(kind, kf), .search_in_neighbors(pts) and .establish(kf, mp_of_idx, split); over the CPU doubles of the
                         device entry points, or the real library with gpu=True
The oracle and .literal() return dict(best, best_median, desc); the shim calls return dict(desc, written).
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIBS = {}


def build() -> None:
    subprocess.check_call(["make", "-C", _HERE, "-s", "-f", "distinctive.mk", "ref"])


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def _lib(name):
    if name not in _LIBS:
        so = os.path.join(_HERE, name)
        if not os.path.exists(so):
            build()
        _LIBS[name] = C.CDLL(so)
    return _LIBS[name]


def _choice(P):
    return dict(best=np.zeros(P, np.int32), best_median=np.zeros(P, np.int32), desc=np.zeros((P, 32), np.uint8))


def oracle(sc):
    K = len(sc["kf_bad"]); P = len(sc["obs_ptr"]) - 1; o = _choice(P)
    a = [np.ascontiguousarray(sc[k], t) for k, t in (("kf_bad", np.uint8), ("obs_ptr", np.int64), ("obs_kf", np.int32), ("obs_desc", np.uint8))]
    rc = _lib("libdistinctive_oracle.so").orc_distinctive_descriptors(K, _p(a[0]), P, _p(a[1]), _p(a[2]), _p(a[3]), _p(o["best"]),
                                                                      _p(o["best_median"]), _p(o["desc"]))
    if rc != 0:
        raise ValueError("orc_distinctive_descriptors: bad input")
    return o


class StandIn:
    def __init__(self, sc, gpu=False):
        self.L = _lib(os.path.join("_ref", "libdistinctive_shim_gpu.so" if gpu else "libdistinctive_shim.so"))
        self.gpu = gpu
        self.L.dd_scene_create.restype = C.c_void_p
        self.L.dd_scene_destroy.argtypes = [C.c_void_p]
        self.L.dd_add_keyframe.argtypes = [C.c_void_p, C.c_uint64, C.c_uint8, C.c_int32, C.c_void_p]
        self.L.dd_add_keyframe.restype = C.c_int32
        self.L.dd_register_store.argtypes = [C.c_void_p]
        self._keep = [np.ascontiguousarray(sc[k], t) for k, t in (
            ("kf_bad", np.uint8), ("kf_uid", np.uint64), ("kf_desc_ptr", np.int64), ("kf_desc", np.uint8), ("mp_bad", np.uint8),
            ("obs_ptr", np.int64), ("obs_kf", np.int32), ("obs_feat", np.int32))]
        k = self._keep
        self.P = len(sc["obs_ptr"]) - 1
        self.h = C.c_void_p(self.L.dd_scene_create(len(sc["kf_bad"]), _p(k[0]), _p(k[1]), _p(k[2]), _p(k[3]), self.P, _p(k[4]), _p(k[5]),
                                                   _p(k[6]), _p(k[7])))

    def close(self):
        if self.h:
            self.L.dd_scene_destroy(self.h); self.h = None

    def _members(self, fn, *args):
        o = dict(desc=np.zeros((self.P, 32), np.uint8), written=np.zeros(self.P, np.uint8))
        if fn(self.h, *args, _p(o["desc"]), _p(o["written"])) != 0:
            raise RuntimeError("the shim threw")
        return o

    def literal(self):
        o = _choice(self.P)
        self.L.dd_literal(self.h, _p(o["best"]), _p(o["best_median"]), _p(o["desc"]))
        return o

    def add_keyframe(self, uid, desc, bad=False):
        desc = np.ascontiguousarray(desc, np.uint8)
        self._keep.append(desc)
        k = self.L.dd_add_keyframe(self.h, int(uid), int(bad), len(desc), _p(desc))
        assert k >= 0
        return k

    def shim(self, prepare):
        """prepare: 0 the member alone, 1 ccm_b200_prepare_descriptors first, 2 ccm_b200_prepare_point_updates first (and both members)"""
        return self._members(self.L.dd_shim, int(prepare))

    def stale(self, kind, kf):
        return self._members(self.L.dd_shim_stale, int(kind), int(kf))

    def search_in_neighbors(self, pts):
        pts = np.ascontiguousarray(pts, np.int32)
        return self._members(self.L.dd_search_in_neighbors, len(pts), _p(pts))

    def establish(self, kf, mp_of_idx, split):
        m = np.ascontiguousarray(mp_of_idx, np.int32)
        return self._members(self.L.dd_establish, int(kf), len(m), _p(m), int(split))

    def register_store(self, handle):
        """a ccm_kf_store* for the shim's preparation (None: rows go with the call).  Over the CPU double any non-null value names the
        double's own store (store_put)."""
        self.L.dd_register_store(handle)

    def store_put(self, uid, desc):
        desc = np.ascontiguousarray(desc, np.uint8)
        self.L.dd_double_store_put(C.c_uint64(uid), len(desc), _p(desc))

    def device_calls(self):
        return self.L.dd_double_device_calls(), self.L.dd_double_store_calls()

    def stats(self):
        """the member's outcome counters so far: (parked choices written, stale entries, host computations)"""
        c = (C.c_ulonglong * 3)()
        self.L.dd_stats(c)
        return np.array(c[:], np.int64)

    def normal_stats(self):
        c = (C.c_ulonglong * 3)()
        self.L.dd_nd_stats(c)
        return np.array(c[:], np.int64)

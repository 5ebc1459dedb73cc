"""ctypes binding of the map-point normal checker (oracle/Makefile).  TEST INFRASTRUCTURE, NOT PRODUCT.

  oracle(sc)             oracle/liboracle.so (normal_depth_oracle.cpp): our restatement of MapPoint::UpdateNormalAndDepth over the flat arrays
  StandIn(sc, gpu=False) a scene of stand-in MapPoint / KeyFrame objects (oracle/ref_stub_mp) with .literal() (the reference body restated
                         on them), .shim(prepare) (shim/MapPoint_shim.cpp's member, with or without the batched preparation) and
                         .stale(kind, kf, shift); over the CPU double of ccm_normal_depth, or the real library with gpu=True
Every call returns dict(normal, max_dist, min_dist, status).
"""
from __future__ import annotations

import ctypes as C

import numpy as np

from oracle import pyoracle


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def _out(P):
    return dict(normal=np.zeros((P, 3), np.float32), max_dist=np.zeros(P, np.float32), min_dist=np.zeros(P, np.float32),
                status=np.zeros(P, np.uint8))


def _args(o):
    return _p(o["normal"]), _p(o["max_dist"]), _p(o["min_dist"]), _p(o["status"])


def oracle(sc):
    K = len(sc["kf_bad"]); P = len(sc["mp_ref"]); o = _out(P)
    a = [np.ascontiguousarray(sc[k], t) for k, t in (("kf_centre", np.float32), ("kf_bad", np.uint8), ("mp_pos", np.float32), ("obs_ptr", np.int64),
                                                     ("obs_kf", np.int32), ("mp_ref", np.int32), ("mp_scale_ref", np.float32), ("mp_scale_last", np.float32))]
    rc = pyoracle.lib().orc_normal_depth(K, _p(a[0]), _p(a[1]), P, _p(a[2]), _p(a[3]), _p(a[4]), _p(a[5]), _p(a[6]), _p(a[7]), *_args(o))
    if rc != 0:
        raise ValueError("orc_normal_depth: bad input")
    return o


class StandIn:
    def __init__(self, sc, gpu=False):
        self.L = pyoracle.ref_lib("libnormal_depth_shim_gpu.so" if gpu else "libnormal_depth_shim.so")
        self.L.nd_scene_create.restype = C.c_void_p
        self.L.nd_scene_destroy.argtypes = [C.c_void_p]
        self.L.nd_shim_stale.argtypes = [C.c_void_p, C.c_int, C.c_int32, C.c_float] + [C.c_void_p] * 4
        self._keep = [np.ascontiguousarray(sc[k], t) for k, t in (
            ("kf_centre", np.float32), ("kf_bad", np.uint8), ("kf_oct0", np.int32), ("mp_pos", np.float32), ("mp_bad", np.uint8),
            ("obs_ptr", np.int64), ("obs_kf", np.int32), ("obs_octave", np.int32), ("mp_ref", np.int32))]
        k = self._keep
        self.P = len(sc["mp_ref"])
        self.h = C.c_void_p(self.L.nd_scene_create(len(sc["kf_bad"]), _p(k[0]), _p(k[1]), _p(k[2]), self.P, _p(k[3]), _p(k[4]), _p(k[5]),
                                                   _p(k[6]), _p(k[7]), _p(k[8])))

    def close(self):
        if self.h:
            self.L.nd_scene_destroy(self.h); self.h = None

    def literal(self):
        o = _out(self.P); self.L.nd_literal(self.h, *_args(o)); return o

    def shim(self, prepare):
        o = _out(self.P)
        if self.L.nd_shim(self.h, int(prepare), *_args(o)) != 0:
            raise RuntimeError("nd_shim threw")
        return o

    def stale(self, kind, kf, shift=0.0):
        o = _out(self.P)
        if self.L.nd_shim_stale(self.h, int(kind), int(kf), float(shift), *_args(o)) != 0:
            raise RuntimeError("nd_shim_stale threw")
        return o

    def device_calls(self):
        return self.L.nd_double_device_calls()

    def stats(self):
        """the member's outcome counters so far: (parked values written, stale entries, host computations)"""
        c = (C.c_ulonglong * 3)()
        self.L.nd_stats(c)
        return np.array(c[:], np.int64)

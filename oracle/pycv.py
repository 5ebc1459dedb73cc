"""ctypes binding of the covisibility checker (oracle/Makefile).  TEST INFRASTRUCTURE, NOT PRODUCT.

  oracle(sc, th)          oracle/liboracle.so (covis_oracle.cpp): our restatement of UpdateConnections' counter and orders over the flat arrays
  StandIn(sc, gpu=False)  a scene of stand-in KeyFrame / MapPoint objects (oracle/ref_stub_cv), keyframe row k at address rank
                          sc["kf_rank"][k], with .literal_flat() (the reference body's counter and ordered list per batch keyframe),
                          .merge(mode), .merge_stale(kind, row), .load_map(split) and .members(); over the CPU double of the device
                          entry point, or the real library with gpu=True
The flat results are dicts shaped as api.covisibility's.
"""
from __future__ import annotations

import ctypes as C

import numpy as np

from oracle import pyoracle


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def _flat(B, cap):
    return dict(conn_ptr=np.zeros(B + 1, np.int64), conn_kf=np.zeros(max(cap, 1), np.int32), conn_w=np.zeros(max(cap, 1), np.int32),
                n_sel=np.zeros(B, np.int32), sel_kf=np.zeros(max(cap, 1), np.int32), sel_w=np.zeros(max(cap, 1), np.int32),
                status=np.zeros(B, np.uint8))


def _trim(o):
    T = int(o["conn_ptr"][-1])
    for k in ("conn_kf", "conn_w", "sel_kf", "sel_w"):
        o[k] = o[k][:T]
    return o


def oracle(sc, th=15, batch=None):
    from ccm_slam_b200.api import covisibility_batch
    b, mptr, mp = covisibility_batch(sc, batch)
    a = [np.ascontiguousarray(sc[k], t) for k, t in (("kf_id", np.uint64), ("kf_rank", np.uint32), ("mp_bad", np.uint8),
                                                     ("obs_ptr", np.int64), ("obs_kf", np.int32))]
    total = np.zeros(1, np.int64)
    L = pyoracle.lib()
    L.orc_covisibility(len(a[0]), _p(a[0]), _p(a[1]), len(b), _p(b), _p(mptr), _p(mp), len(a[2]), _p(a[2]), _p(a[3]), _p(a[4]), int(th),
                       C.c_int64(0), None, None, None, None, None, None, None, _p(total))
    o = _flat(len(b), int(total[0]))
    rc = L.orc_covisibility(len(a[0]), _p(a[0]), _p(a[1]), len(b), _p(b), _p(mptr), _p(mp), len(a[2]), _p(a[2]), _p(a[3]), _p(a[4]),
                            int(th), C.c_int64(int(total[0])), *[_p(o[k]) for k in ("conn_ptr", "conn_kf", "conn_w", "n_sel", "sel_kf",
                                                                                    "sel_w", "status")], _p(total))
    if rc != 0:
        raise ValueError("orc_covisibility: bad input")
    return _trim(o)


class StandIn:
    def __init__(self, sc, gpu=False, first_connection=None, fill_mvp=True):
        """first_connection: (K,) u8 mbFirstConnection of each row (None: all true); fill_mvp=False leaves mvpMapPoints empty (for
        load_map)"""
        self.L = pyoracle.ref_lib("libcovis_shim_gpu.so" if gpu else "libcovis_shim.so")
        self.L.cv_scene_create.restype = C.c_void_p
        self.L.cv_scene_destroy.argtypes = [C.c_void_p]
        for f in ("cv_merge", "cv_load_map"):
            getattr(self.L, f).argtypes = [C.c_void_p, C.c_int]
        self.L.cv_merge_stale.argtypes = [C.c_void_p, C.c_int, C.c_int32, C.c_int]
        K = len(sc["kf_id"])
        self.K, self.B = K, len(sc["batch"])
        fc = np.ones(K, np.uint8) if first_connection is None else first_connection
        self._keep = [np.ascontiguousarray(x, t) for x, t in (
            (sc["kf_id"], np.uint64), (sc["kf_rank"], np.uint32), (sc["kf_bad"], np.uint8), (fc, np.uint8), (sc["mvp_ptr"], np.int64),
            (sc["mvp"], np.int32), (sc["mp_bad"], np.uint8), (sc["obs_ptr"], np.int64), (sc["obs_kf"], np.int32), (sc["obs_idx"], np.int32),
            (sc["batch"], np.int32))]
        k = self._keep
        self.h = C.c_void_p(self.L.cv_scene_create(K, _p(k[0]), _p(k[1]), _p(k[2]), _p(k[3]), _p(k[4]), _p(k[5]), len(sc["mp_bad"]),
                                                   _p(k[6]), _p(k[7]), _p(k[8]), _p(k[9]), self.B, _p(k[10]), int(fill_mvp)))

    def close(self):
        if self.h:
            self.L.cv_scene_destroy(self.h); self.h = None

    def literal_flat(self, cap=None):
        cap = cap if cap is not None else self.B * self.K + 1
        o = _flat(self.B, cap)
        assert self.L.cv_literal_flat(self.h, C.c_int64(cap), *[_p(o[k]) for k in ("conn_ptr", "conn_kf", "conn_w", "n_sel", "sel_kf",
                                                                                    "sel_w", "status")]) == 0
        return _trim(o)

    def merge(self, mode):
        """mode 0: the literal body per keyframe; 1: the shim member alone; 2: one prepare, then the shim member"""
        if self.L.cv_merge(self.h, int(mode)) != 0:
            raise RuntimeError("the loop threw")

    def merge_stale(self, kind, row, literal=False):
        """kind 1 a map point index changed, 2 an observation added, 3 a point set bad, 4 an observer replaced at equal count, on
        every third batch keyframe after the preparation; then the shim loop (literal=True: the same changes, then the literal body)"""
        if self.L.cv_merge_stale(self.h, int(kind), int(row), int(literal)) != 0:
            raise RuntimeError("the loop threw")

    def load_map(self, split):
        if self.L.cv_load_map(self.h, int(split)) != 0:
            raise RuntimeError("the loop threw")

    def members(self):
        """every row's mConnectedKeyFrameWeights, ordered list and weights, children (rows, in container order), parent row and
        mbFirstConnection, as numpy arrays"""
        cap = self.K * self.K + 1
        o = dict(w_ptr=np.zeros(self.K + 1, np.int64), w_kf=np.zeros(cap, np.int32), w_w=np.zeros(cap, np.int32),
                 o_ptr=np.zeros(self.K + 1, np.int64), o_kf=np.zeros(cap, np.int32), o_w=np.zeros(cap, np.int32),
                 c_ptr=np.zeros(self.K + 1, np.int64), c_kf=np.zeros(cap, np.int32), parent=np.zeros(self.K, np.int32),
                 first=np.zeros(self.K, np.uint8))
        assert self.L.cv_members(self.h, C.c_int64(cap), *[_p(o[k]) for k in ("w_ptr", "w_kf", "w_w", "o_ptr", "o_kf", "o_w", "c_ptr",
                                                                               "c_kf", "parent", "first")]) == 0
        for p, ks in (("w_ptr", ("w_kf", "w_w")), ("o_ptr", ("o_kf", "o_w")), ("c_ptr", ("c_kf",))):
            for k in ks:
                o[k] = o[k][:int(o[p][-1])]
        return o

    def stats(self):
        """the member's outcome counters so far: (parked counters used, stale entries, host counts)"""
        c = (C.c_ulonglong * 3)()
        self.L.cv_stats(c)
        return np.array(c[:], np.int64)

    def device_calls(self):
        return self.L.cv_double_device_calls()

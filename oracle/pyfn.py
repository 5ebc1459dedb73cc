"""ctypes binding of the neighbour-fusion checker (oracle/fuse_neighbours.mk).  TEST INFRASTRUCTURE, NOT PRODUCT.

  oracle(sc)   oracle/libfuse_neighbours_oracle.so: every pair LocalMapping::SearchInNeighbors searches, Fuse's prelude with the host's
               logf and the reference-pinned window search, over a scene as synth_match.make_fuse_scene builds it -> (fwd, bwd), shaped
               as api.fuse_neighbours' first two results
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = None


def build() -> None:
    subprocess.check_call(["make", "-C", _HERE, "-s", "-f", "fuse_neighbours.mk", "ref"])


def lib():
    global _LIB
    if _LIB is None:
        so = os.path.join(_HERE, "libfuse_neighbours_oracle.so")
        if not os.path.exists(so):
            build()
        _LIB = C.CDLL(so)
    return _LIB


def oracle(sc):
    from ccm_slam_b200 import api
    keep = []
    cur, tg, T, pts, cp, cand = api.fuse_structs(sc, keep)
    fwd = np.full((T, len(cp)), -3, np.int32)
    bwd = np.full(len(cand), -3, np.int32)
    lib().orc_fuse_neighbours(C.byref(cur), tg, T, C.byref(pts), cp.ctypes.data_as(C.c_void_p), cand.ctypes.data_as(C.c_void_p), len(cand),
                              fwd.ctypes.data_as(C.c_void_p), bwd.ctypes.data_as(C.c_void_p))
    return fwd, bwd


class StandIn:
    """A scene of synth_match.make_fuse_scene as stand-in KeyFrame / MapPoint / LocalMapping objects (oracle/ref_stub_fn): keyframe 0 the
    current one, 1 + t target t, then a third keyframe that no target lists (third_point).  run(mode): 0 the literal restatement of
    LocalMapping::SearchInNeighbors (oracle/ref_fuse_neighbours_wrap.cpp), 1 shim/FuseNeighbours_shim.cpp; over the host entry point
    standing in for the device, or the real library with gpu=True."""

    def __init__(self, sc, gpu=False):
        from ccm_slam_b200 import api
        so = os.path.join(_HERE, "_ref", "libfuse_neighbours_shim_gpu.so" if gpu else "libfuse_neighbours_shim.so")
        if not os.path.exists(so):
            build()
        self.L = C.CDLL(so)
        self.L.fn_scene_create.restype = C.c_void_p
        self.L.fn_scene_destroy.argtypes = [C.c_void_p]
        self.L.fn_run.argtypes = [C.c_void_p, C.c_int]
        self.keep = []
        kfs = [sc["cur"]] + list(sc["targets"]) + [sc["cur"]]
        slots = [sc["cur_point"]] + list(sc["target_point"]) + [sc["third_point"]]
        K = len(kfs)
        arr = (api.FuseKfC * K)()
        for k, d in enumerate(kfs):
            sub = dict(sc, cur=d, targets=[])
            cur, _, _, _, _, _ = api.fuse_structs(sub, self.keep)
            arr[k] = cur
        conn = [[0 if c < 0 else 1 + c for c in row] for row in sc["conn"]] + [[]]
        cptr = np.concatenate([[0], np.cumsum([len(c) for c in conn])]).astype(np.int32)
        cflat = np.asarray([c for row in conn for c in row] or [0], np.int32)
        sptr = np.concatenate([[0], np.cumsum([len(s) for s in slots])]).astype(np.int32)
        sflat = np.concatenate([np.asarray(s, np.int32) for s in slots])
        p = sc["points"]
        bad = np.ascontiguousarray(p["bad"], np.uint8)
        a = dict(pos=np.ascontiguousarray(p["pos"], np.float32), nrm=np.ascontiguousarray(p["normal"], np.float32),
                 mx=np.ascontiguousarray(p["max_d"], np.float32), mn=np.ascontiguousarray(p["min_d"], np.float32),
                 desc=np.ascontiguousarray(p["desc"], np.uint8), dnr=(np.asarray(p["skip"], np.uint8) & (1 - bad)).astype(np.uint8), bad=bad,
                 kbad=np.zeros(K, np.uint8), cptr=cptr, cflat=cflat, sptr=sptr, sflat=sflat)
        self.keep += [arr, a]
        self.sizes = [len(s) for s in slots]
        self.P = len(a["mx"])
        v = lambda x: x.ctypes.data_as(C.c_void_p)  # noqa: E731
        self.h = C.c_void_p(self.L.fn_scene_create(K, arr, v(a["kbad"]), v(cptr), v(cflat), v(sptr), v(sflat), self.P, v(a["pos"]), v(a["nrm"]),
                                                   v(a["mx"]), v(a["mn"]), v(a["desc"]), v(a["dnr"]), v(a["bad"])))
        self.K = K

    def close(self):
        if self.h:
            self.L.fn_scene_destroy(self.h); self.h = None

    def run(self, mode):
        if self.L.fn_run(self.h, int(mode)) != 0:
            raise RuntimeError("the member threw")

    def members(self):
        """what the member changed: every keyframe's mvpMapPoints; per point bad, mpReplaced, descriptor, candidate mark, observations
        in map order and the members called on it; per keyframe the fuse-target mark and UpdateConnections calls"""
        P, K = self.P, self.K
        o = dict(mvp=np.zeros(sum(self.sizes), np.int32), bad=np.zeros(P, np.uint8), replaced=np.zeros(P, np.int32), desc=np.zeros((P, 32), np.uint8),
                 cand_mark=np.zeros(P, np.int64), obs_ptr=np.zeros(P + 1, np.int32), obs=np.zeros(64 * P + 2, np.int32),
                 log_ptr=np.zeros(P + 1, np.int32), log=np.zeros(64 * P + 1, np.uint8), target_mark=np.zeros(K, np.int64),
                 conn_updates=np.zeros(K, np.int32))
        v = lambda x: x.ctypes.data_as(C.c_void_p)  # noqa: E731
        self.L.fn_members(self.h, v(o["mvp"]), v(o["bad"]), v(o["replaced"]), v(o["desc"]), v(o["cand_mark"]), v(o["obs_ptr"]), v(o["obs"]),
                          len(o["obs"]), v(o["log_ptr"]), v(o["log"]), len(o["log"]), v(o["target_mark"]), v(o["conn_updates"]))
        o["obs"] = o["obs"][:o["obs_ptr"][-1]]
        o["log"] = o["log"][:o["log_ptr"][-1]]
        return o

    def stats(self):
        """(library calls made by the shim member, pairs searched again on the host) since the process started"""
        c = (C.c_ulonglong * 2)()
        self.L.fn_shim_stats(c)
        return np.array(c[:], np.int64)

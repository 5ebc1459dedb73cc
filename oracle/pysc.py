"""ctypes binding of the Sim3 correction checker (oracle/Makefile).  TEST INFRASTRUCTURE, NOT PRODUCT.

  oracle(sc, fn=None)    oracle/liboracle.so (sim3_correction_oracle.cpp): the entries walked in order as LoopFinder::CorrectLoop /
                         MapMerger::MergeMaps walk them, over the flat arrays of ccm_sim3_correction.  fn: any function with the
                         same C signature (the g++ build of the product's arithmetic in the tests) instead of the oracle
Returns the outputs of ccm_slam_b200.api.sim3_correction.
"""
from __future__ import annotations

import ctypes as C

from oracle import pyoracle


def oracle(sc, fn=None):
    from ccm_slam_b200 import api
    out = api.sim3_correction_out(len(sc["entry_kf"]), len(sc["mp_skip"]))
    argv, _keep = api.sim3_correction_args(sc, out)
    rc = (fn or pyoracle.lib().orc_sim3_correction)(*argv)
    if rc != 0:
        raise ValueError("orc_sim3_correction: bad input")
    return out


class StandIn:
    """a scene of stand-in KeyFrame / MapPoint objects (oracle/ref_stub_sc) from a synth.make_sim3_correction scene, with .literal(merge)
    (the reference loop restated on them), .shim(merge) (shim/Sim3Correction_shim.cpp) and .read(); over the CPU double of
    ccm_sim3_correction, or the real library with gpu=True.  The scene must give every observed point a reference keyframe."""

    def __init__(self, sc, gpu=False):
        self.L = pyoracle.ref_lib("libsim3_correction_shim_gpu.so" if gpu else "libsim3_correction_shim.so")
        self.L.sc_scene_create.restype = C.c_void_p
        self.L.sc_scene_destroy.argtypes = [C.c_void_p]
        self.L.sc_literal.argtypes = [C.c_void_p, C.c_int]
        self.L.sc_shim.argtypes = [C.c_void_p, C.c_int]
        self.L.sc_read.argtypes = [C.c_void_p] + [C.c_void_p] * 16
        self.L.sc_map_order.argtypes = [C.c_void_p, C.c_void_p]
        import numpy as np
        self.np = np
        k = self._keep = [np.ascontiguousarray(sc[n], t) for n, t in (
            ("kf_Tcw", np.float32), ("kf_bad", np.uint8), ("kf_rank", np.uint32), ("entry_kf", np.int32), ("entry_Siw_new", np.float64),
            ("entry_Siw_old", np.float64), ("slot_ptr", np.int64), ("slot_mp", np.int32), ("mp_pos", np.float32), ("mp_bad", np.uint8),
            ("mp_tagged", np.uint8), ("obs_ptr", np.int64), ("obs_kf", np.int32), ("mp_ref", np.int32))]
        self.K, self.E, self.P = len(k[1]), len(k[3]), len(k[9])
        p = [a.ctypes.data_as(C.c_void_p) for a in k]
        self.h = C.c_void_p(self.L.sc_scene_create(self.K, p[0], p[1], p[2], int(sc["cur"]), self.E, p[3], p[4], p[5], p[6], p[7], self.P, p[8],
                                                   p[9], p[10], p[11], p[12], p[13]))

    def close(self):
        if self.h:
            self.L.sc_scene_destroy(self.h); self.h = None

    def map_order(self):
        r = self.np.zeros(self.E, self.np.int32); self.L.sc_map_order(self.h, r.ctypes.data_as(C.c_void_p)); return r

    def literal(self, merge):
        self.L.sc_literal(self.h, int(merge))

    def shim(self, merge):
        if self.L.sc_shim(self.h, int(merge)) != 0:
            raise RuntimeError("ccm_b200_correct_sim3 threw")

    def read(self):
        np, K, P = self.np, self.K, self.P
        o = dict(Tcw=np.zeros((K, 16), np.float32), Twc=np.zeros((K, 16), np.float32), Ow=np.zeros((K, 3), np.float32),
                 corrected_mm=np.zeros((K, 2), np.uint64), conn=np.zeros((K, 2), np.int32), changed=np.zeros(K, np.uint8),
                 pos=np.zeros((P, 3), np.float32), normal=np.zeros((P, 3), np.float32), max_dist=np.zeros(P, np.float32),
                 min_dist=np.zeros(P, np.float32), written=np.zeros(P, np.uint8), tag_lc=np.zeros((P, 2), np.uint64),
                 tag_mm=np.zeros((P, 2), np.uint64), ref_lc=np.zeros(P, np.uint64), ref_mm=np.zeros(P, np.uint64))
        log = np.zeros(max(self.E, 1), np.int32)
        keys = ("Tcw", "Twc", "Ow", "corrected_mm", "conn", "changed", "pos", "normal", "max_dist", "min_dist", "written", "tag_lc", "tag_mm",
                "ref_lc", "ref_mm")
        n = self.L.sc_read(self.h, *[o[k].ctypes.data_as(C.c_void_p) for k in keys], log.ctypes.data_as(C.c_void_p))
        o["log"] = log[:n].copy()
        return o

    def stats(self):
        """(shim calls, points moved, fallbacks, normals parked hits, stale, host, keyframes prepared), process-wide"""
        c = (C.c_ulonglong * 7)()
        self.L.sc_stats(c)
        return self.np.array(c[:], self.np.int64)

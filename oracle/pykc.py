"""ctypes binding of the keyframe-culling checker (oracle/keyframe_culling.mk).  TEST INFRASTRUCTURE, NOT PRODUCT.

  oracle(sc, slip=0)   oracle/libkeyframe_culling_oracle.so: LocalMapping::KeyFrameCullingV3 walked literally over live state, on the
                       flat arrays of ccm_keyframe_culling -> dict(cull, n_mps, n_red) as api.keyframe_culling returns them (without
                       n_settled).  slip selects a deliberately wrong reading: 1 `>=`, 2 the f32 threshold, 3 no cascade, 4 the
                       candidate's own observation counted, 5 `<` on the octave.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = None
SLIPS = {"ge": 1, "f32": 2, "no_cascade": 3, "own": 4, "octave_lt": 5}


def build() -> None:
    subprocess.check_call(["make", "-C", _HERE, "-s", "-f", "keyframe_culling.mk", "ref"])


def lib():
    global _LIB
    if _LIB is None:
        so = os.path.join(_HERE, "libkeyframe_culling_oracle.so")
        if not os.path.exists(so):
            build()
        _LIB = C.CDLL(so)
    return _LIB


def oracle(sc, slip=0):
    from ccm_slam_b200 import api
    out = api.keyframe_culling_out(len(sc["cand_kf"]))
    argv, _keep = api.keyframe_culling_args(sc, out)
    if lib().orc_keyframe_culling(*argv[:-1], int(slip)) != 0:
        raise ValueError("orc_keyframe_culling: bad input")
    return dict(cull=out["cull"], n_mps=out["n_mps"], n_red=out["n_red"])


class StandIn:
    """A map scene of synth.make_keyframe_culling_scene as stand-in LocalMapping / KeyFrame / MapPoint / Map objects (oracle/ref_stub_kc):
    one KeyFrame per row (mId.first from kf_id, mvKeysUn octaves from the slots), one MapPoint per point, the query's ordered
    connections = covis, mlpRecentAddedKFs = recent, and GetRandKfPtr scripted to answer `picks` (rows, -1 for a null pointer) in turn
    (default: the query).  run(mode): 0 the literal restatement of KeyFrameCullingV3 (oracle/ref_keyframe_culling_wrap.cpp), 1
    shim/KeyFrameCulling_shim.cpp; over the host entry point standing in for the device, or the real library with gpu=True."""

    def __init__(self, sc, gpu=False, picks=None, checked=()):
        so = os.path.join(_HERE, "_ref", "libkeyframe_culling_shim_gpu.so" if gpu else "libkeyframe_culling_shim.so")
        if not os.path.exists(so):
            build()
        self.L = C.CDLL(so)
        self.L.kc_scene_create.restype = C.c_void_p
        self.L.kc_scene_destroy.argtypes = [C.c_void_p]
        self.L.kc_run.argtypes = [C.c_void_p, C.c_int]
        picks = [int(sc["query"])] if picks is None else list(picks)
        k = dict(kf_bad=np.ascontiguousarray(sc["kf_bad"], np.uint8), kf_not_erase=np.ascontiguousarray(sc["kf_not_erase"], np.uint8),
                 kf_id=np.ascontiguousarray(sc["kf_id"], np.int64), sptr=np.ascontiguousarray(sc["kf_slot_ptr"], np.int64),
                 smp=np.ascontiguousarray(sc["kf_slot_mp"], np.int32), soct=np.ascontiguousarray(sc["kf_slot_octave"], np.int32),
                 mp_bad=np.ascontiguousarray(sc["mp_bad"], np.uint8), nobs=np.ascontiguousarray(sc["mp_nobs"], np.int32),
                 ref=np.ascontiguousarray(sc["mp_ref"], np.int32), optr=np.ascontiguousarray(sc["obs_ptr"], np.int64),
                 okf=np.ascontiguousarray(sc["obs_kf"], np.int32), oidx=np.ascontiguousarray(sc["obs_idx"], np.int32),
                 covis=np.ascontiguousarray(sc["covis"], np.int32), recent=np.ascontiguousarray(sc["recent"], np.int32),
                 picks=np.ascontiguousarray(picks, np.int32), checked=np.ascontiguousarray(list(checked) or [0], np.int32))
        self.keep = k
        self.K, self.P, self.S = len(k["kf_bad"]), len(k["mp_bad"]), len(k["smp"])
        v = lambda x: x.ctypes.data_as(C.c_void_p)  # noqa: E731
        self.h = C.c_void_p(self.L.kc_scene_create(self.K, v(k["kf_bad"]), v(k["kf_not_erase"]), v(k["kf_id"]), v(k["sptr"]), v(k["smp"]),
                                                   v(k["soct"]), self.P, v(k["mp_bad"]), v(k["nobs"]), v(k["ref"]), v(k["optr"]), v(k["okf"]),
                                                   v(k["oidx"]), int(sc["query"]), v(k["covis"]), len(k["covis"]), v(k["recent"]),
                                                   len(k["recent"]), v(k["picks"]), len(picks), v(k["checked"]), len(checked)))

    def close(self):
        if self.h:
            self.L.kc_scene_destroy(self.h); self.h = None

    def run(self, mode):
        if self.L.kc_run(self.h, int(mode)) != 0:
            raise RuntimeError("the member threw")

    def members(self):
        """what the member left: per keyframe mbBad, mbToBeErased and mvpMapPoints; per point mbBad, nObs, mpRefKF and the observations
        (keyframe row, index) in map order; mCulledKfs and the set mspKFsCheckedForCulling"""
        K, P = self.K, self.P
        o = dict(kf_bad=np.zeros(K, np.uint8), to_be_erased=np.zeros(K, np.uint8), slots=np.zeros(self.S, np.int32), mp_bad=np.zeros(P, np.uint8),
                 nobs=np.zeros(P, np.int32), ref=np.zeros(P, np.int32), obs_ptr=np.zeros(P + 1, np.int64),
                 obs=np.zeros(2 * len(self.keep["okf"]) + 2, np.int32), culled=np.zeros(1, np.int64), checked=np.zeros(K, np.uint8))
        v = lambda x: x.ctypes.data_as(C.c_void_p)  # noqa: E731
        self.L.kc_members(self.h, v(o["kf_bad"]), v(o["to_be_erased"]), v(o["slots"]), v(o["mp_bad"]), v(o["nobs"]), v(o["ref"]), v(o["obs_ptr"]),
                          v(o["obs"]), v(o["culled"]), v(o["checked"]))
        o["obs"] = o["obs"][:2 * o["obs_ptr"][-1]]
        return o

    def stats(self):
        """(library calls made by the shim member, candidates counted again on the host) since the process started"""
        c = (C.c_ulonglong * 2)()
        self.L.kc_shim_stats(c)
        return np.array(c[:], np.int64)

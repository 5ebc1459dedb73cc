"""ctypes binding of the loop / merge fusion checker (oracle/search_and_fuse.mk).  TEST INFRASTRUCTURE, NOT PRODUCT.

  oracle(sc)   oracle/libsearch_and_fuse_oracle.so: every (corrected keyframe, loop point) pair LoopFinder / MapMerger::SearchAndFuse
               searches, Fuse(Scw)'s prelude with the host's logf and the reference-pinned window search, over a scene as
               synth_match.make_search_and_fuse_scene builds it -> best (K, P), shaped as api.search_and_fuse's first result.
               th, chi2, camera and skip select the wrong variants the tests must tell apart from the real one.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = None


def build() -> None:
    subprocess.check_call(["make", "-C", _HERE, "-s", "-f", "search_and_fuse.mk", "ref"])


def lib():
    global _LIB
    if _LIB is None:
        so = os.path.join(_HERE, "libsearch_and_fuse_oracle.so")
        if not os.path.exists(so):
            build()
        _LIB = C.CDLL(so)
    return _LIB


def oracle(sc, th=4.0, chi2=False, camera="split", skip="skip"):
    """camera "split": Tcw / Ow as Fuse(Scw) splits the corrected Scw; "pose": the keyframe's [R t/s] pose (Tcw_pose / Ow_pose).
    skip names the points' skip flags ("skip" = isBad())."""
    from ccm_slam_b200 import api
    keep = []
    T, O = ("Tcw", "Ow") if camera == "split" else ("Tcw_pose", "Ow_pose")
    kfs, K, pts = api.search_and_fuse_structs(sc, keep, T, O, skip)
    best = np.full((K, pts.n), -3, np.int32)
    lib().orc_search_and_fuse(kfs, K, C.byref(pts), C.c_float(th), int(chi2), best.ctypes.data_as(C.c_void_p))
    return best


class StandIn:
    """A scene of synth_match.make_search_and_fuse_scene as stand-in KeyFrame / MapPoint objects (oracle/ref_stub_sf) in a real
    KeyFrameAndPose: points 0..P-1 the loop points (vpLoopMapPoints in row order), then one occupant per kf_slot of -2.  run(mode, merge):
    mode 0 the literal restatement of LoopFinder / MapMerger::SearchAndFuse (oracle/ref_search_and_fuse_wrap.cpp), 1
    shim/SearchAndFuse_shim.cpp; over the host entry point standing in for the device, or the real library with gpu=True."""

    def __init__(self, sc, gpu=False, empty_kf=()):
        from ccm_slam_b200 import api
        so = os.path.join(_HERE, "_ref", "libsearch_and_fuse_shim_gpu.so" if gpu else "libsearch_and_fuse_shim.so")
        if not os.path.exists(so):
            build()
        self.L = C.CDLL(so)
        self.L.sf_scene_create.restype = C.c_void_p
        self.L.sf_scene_destroy.argtypes = [C.c_void_p]
        self.L.sf_run.argtypes = [C.c_void_p, C.c_int, C.c_int]
        self.keep = []
        kfs_c, K, _ = api.search_and_fuse_structs(sc, self.keep)
        p = sc["points"]
        P0 = len(p["skip"])
        slots, occ = [], 0
        for sl in sc["kf_slot"]:
            sl = np.asarray(sl, np.int32).copy()
            at = np.flatnonzero(sl == -2)
            sl[at] = P0 + occ + np.arange(len(at))
            occ += len(at)
            slots.append(sl)
        rng = np.random.default_rng(0)
        pad = lambda x, fill: np.concatenate([np.asarray(x), np.broadcast_to(fill, (occ,) + np.asarray(x).shape[1:])])  # noqa: E731
        a = dict(pos=np.ascontiguousarray(pad(p["pos"], np.float32(0)), np.float32), nrm=np.ascontiguousarray(pad(p["normal"], np.float32(0)), np.float32),
                 mx=np.ascontiguousarray(pad(p["max_d"], np.float32(1)), np.float32), mn=np.ascontiguousarray(pad(p["min_d"], np.float32(1)), np.float32),
                 desc=np.ascontiguousarray(np.concatenate([p["desc"], rng.integers(0, 256, (occ, 32), dtype=np.uint8)]), np.uint8),
                 bad=np.ascontiguousarray(pad(p["skip"], np.uint8(0)), np.uint8),
                 sim3=np.ascontiguousarray(np.stack([k["sim3"] for k in sc["kfs"]] or [np.zeros(8)]), np.float64),
                 empty=np.array([1 if k in empty_kf else 0 for k in range(K)], np.uint8),
                 sptr=np.concatenate([[0], np.cumsum([len(s) for s in slots])]).astype(np.int32), sflat=np.concatenate(slots + [np.zeros(1, np.int32)]).astype(np.int32),
                 loop=np.arange(P0, dtype=np.int32))
        self.keep.append(a)
        self.sizes = [len(s) for s in slots]
        self.P, self.K = len(a["bad"]), K
        v = lambda x: x.ctypes.data_as(C.c_void_p)  # noqa: E731
        self.h = C.c_void_p(self.L.sf_scene_create(K, kfs_c, v(a["sim3"]), v(a["empty"]), v(a["sptr"]), v(a["sflat"]), self.P, v(a["pos"]),
                                                   v(a["nrm"]), v(a["mx"]), v(a["mn"]), v(a["desc"]), v(a["bad"]), v(a["loop"]), P0))

    def close(self):
        if self.h:
            self.L.sf_scene_destroy(self.h); self.h = None

    def run(self, mode, merge):
        if self.L.sf_run(self.h, int(mode), int(merge)) != 0:
            raise RuntimeError("the member threw")

    def members(self):
        """what the member changed: every keyframe's mvpMapPoints and call log; per point bad, mpReplaced, descriptor, observations in
        map order and the members called on it (lower case unlocked, upper case with the lock flag)"""
        P, K = self.P, self.K
        o = dict(mvp=np.zeros(sum(self.sizes), np.int32), bad=np.zeros(P, np.uint8), replaced=np.zeros(P, np.int32), desc=np.zeros((P, 32), np.uint8),
                 obs_ptr=np.zeros(P + 1, np.int32), obs=np.zeros(64 * P + 2, np.int32), log_ptr=np.zeros(P + 1, np.int32),
                 log=np.zeros(64 * P + 1, np.uint8), klog_ptr=np.zeros(K + 1, np.int32), klog=np.zeros(64 * P + 1, np.uint8))
        v = lambda x: x.ctypes.data_as(C.c_void_p)  # noqa: E731
        self.L.sf_members(self.h, v(o["mvp"]), v(o["bad"]), v(o["replaced"]), v(o["desc"]), v(o["obs_ptr"]), v(o["obs"]), len(o["obs"]),
                          v(o["log_ptr"]), v(o["log"]), len(o["log"]), v(o["klog_ptr"]), v(o["klog"]), len(o["klog"]))
        o["obs"] = o["obs"][:o["obs_ptr"][-1]]
        o["log"] = o["log"][:o["log_ptr"][-1]]
        o["klog"] = o["klog"][:o["klog_ptr"][-1]]
        return o

    def stats(self):
        """(library calls made by the shim member, points searched again on the host) since the process started"""
        c = (C.c_ulonglong * 2)()
        self.L.sf_shim_stats(c)
        return np.array(c[:], np.int64)

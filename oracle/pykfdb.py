"""ctypes binding of the keyframe-database checker (oracle/Makefile).  TEST INFRASTRUCTURE, NOT PRODUCT.

  Oracle(n_words, scoring)     oracle/liboracle.so (kfdb_oracle.cpp): our restatement of S/Database.cpp's queries and DBoW2's six scores
  Reference(n_words, scoring)  oracle/_ref/libkfdb_ref.so: the reference's own Database.cpp / ScoringObject.cpp compiled in place
                               against stand-in KeyFrame / Map / Frame records (None where neither the reference tree nor a
                               prebuilt library is present)
  Shim / ShimGPU               this repository's shim/Database_shim.cpp in place of Database.cpp, same stand-ins and wrapper, over
                               the CPU double of the device entry points / the real library
Both take keyframe records (uid = mUniqueId, client, BowVector), covisibility lists, add / erase / clear, and the three queries, and
return the vector<kfptr> as uids; marker members can be read back after every call.
"""
from __future__ import annotations

import ctypes as C

import numpy as np

from oracle import pyoracle

NONE = np.uint64(0xFFFFFFFFFFFFFFFF)     # defpair
_LIBS = {}
_REF_SO = {"ref": "libkfdb_ref.so", "shim": "libkfdb_shim.so", "shim_gpu": "libkfdb_shim_gpu.so"}


def _load(kind):
    """kind: "orc" (the oracle), "ref" (the reference's Database.cpp), "shim" / "shim_gpu" (shim/Database_shim.cpp over the CPU double /
    the real device library); the last three share ref_kfdb_wrap.cpp's C interface"""
    if kind not in _LIBS:
        L = pyoracle.lib() if kind == "orc" else pyoracle.ref_lib(_REF_SO[kind])
        if L is None:
            return None
        prefix = "orc" if kind == "orc" else "ref"
        f = lambda name: getattr(L, f"{prefix}_{name}")
        f("kfdb_create").restype = C.c_void_p
        f("kfdb_create").argtypes = [C.c_int32, C.c_int32]
        for name in ("kfdb_destroy", "kfdb_clear"):
            f(name).argtypes = [C.c_void_p]
        f("kfdb_keyframe").argtypes = [C.c_void_p, C.c_uint64, C.c_uint32, C.c_int32, C.c_void_p, C.c_void_p]
        f("kfdb_set_covis").argtypes = [C.c_void_p, C.c_uint64, C.c_int32, C.c_void_p]
        f("kfdb_add").argtypes = [C.c_void_p, C.c_uint64]
        f("kfdb_erase").argtypes = [C.c_void_p, C.c_uint64]
        f("kfdb_detect_loop").argtypes = [C.c_void_p, C.c_uint64, C.c_float, C.c_int32, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p]
        f("kfdb_detect_map_match").argtypes = [C.c_void_p, C.c_uint64, C.c_float, C.c_int32, C.c_void_p, C.c_void_p]
        f("kfdb_detect_reloc").argtypes = [C.c_void_p, C.c_uint64, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p]
        for name in ("kfdb_detect_loop", "kfdb_detect_map_match", "kfdb_detect_reloc"):
            f(name).restype = C.c_int32
        f("kfdb_markers").argtypes = [C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p, C.c_void_p]
        if prefix == "orc":
            L.orc_bow_score.restype = C.c_double
            L.orc_bow_score.argtypes = [C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p]
            L.orc_kfdb_last_scored.restype = C.c_int32
            L.orc_kfdb_last_scored.argtypes = [C.c_void_p] * 5
        _LIBS[kind] = L
    return _LIBS[kind]


def _p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def _bow(word, value):
    return np.ascontiguousarray(word, np.uint32), np.ascontiguousarray(value, np.float64)


def bow_score(scoring, w1, v1, w2, v2):
    """mpVoc->score(v1, v2): DBoW2's ScoringObject restated (oracle side)"""
    w1, v1 = _bow(w1, v1); w2, v2 = _bow(w2, v2)
    return _load("orc").orc_bow_score(int(scoring), len(w1), _p(w1), _p(v1), len(w2), _p(w2), _p(v2))


class _DB:
    prefix = None
    kind = None

    def __init__(self, n_words, scoring=0):
        self.L = _load(self.kind)
        self.h = self.L and getattr(self.L, f"{self.prefix}_kfdb_create")(int(n_words), int(scoring))
        self.size_hint = 16

    def _f(self, name):
        return getattr(self.L, f"{self.prefix}_kfdb_{name}")

    def close(self):
        if self.h:
            self._f("destroy")(self.h); self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def keyframe(self, uid, client, word, value):
        w, v = _bow(word, value)
        self._f("keyframe")(self.h, int(uid), int(client), len(w), _p(w), _p(v))
        self.size_hint += 1

    def set_covis(self, uid, neighbours):
        nb = np.ascontiguousarray(neighbours, np.uint64)
        self._f("set_covis")(self.h, int(uid), len(nb), _p(nb))

    def add(self, uid):
        self._f("add")(self.h, int(uid))

    def erase(self, uid):
        self._f("erase")(self.h, int(uid))

    def clear(self):
        self._f("clear")(self.h)

    def _out(self):
        return np.zeros(self.size_hint + 16, np.uint64)

    def DetectLoopCandidates(self, q_uid, min_score, connected, in_map):
        c = np.ascontiguousarray(list(connected), np.uint64); m = np.ascontiguousarray(list(in_map), np.uint64); out = self._out()
        n = self._f("detect_loop")(self.h, int(q_uid), C.c_float(min_score), len(c), _p(c), len(m), _p(m), _p(out))
        return out[:n].copy()

    def DetectMapMatchCandidates(self, q_uid, min_score, assoc_clients):
        a = np.ascontiguousarray(list(assoc_clients), np.uint32); out = self._out()
        n = self._f("detect_map_match")(self.h, int(q_uid), C.c_float(min_score), len(a), _p(a), _p(out))
        return out[:n].copy()

    def DetectRelocalizationCandidates(self, frame_id, word, value):
        w, v = _bow(word, value); out = self._out()
        n = self._f("detect_reloc")(self.h, int(frame_id), len(w), _p(w), _p(v), _p(out))
        return out[:n].copy()

    def markers(self, uid):
        """(mLoopQuery, mMatchQuery, mRelocQuery), (mnLoopWords, mnRelocWords), (mLoopScore, mRelocScore) as raw values"""
        q = np.zeros(3, np.uint64); i = np.zeros(2, np.int32); f = np.zeros(2, np.float32)
        self._f("markers")(self.h, int(uid), _p(q), _p(i), _p(f))
        return q, i, f


class Oracle(_DB):
    prefix = kind = "orc"

    def last_scored(self):
        """the scored list of the last query (what the device returns): uid, shared words, f64 score; and max / min common words"""
        cap = self.size_hint + 16
        uid = np.zeros(cap, np.uint64); words = np.zeros(cap, np.int32); sc = np.zeros(cap); hdr = np.zeros(3, np.int32)
        n = self.L.orc_kfdb_last_scored(self.h, _p(uid), _p(words), _p(sc), _p(hdr))
        return dict(uid=uid[:n].copy(), n_words=words[:n].copy(), score_f64=sc[:n].copy(), max_common=int(hdr[0]), min_common=int(hdr[1]),
                    n_sharing=int(hdr[2]))


class Reference(_DB):
    prefix = kind = "ref"

    @classmethod
    def available(cls):
        return _load(cls.kind) is not None


class Shim(Reference):
    """shim/Database_shim.cpp behind the same wrapper, device entry points doubled on the CPU (oracle/_ref/libkfdb_shim.so)"""
    kind = "shim"


class ShimGPU(Reference):
    """shim/Database_shim.cpp over the real library (oracle/_ref/libkfdb_shim_gpu.so)"""
    kind = "shim_gpu"

"""Host-side mirror of the reference's ORB front-end interface on top of the C ABI (ctypes).

  ORBextractor(nfeatures, scaleFactor, nlevels, iniThFAST, minThFAST)  ~ cslam::ORBextractor  (I/ORBextractor.h:103-138)
  ORBmatcher(nnratio, checkOri).SearchByBoW / SearchForTriangulation   ~ cslam::ORBmatcher    (I/ORBmatcher.h:97-145)
      .SearchByProjection_* / Fuse / SearchBySim3                       ~ the projection-guided overloads (S/ORBmatcher.cpp:71-148,
                                                                          308-446, 854-1348, 1350-1605), from GetFeaturesInArea on
  ORBVocabulary(rows).transform(descriptors, levelsup)                 ~ DBoW2 TemplatedVocabulary::transform (D/TemplatedVocabulary.h:1127-1192)

Same names, argument meaning and outputs as the reference classes, on flat numpy arrays instead of cv::Mat / KeyFrame.
"""
from __future__ import annotations

import ctypes as C

import numpy as np

from . import api
from .api import FeatureVectorC, KeyPointC, ORBConfigC, TriViewC, _chk, _p, lib

KP_DTYPE = np.dtype([("x", "f4"), ("y", "f4"), ("size", "f4"), ("angle", "f4"), ("response", "f4"), ("octave", "i4")])


class ORBextractor:
    def __init__(self, nfeatures=1000, scaleFactor=1.2, nlevels=8, iniThFAST=20, minThFAST=7, width=752, height=480, blur_2413=False):
        self.cfg = ORBConfigC(nfeatures, scaleFactor, nlevels, iniThFAST, minThFAST, int(blur_2413))
        self.width, self.height, self.nlevels = width, height, nlevels
        self._h = C.c_void_p()
        _chk(lib().ccm_orb_create(C.byref(self.cfg), width, height, C.byref(self._h)))
        n = C.c_int32()
        _chk(lib().ccm_orb_max_keypoints(self._h, C.byref(n)))
        self.max_kp = n.value

    def __call__(self, image):
        """operator()(image, mask, keypoints, descriptors): returns (keypoints structured array, descriptors N x 32 u8)."""
        img = np.ascontiguousarray(image, np.uint8)
        assert img.shape == (self.height, self.width)
        kps = np.zeros(self.max_kp, KP_DTYPE); desc = np.zeros((self.max_kp, 32), np.uint8); n = C.c_int32()
        _chk(lib().ccm_orb_extract(self._h, _p(img), img.strides[0], _p(kps), self.max_kp, C.byref(n), _p(desc)))
        return kps[:n.value].copy(), desc[:n.value].copy()

    def image_pyramid(self, level):
        """mvImagePyramid[level]"""
        w = C.c_int32(); h = C.c_int32()
        _chk(lib().ccm_orb_get_level(self._h, level, None, C.byref(w), C.byref(h)))
        out = np.empty((h.value, w.value), np.uint8)
        _chk(lib().ccm_orb_get_level(self._h, level, _p(out), C.byref(w), C.byref(h)))
        return out

    def close(self):
        if self._h:
            lib().ccm_orb_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class FeatureVector:
    """DBoW2::FeatureVector flattened (nodes ascending; features per node in insertion order)."""

    def __init__(self, node_of_feature):
        node_of_feature = np.asarray(node_of_feature)
        order = np.argsort(node_of_feature, kind="stable")
        nodes, counts = np.unique(node_of_feature, return_counts=True)
        self.node_id = nodes.astype(np.uint32)
        self.node_ptr = np.concatenate([[0], np.cumsum(counts)]).astype(np.int32)
        self.feat = order.astype(np.uint32)

    def c(self):
        return FeatureVectorC(len(self.node_id), _p(self.node_id), _p(self.node_ptr), _p(self.feat))


class ORBmatcher:
    TH_LOW, TH_HIGH, HISTO_LENGTH = 50, 100, 30

    def __init__(self, nnratio=0.6, checkOri=True):
        self.nnratio, self.checkOri = float(nnratio), bool(checkOri)

    @staticmethod
    def DescriptorDistance(a, b):
        return int(api.hamming_matrix(np.asarray(a).reshape(1, 32), np.asarray(b).reshape(1, 32))[0, 0])

    def SearchByBoW_KF_Frame(self, desc_kf, kf_has_mp, angle_kf, fv_kf, desc_f, angle_f, fv_f, D=None):
        """D: optional precomputed distance matrix (n_kf x n_f u16) -> host selection only (ccm_select_bow_kf_frame)"""
        desc_kf = np.ascontiguousarray(desc_kf, np.uint8); desc_f = np.ascontiguousarray(desc_f, np.uint8)
        has = np.ascontiguousarray(kf_has_mp, np.uint8); ak = np.ascontiguousarray(angle_kf, np.float32); af = np.ascontiguousarray(angle_f, np.float32)
        out = np.empty(desc_f.shape[0], np.int32); n = C.c_int32()
        fk, ff = fv_kf.c(), fv_f.c()
        if D is not None:
            D = np.ascontiguousarray(D, np.uint16)
            _chk(lib().ccm_select_bow_kf_frame(_p(D), desc_kf.shape[0], _p(has), _p(ak), C.byref(fk), desc_f.shape[0], _p(af), C.byref(ff),
                                               C.c_float(self.nnratio), int(self.checkOri), _p(out), C.byref(n)))
            return out, n.value
        _chk(lib().ccm_match_bow_kf_frame(_p(desc_kf), desc_kf.shape[0], _p(has), _p(ak), C.byref(fk), _p(desc_f), desc_f.shape[0], _p(af),
                                          C.byref(ff), C.c_float(self.nnratio), int(self.checkOri), _p(out), C.byref(n)))
        return out, n.value

    def SearchByBoW_KF_KF(self, d1, has1, a1, fv1, d2, has2, a2, fv2, D=None):
        d1 = np.ascontiguousarray(d1, np.uint8); d2 = np.ascontiguousarray(d2, np.uint8)
        has1 = np.ascontiguousarray(has1, np.uint8); has2 = np.ascontiguousarray(has2, np.uint8)
        a1 = np.ascontiguousarray(a1, np.float32); a2 = np.ascontiguousarray(a2, np.float32)
        out = np.empty(d1.shape[0], np.int32); n = C.c_int32()
        f1, f2 = fv1.c(), fv2.c()
        if D is not None:
            D = np.ascontiguousarray(D, np.uint16)
            _chk(lib().ccm_select_bow_kf_kf(_p(D), d1.shape[0], _p(has1), _p(a1), C.byref(f1), d2.shape[0], _p(has2), _p(a2), C.byref(f2),
                                            C.c_float(self.nnratio), int(self.checkOri), _p(out), C.byref(n)))
            return out, n.value
        _chk(lib().ccm_match_bow_kf_kf(_p(d1), d1.shape[0], _p(has1), _p(a1), C.byref(f1), _p(d2), d2.shape[0], _p(has2), _p(a2), C.byref(f2),
                                       C.c_float(self.nnratio), int(self.checkOri), _p(out), C.byref(n)))
        return out, n.value

    def SearchForTriangulation(self, v1, v2, F12, ex, ey, level_sigma2, scale_factors, D=None):
        keep = []

        def view(v):
            arrs = dict(desc=np.ascontiguousarray(v["desc"], np.uint8), has=np.ascontiguousarray(v["has_mp"], np.uint8),
                        xy=np.ascontiguousarray(v["kp_xy"], np.float32), oc=np.ascontiguousarray(v["octave"], np.int32),
                        an=np.ascontiguousarray(v["angle"], np.float32))
            fv = v["fv"].c(); keep.extend([arrs, fv])
            fx, fy, cx, cy = v["intr"]
            return TriViewC(_p(arrs["desc"]), arrs["desc"].shape[0], _p(arrs["has"]), _p(arrs["xy"]), _p(arrs["oc"]), _p(arrs["an"]),
                            C.pointer(fv), fx, fy, cx, cy)
        a, b = view(v1), view(v2)
        F = np.ascontiguousarray(F12, np.float32); ls = np.ascontiguousarray(level_sigma2, np.float32); sf = np.ascontiguousarray(scale_factors, np.float32)
        pairs = np.empty((min(a.n, b.n) + 1, 2), np.int32); n = C.c_int32()
        if D is not None:
            D = np.ascontiguousarray(D, np.uint16)
            _chk(lib().ccm_select_triangulation(_p(D), C.byref(a), C.byref(b), _p(F), C.c_float(ex), C.c_float(ey), _p(ls), _p(sf), len(ls),
                                                int(self.checkOri), _p(pairs), C.byref(n)))
            return pairs[:n.value].copy()
        _chk(lib().ccm_match_triangulation(C.byref(a), C.byref(b), _p(F), C.c_float(ex), C.c_float(ey), _p(ls), _p(sf), len(ls),
                                           int(self.checkOri), _p(pairs), C.byref(n)))
        return pairs[:n.value].copy()

    # ---- projection-guided overloads (SURVEY.md §8(f) rank 3).  g = grid dict, q = query dict (ccm_slam_b200.synth_match) ----
    def SearchByProjection_Track(self, g, q, query_has_obs, feat_blocked, D=None):
        """SearchByProjection(Frame&, const vector<mpptr>&, th)  (S/ORBmatcher.cpp:71-148); nnratio from the constructor.
        D: optional precomputed distance matrix (m x n u16) -> host selection only (ccm_select_*)."""
        keep = []; G = grid_struct(g, keep); Q = queries_struct(q, keep)
        ho = np.ascontiguousarray(query_has_obs, np.uint8); fb = np.ascontiguousarray(feat_blocked, np.uint8)
        out = np.empty(G.n, np.int32); n = C.c_int32()
        if D is None:
            _chk(lib().ccm_search_by_projection_track(C.byref(G), C.byref(Q), _p(ho), _p(fb), C.c_float(self.nnratio), _p(out), C.byref(n)))
        else:
            D = _dist(D, Q.m, G.n)
            _chk(lib().ccm_select_by_projection_track(C.byref(G), C.byref(Q), _p(D), _p(ho), _p(fb), C.c_float(self.nnratio), _p(out), C.byref(n)))
        return out, n.value

    def SearchByProjection_Frame(self, g, q, query_has_obs, feat_blocked, reloc=False, ORBdist=100, D=None):
        """reloc=False: SearchByProjection(Frame&, const Frame& LastFrame, th) (:1350-1476);
        reloc=True: SearchByProjection(Frame&, kfptr, sAlreadyFound, th, ORBdist) (:1478-1605).  checkOri from the constructor."""
        keep = []; G = grid_struct(g, keep); Q = queries_struct(q, keep)
        ho = np.ascontiguousarray(query_has_obs, np.uint8); fb = np.ascontiguousarray(feat_blocked, np.uint8)
        out = np.empty(G.n, np.int32); n = C.c_int32()
        if D is None:
            _chk(lib().ccm_search_by_projection_frame(C.byref(G), C.byref(Q), _p(ho), _p(fb), int(reloc), int(ORBdist), int(self.checkOri),
                                                      _p(out), C.byref(n)))
        else:
            D = _dist(D, Q.m, G.n)
            _chk(lib().ccm_select_by_projection_frame(C.byref(G), C.byref(Q), _p(D), _p(ho), _p(fb), int(reloc), int(ORBdist),
                                                      int(self.checkOri), _p(out), C.byref(n)))
        return out, n.value

    def SearchByProjection_Sim3(self, g, q, feat_matched, existing_idx, D=None):
        """SearchByProjection(kfptr, Scw, vpPoints, vpMatched, th)  (:308-446) -> (best_idx per query, match_of_feat, nmatches)"""
        keep = []; G = grid_struct(g, keep); Q = queries_struct(q, keep)
        fm = np.ascontiguousarray(feat_matched, np.uint8); ex = np.ascontiguousarray(existing_idx, np.int32)
        best = np.empty(Q.m, np.int32); out = np.empty(G.n, np.int32); n = C.c_int32()
        if D is None:
            _chk(lib().ccm_search_by_projection_sim3(C.byref(G), C.byref(Q), _p(fm), _p(ex), _p(best), _p(out), C.byref(n)))
        else:
            D = _dist(D, Q.m, G.n)
            _chk(lib().ccm_select_by_projection_sim3(C.byref(G), C.byref(Q), _p(D), _p(fm), _p(ex), _p(best), _p(out), C.byref(n)))
        return best, out, n.value

    def Fuse(self, g, q, inv_level_sigma2=None, D=None):
        """search half of Fuse(kfptr, vpMapPoints, th) (:854-993, pass mvInvLevelSigma2) / Fuse(kfptr, Scw, ...) (:995-1122, None)"""
        keep = []; G = grid_struct(g, keep); Q = queries_struct(q, keep)
        w = None if inv_level_sigma2 is None else np.ascontiguousarray(inv_level_sigma2, np.float32)
        nl = 0 if w is None else len(w)
        best = np.empty(Q.m, np.int32); n = C.c_int32()
        if D is None:
            _chk(lib().ccm_fuse_search(C.byref(G), C.byref(Q), _p(w), nl, _p(best), C.byref(n)))
        else:
            D = _dist(D, Q.m, G.n)
            _chk(lib().ccm_fuse_select(C.byref(G), C.byref(Q), _p(D), _p(w), nl, _p(best), C.byref(n)))
        return best, n.value

    def SearchBySim3(self, g1, g2, q12, q21, D12=None, D21=None):
        """SearchBySim3(pKF1, pKF2, vpMatches12, s12, R12, t12, th)  (:1124-1348) -> (match12, nFound)"""
        keep = []; G1 = grid_struct(g1, keep); G2 = grid_struct(g2, keep); Q12 = queries_struct(q12, keep); Q21 = queries_struct(q21, keep)
        out = np.empty(Q12.m, np.int32); n = C.c_int32()
        if D12 is None:
            _chk(lib().ccm_search_by_sim3(C.byref(G1), C.byref(G2), C.byref(Q12), C.byref(Q21), _p(out), C.byref(n)))
        else:
            D12 = _dist(D12, Q12.m, G2.n); D21 = _dist(D21, Q21.m, G1.n)
            _chk(lib().ccm_select_by_sim3(C.byref(G1), C.byref(G2), C.byref(Q12), C.byref(Q21), _p(D12), _p(D21), _p(out), C.byref(n)))
        return out, n.value

    def SearchForInitialization(self, g2, q, D=None):
        """SearchForInitialization(F1, F2, vbPrevMatched, vnMatches12, windowSize)  (:448-563) -> (vnMatches12, nmatches);
        q: one query per keypoint of F1 (level = octave, uv = vbPrevMatched, radius = windowSize)."""
        keep = []; G = grid_struct(g2, keep); Q = queries_struct(q, keep)
        out = np.empty(Q.m, np.int32); n = C.c_int32()
        if D is None:
            _chk(lib().ccm_search_for_initialization(C.byref(G), C.byref(Q), C.c_float(self.nnratio), int(self.checkOri), _p(out), C.byref(n)))
        else:
            D = _dist(D, Q.m, G.n)
            _chk(lib().ccm_select_for_initialization(C.byref(G), C.byref(Q), _p(D), C.c_float(self.nnratio), int(self.checkOri), _p(out), C.byref(n)))
        return out, n.value


class FeatureGridC(C.Structure):
    _fields_ = [("n", C.c_int32), ("desc", C.c_void_p), ("kp_xy", C.c_void_p), ("octave", C.c_void_p), ("angle", C.c_void_p),
                ("min_x", C.c_float), ("min_y", C.c_float), ("max_x", C.c_float), ("max_y", C.c_float),
                ("grid_w_inv", C.c_float), ("grid_h_inv", C.c_float), ("grid_cols", C.c_int32), ("grid_rows", C.c_int32)]


class ProjQueriesC(C.Structure):
    _fields_ = [("m", C.c_int32), ("valid", C.c_void_p), ("uv", C.c_void_p), ("radius", C.c_void_p), ("level", C.c_void_p),
                ("desc", C.c_void_p), ("angle", C.c_void_p)]


def _dist(D, m, n):
    D = np.ascontiguousarray(D, np.uint16)
    assert D.shape == (m, n)
    return D


def grid_struct(g, keep):
    """ccm_feature_grid from dict(desc, kp_xy, octave, angle, bounds=(mnMinX, mnMinY, mnMaxX, mnMaxY), cols, rows)"""
    a = dict(desc=np.ascontiguousarray(g["desc"], np.uint8), xy=np.ascontiguousarray(g["kp_xy"], np.float32),
             oc=np.ascontiguousarray(g["octave"], np.int32), an=np.ascontiguousarray(g["angle"], np.float32))
    keep.append(a)
    x0, y0, x1, y1 = [np.float32(v) for v in g["bounds"]]
    wi = np.float32(g["cols"]) / np.float32(x1 - x0)   # mfGridElementWidthInv  (S/Frame.cpp:86)
    hi = np.float32(g["rows"]) / np.float32(y1 - y0)   # mfGridElementHeightInv (S/Frame.cpp:87)
    return FeatureGridC(a["desc"].shape[0], _p(a["desc"]), _p(a["xy"]), _p(a["oc"]), _p(a["an"]), x0, y0, x1, y1, wi, hi,
                        int(g["cols"]), int(g["rows"]))


def queries_struct(q, keep):
    """ccm_proj_queries from dict(valid, uv, radius, level, desc[, angle])"""
    m = len(q["valid"])
    a = dict(valid=np.ascontiguousarray(q["valid"], np.uint8), uv=np.ascontiguousarray(q["uv"], np.float32),
             r=np.ascontiguousarray(q["radius"], np.float32), lv=np.ascontiguousarray(q["level"], np.int32),
             desc=np.ascontiguousarray(q["desc"], np.uint8), an=np.ascontiguousarray(q.get("angle", np.zeros(m)), np.float32))
    keep.append(a)
    return ProjQueriesC(m, _p(a["valid"]), _p(a["uv"]), _p(a["r"]), _p(a["lv"]), _p(a["desc"]), _p(a["an"]))


def GetFeaturesInArea(g, x, y, r, minLevel=-1, maxLevel=-1):
    """Frame::GetFeaturesInArea (S/Frame.cpp:200-253); with the default levels also KeyFrame's (S/KeyFrame.cpp:1162-1201).  Host only."""
    keep = []; G = grid_struct(g, keep)
    out = np.empty(G.n + 1, np.int32); n = C.c_int32()
    _chk(lib().ccm_features_in_area(C.byref(G), C.c_float(x), C.c_float(y), C.c_float(r), int(minLevel), int(maxLevel), _p(out), G.n, C.byref(n)))
    return out[:n.value].copy()


def bow_assemble(scoring, weighting, word, weight, node):
    """The container half of DBoW2's transform (host only): per-feature (word, weight, node) -> BowVector, FeatureVector."""
    word = np.ascontiguousarray(word, np.uint32); weight = np.ascontiguousarray(weight, np.float64); node = np.ascontiguousarray(node, np.uint32)
    n = len(word)
    bid = np.empty(n, np.uint32); bval = np.empty(n, np.float64); bn = C.c_int32()
    fid = np.empty(n, np.uint32); fptr = np.empty(n + 1, np.int32); ff = np.empty(n, np.uint32); fn = C.c_int32()
    _chk(lib().ccm_bow_assemble(int(scoring), int(weighting), n, _p(word), _p(weight), _p(node), _p(bid), _p(bval), C.byref(bn),
                                _p(fid), _p(fptr), _p(ff), C.byref(fn)))
    return dict(bow_id=bid[:bn.value].copy(), bow_val=bval[:bn.value].copy(), fv_node_id=fid[:fn.value].copy(),
                fv_node_ptr=fptr[:fn.value + 1].copy(), fv_feat=ff[:fptr[fn.value] if fn.value else 0].copy())


class ORBVocabulary:
    """DBoW2::TemplatedVocabulary<FORB> resident on the device.  `v` holds the rows of the text file (row 0 = root):
    dict(k, L, scoring, weighting, parent, is_leaf, desc, weight) — see load_text() for ORBvoc.txt itself."""

    def __init__(self, v):
        parent = np.ascontiguousarray(v["parent"], np.int32); leaf = np.ascontiguousarray(v["is_leaf"], np.uint8)
        desc = np.ascontiguousarray(v["desc"], np.uint8); weight = np.ascontiguousarray(v["weight"], np.float64)
        assert desc.shape == (len(parent), 32)
        self.h = C.c_void_p()
        _chk(lib().ccm_voc_create(int(v["k"]), int(v["L"]), int(v["scoring"]), int(v["weighting"]), len(parent), _p(parent), _p(leaf),
                                  _p(desc), _p(weight), C.byref(self.h)))

    @staticmethod
    def load_text(path):
        """Rows of an ORBvoc.txt-style file (loadFromTextFile, D/TemplatedVocabulary.h:1338-1422) as the dict the constructor takes."""
        with open(path) as f:
            k, L, n1, n2 = [int(t) for t in f.readline().split()[:4]]
            rows = np.loadtxt(f, dtype=np.float64, ndmin=2)
        n = rows.shape[0] + 1
        parent = np.zeros(n, np.int32); leaf = np.zeros(n, np.uint8); desc = np.zeros((n, 32), np.uint8); weight = np.zeros(n, np.float64)
        parent[1:] = rows[:, 0].astype(np.int32); leaf[1:] = rows[:, 1] > 0
        desc[1:] = rows[:, 2:34].astype(np.uint8); weight[1:] = rows[:, 34]
        return dict(k=k, L=L, scoring=n1, weighting=n2, parent=parent, is_leaf=leaf, desc=desc, weight=weight)

    def words(self):
        return lib().ccm_voc_words(self.h)

    def transform(self, desc, levelsup=4):
        """-> dict(word, node, weight per feature; bow_id/bow_val = BowVector; fv_node_id/fv_node_ptr/fv_feat = FeatureVector)"""
        desc = np.ascontiguousarray(desc, np.uint8); n = desc.shape[0]
        word = np.empty(n, np.uint32); node = np.empty(n, np.uint32); w = np.empty(n, np.float64)
        bid = np.empty(n, np.uint32); bval = np.empty(n, np.float64); bn = C.c_int32()
        fid = np.empty(n, np.uint32); fptr = np.empty(n + 1, np.int32); ff = np.empty(n, np.uint32); fn = C.c_int32()
        _chk(lib().ccm_voc_transform(self.h, _p(desc), n, int(levelsup), _p(word), _p(node), _p(w), _p(bid), _p(bval), C.byref(bn),
                                     _p(fid), _p(fptr), _p(ff), C.byref(fn)))
        return dict(word=word, node=node, weight=w, bow_id=bid[:bn.value].copy(), bow_val=bval[:bn.value].copy(),
                    fv_node_id=fid[:fn.value].copy(), fv_node_ptr=fptr[:fn.value + 1].copy(), fv_feat=ff[:fptr[fn.value] if fn.value else 0].copy())

    def close(self):
        if self.h:
            lib().ccm_voc_destroy(self.h); self.h = C.c_void_p()


WIRE_KP_DTYPE = np.dtype([("x", "<f4"), ("y", "<f4"), ("size", "u1"), ("angle", "<f4"), ("response", "u1"), ("octave", "i1")])   # packed: 15 bytes
assert WIRE_KP_DTYPE.itemsize == 15


def wire_keypoints(kps):
    """ccmslam_msgs/CvKeyPoint[] as ROS serialises it, from a KP_DTYPE array (Converter::toCvKeyPointMsg, S/Converter.cc:166-178:
    size and response are truncated to uint8, octave to int8)"""
    w = np.zeros(len(kps), WIRE_KP_DTYPE)
    w["x"], w["y"], w["angle"] = kps["x"], kps["y"], kps["angle"]
    w["size"] = kps["size"].astype(np.uint8); w["response"] = kps["response"].astype(np.uint8); w["octave"] = kps["octave"].astype(np.int8)
    return w


def wire_keypoints_decode(wire):
    """host only: Converter::fromCvKeyPointMsg over n packed wire records"""
    wire = np.ascontiguousarray(wire)
    out = np.zeros(len(wire), KP_DTYPE)
    _chk(lib().ccm_wire_keypoints_decode(_p(wire.view(np.uint8)), len(wire), _p(out)))
    return out


class KeyFrameStore:
    """Device-resident keyframe features (SURVEY.md §8(f) rank 4): descriptors uploaded once at ingest (KeyFrame::WriteMembersFromMessage,
    S/KeyFrame.cpp:1662-1726), server-side matchers address keyframes by mUniqueId."""

    def __init__(self):
        self._h = C.c_void_p()
        L = lib()
        L.ccm_kfstore_features.restype = C.c_int32
        L.ccm_kfstore_keyframes.restype = C.c_int64
        L.ccm_kfstore_h2d_bytes.restype = C.c_int64
        for f in (L.ccm_kfstore_features, L.ccm_kfstore_erase):
            f.argtypes = [C.c_void_p, C.c_uint64]
        L.ccm_kfstore_keyframes.argtypes = [C.c_void_p]; L.ccm_kfstore_h2d_bytes.argtypes = [C.c_void_p]
        L.ccm_kfstore_destroy.argtypes = [C.c_void_p]
        _chk(L.ccm_kfstore_create(C.byref(self._h)))

    def close(self):
        if self._h:
            lib().ccm_kfstore_destroy(self._h)
            self._h = C.c_void_p()

    def put_wire(self, uid, wire_kps, desc):
        wire_kps = np.ascontiguousarray(wire_kps); desc = np.ascontiguousarray(desc, np.uint8)
        out = np.zeros(len(wire_kps), KP_DTYPE)
        _chk(lib().ccm_kfstore_put_wire(self._h, C.c_uint64(uid), len(wire_kps), _p(wire_kps.view(np.uint8)), _p(desc), _p(out)))
        return out

    def put(self, uid, kps, desc):
        kps = np.ascontiguousarray(kps); desc = np.ascontiguousarray(desc, np.uint8)
        _chk(lib().ccm_kfstore_put(self._h, C.c_uint64(uid), len(kps), _p(kps), _p(desc)))

    def erase(self, uid):
        _chk(lib().ccm_kfstore_erase(self._h, C.c_uint64(uid)))

    def features(self, uid):
        return lib().ccm_kfstore_features(self._h, C.c_uint64(uid))

    def keyframes(self):
        return lib().ccm_kfstore_keyframes(self._h)

    def h2d_bytes(self):
        return lib().ccm_kfstore_h2d_bytes(self._h)

    def get(self, uid):
        n = self.features(uid)
        kps = np.zeros(max(n, 0), KP_DTYPE); desc = np.zeros((max(n, 0), 32), np.uint8)
        _chk(lib().ccm_kfstore_get(self._h, C.c_uint64(uid), _p(kps), _p(desc)))
        return kps, desc

    def hamming(self, uid1, uid2):
        D = np.zeros((max(self.features(uid1), 0), max(self.features(uid2), 0)), np.uint16)   # unknown ids: the call reports them
        _chk(lib().ccm_kfstore_hamming(self._h, C.c_uint64(uid1), C.c_uint64(uid2), _p(D)))
        return D

    def hamming_query(self, Q, uid):
        Q = np.ascontiguousarray(Q, np.uint8)
        D = np.zeros((len(Q), max(self.features(uid), 0)), np.uint16)
        _chk(lib().ccm_kfstore_hamming_query(self._h, _p(Q), len(Q), C.c_uint64(uid), _p(D)))
        return D

    def SearchByBoW_KF_KF(self, uid1, has1, fv1, uid2, has2, fv2, nnratio=0.6, checkOri=True):
        has1 = np.ascontiguousarray(has1, np.uint8); has2 = np.ascontiguousarray(has2, np.uint8)
        out = np.empty(max(self.features(uid1), 0), np.int32); n = C.c_int32()
        f1, f2 = fv1.c(), fv2.c()
        _chk(lib().ccm_kfstore_match_bow_kf_kf(self._h, C.c_uint64(uid1), _p(has1), C.byref(f1), C.c_uint64(uid2), _p(has2), C.byref(f2),
                                               C.c_float(nnratio), int(checkOri), _p(out), C.byref(n)))
        return out, n.value

    def transform(self, uid, voc, levelsup=4):
        """as ORBVocabulary.transform, over the resident descriptors of keyframe uid"""
        n = max(self.features(uid), 0)
        word = np.zeros(n, np.uint32); node = np.zeros(n, np.uint32); weight = np.zeros(n)
        bow_id = np.zeros(n, np.uint32); bow_val = np.zeros(n); bn = C.c_int32()
        fid = np.zeros(n, np.uint32); fptr = np.zeros(n + 1, np.int32); ffeat = np.zeros(n, np.uint32); fn = C.c_int32()
        _chk(lib().ccm_kfstore_transform(self._h, C.c_uint64(uid), voc.h, int(levelsup), _p(word), _p(node), _p(weight), _p(bow_id), _p(bow_val),
                                         C.byref(bn), _p(fid), _p(fptr), _p(ffeat), C.byref(fn)))
        return dict(word=word, node=node, weight=weight, bow_id=bow_id[:bn.value].copy(), bow_val=bow_val[:bn.value].copy(),
                    fv_node_id=fid[:fn.value].copy(), fv_node_ptr=fptr[:fn.value + 1].copy(), fv_feat=ffeat[:fptr[fn.value] if fn.value else 0].copy())

    def distinctive_descriptors(self, kf_uid, kf_bad, obs_ptr, obs_kf, obs_feat):
        """MapPoint::ComputeDistinctiveDescriptors for a batch of points over the resident descriptors (ccm_kfstore_distinctive_descriptors):
        keyframe row k is uid kf_uid[k]; observation j is feature obs_feat[j] of row obs_kf[j].  Returns dict(best, best_median, desc)
        as api.distinctive_descriptors."""
        uid = np.ascontiguousarray(kf_uid, np.uint64); bad = np.ascontiguousarray(kf_bad, np.uint8)
        ptr = np.ascontiguousarray(obs_ptr, np.int64); okf = np.ascontiguousarray(obs_kf, np.int32); feat = np.ascontiguousarray(obs_feat, np.int32)
        P = len(ptr) - 1
        out = dict(best=np.zeros(P, np.int32), best_median=np.zeros(P, np.int32), desc=np.zeros((P, 32), np.uint8))
        _chk(lib().ccm_kfstore_distinctive_descriptors(self._h, len(uid), _p(uid), _p(bad), P, _p(ptr), _p(okf), _p(feat), _p(out["best"]),
                                                       _p(out["best_median"]), _p(out["desc"])))
        return out

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class KfdbRequestC(C.Structure):
    _fields_ = [("n", C.c_int32), ("word", C.c_void_p), ("value", C.c_void_p), ("client_mask", C.c_uint64), ("n_exclude", C.c_int32),
                ("exclude_uid", C.c_void_p)]


class KfdbResultC(C.Structure):
    _fields_ = [("cand", C.c_void_p), ("cap", C.c_int32), ("n", C.c_int32), ("n_sharing", C.c_int32), ("max_common", C.c_int32),
                ("min_common", C.c_int32)]


KFDB_CAND_DTYPE = np.dtype([("uid", "<u8"), ("n_words", "<i4"), ("score", "<f4"), ("score_f64", "<f8")])   # ccm_kfdb_candidate
ALL_CLIENTS = (1 << 64) - 1


class KeyFrameDatabase:
    """cslam::KeyFrameDatabase (I/Database.h, S/Database.cpp) with the inverted file and the BowVectors on the device.
    Keyframes are named by uid = mUniqueId and carry client = mId.second; a BowVector is (word ids ascending, values).

      add / erase / clear                          S/Database.cpp:37-70
      DetectLoopCandidates / DetectMapMatchCandidates / DetectRelocalizationCandidates   :72-439
      query / query_batch                          the device half alone: the scored candidates in the reference's order
      score_many                                   mpVoc->score(query, keyframe) for a list of resident keyframes

    `covis` (the Detect* methods) maps a uid to its GetBestCovisibilityKeyFrames(10) (a dict or a callable); it is read for the
    scored candidates only.  `last_result` holds the device result (the scored candidates) of the last Detect* call."""

    def __init__(self, n_words, scoring=0):
        L = lib()
        L.ccm_kfdb_size.restype = C.c_int64
        L.ccm_kfdb_size.argtypes = [C.c_void_p]
        L.ccm_kfdb_destroy.argtypes = [C.c_void_p]
        L.ccm_kfdb_add.argtypes = [C.c_void_p, C.c_uint64, C.c_uint32, C.c_int32, C.c_void_p, C.c_void_p]
        L.ccm_kfdb_erase.argtypes = [C.c_void_p, C.c_uint64]
        L.ccm_kfdb_select.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_float, C.c_void_p, C.c_void_p]
        self._h = C.c_void_p()
        self.n_words, self.scoring = int(n_words), int(scoring)
        _chk(L.ccm_kfdb_create(self.n_words, self.scoring, C.byref(self._h)))
        self.client_of = {}
        self.last_result = None

    def close(self):
        if self._h:
            lib().ccm_kfdb_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def add(self, uid, client, word, value):
        w = np.ascontiguousarray(word, np.uint32); v = np.ascontiguousarray(value, np.float64)
        _chk(lib().ccm_kfdb_add(self._h, int(uid), int(client), len(w), _p(w), _p(v)))
        self.client_of[int(uid)] = int(client)

    def erase(self, uid):
        _chk(lib().ccm_kfdb_erase(self._h, int(uid)))
        self.client_of.pop(int(uid), None)

    def clear(self):
        _chk(lib().ccm_kfdb_clear(self._h))
        self.client_of.clear()

    def size(self):
        return lib().ccm_kfdb_size(self._h)

    def score_many(self, word, value, uids):
        w = np.ascontiguousarray(word, np.uint32); v = np.ascontiguousarray(value, np.float64); u = np.ascontiguousarray(uids, np.uint64)
        out = np.zeros(len(u))
        _chk(lib().ccm_kfdb_score_many(self._h, len(w), _p(w), _p(v), len(u), _p(u), _p(out)))
        return out

    @staticmethod
    def request(word, value, client_mask=ALL_CLIENTS, exclude=()):
        """one query: (word, value) = its BowVector; keyframes of clients outside client_mask and the uids in exclude are invisible"""
        keep = dict(w=np.ascontiguousarray(word, np.uint32), v=np.ascontiguousarray(value, np.float64),
                    x=np.ascontiguousarray(list(exclude) if not isinstance(exclude, np.ndarray) else exclude, np.uint64))
        return KfdbRequestC(len(keep["w"]), _p(keep["w"]), _p(keep["v"]), int(client_mask) & ALL_CLIENTS, len(keep["x"]), _p(keep["x"])), keep

    def query_batch(self, requests):
        """requests: list of request() tuples -> list of dict(cand = KFDB_CAND_DTYPE array, n_sharing, max_common, min_common)"""
        nq = len(requests)
        cap = max(1, self.size())
        Q = (KfdbRequestC * max(nq, 1))(*[r[0] for r in requests])
        cands = [np.zeros(cap, KFDB_CAND_DTYPE) for _ in range(nq)]
        R = (KfdbResultC * max(nq, 1))(*[KfdbResultC(_p(c), cap, 0, 0, 0, 0) for c in cands])
        _chk(lib().ccm_kfdb_query_batch(self._h, Q, nq, R))
        return [dict(cand=cands[b][:R[b].n].copy(), n_sharing=R[b].n_sharing, max_common=R[b].max_common, min_common=R[b].min_common,
                     _res=R[b]) for b in range(nq)]

    def query(self, word, value, client_mask=ALL_CLIENTS, exclude=()):
        return self.query_batch([self.request(word, value, client_mask, exclude)])[0]

    @staticmethod
    def select(result, covis, reloc=False, min_score=0.0):
        """ccm_kfdb_select (host only): covisibility accumulation and retain over a query result -> uids of the returned vector<kfptr>"""
        cand = np.ascontiguousarray(result["cand"])
        get = covis if callable(covis) else (lambda u: covis.get(int(u), ()))
        lists = [np.asarray(get(u), np.uint64) for u in cand["uid"]]
        ptr = np.concatenate([[0], np.cumsum([len(x) for x in lists])]).astype(np.int32)
        cu = np.concatenate(lists).astype(np.uint64) if lists else np.zeros(0, np.uint64)
        res = KfdbResultC(_p(cand), len(cand), len(cand), result["n_sharing"], result["max_common"], result["min_common"])
        out = np.zeros(max(1, len(cand)), np.uint64); n = C.c_int32()
        _chk(lib().ccm_kfdb_select(C.byref(res), _p(ptr), _p(cu), int(bool(reloc)), C.c_float(min_score), _p(out), C.byref(n)))
        return out[:n.value].copy()

    def _mask(self, clients):
        m = 0
        for c in clients:
            m |= 1 << int(c)
        return m

    def DetectLoopCandidates(self, q_uid, word, value, min_score, connected, in_map, covis):
        """pKF = (q_uid, BowVector); connected = GetConnectedKeyFrames(); in_map = the uids of GetMapptr()->GetMmpKeyFrames()"""
        in_map = set(int(u) for u in in_map)
        clients = {self.client_of[u] for u in in_map if u in self.client_of}
        hide = {int(q_uid)} | {int(u) for u in connected}
        hide |= {u for u, c in self.client_of.items() if c in clients and u not in in_map}   # in the database, not in the map
        r = self.last_result = self.query(word, value, self._mask(clients), sorted(hide))
        return self.select(r, covis, False, min_score)

    def DetectMapMatchCandidates(self, word, value, min_score, assoc_clients, covis):
        """pMap->msuAssClients = assoc_clients"""
        r = self.last_result = self.query(word, value, ALL_CLIENTS & ~self._mask(assoc_clients))
        return self.select(r, covis, False, min_score)

    def DetectRelocalizationCandidates(self, word, value, covis):
        r = self.last_result = self.query(word, value)
        return self.select(r, covis, True)

    def set_timing(self, on=True):
        _chk(lib().ccm_kfdb_set_timing(self._h, int(bool(on))))

    def timing(self):
        a = C.c_double(); b = C.c_double(); n = C.c_int64()
        _chk(lib().ccm_kfdb_get_timing(self._h, C.byref(a), C.byref(b), C.byref(n)))
        return a.value, b.value, n.value

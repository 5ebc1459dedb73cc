// ORBmatcher_proj_shim.cpp — the projection-guided overloads of cslam::ORBmatcher on top of libccm_b200.so
// (SURVEY.md §8(f) rank 3).  Replaces, in cslam/src/ORBmatcher.cpp:
//   SearchByProjection(Frame&, const vector<mpptr>&, th)                        :71-148
//   SearchForInitialization(F1, F2, vbPrevMatched, vnMatches12, windowSize)     :448-563
//   SearchByProjection(kfptr, cv::Mat Scw, vpPoints, vpMatched, th)             :308-446
//   Fuse(kfptr, const vector<mpptr>&, th)                                       :854-993
//   Fuse(kfptr, cv::Mat Scw, vpPoints, th, vpReplacePoint)                      :995-1122
//   SearchBySim3(pKF1, pKF2, vpMatches12, s12, R12, t12, th)                    :1124-1348
//   SearchByProjection(Frame& CurrentFrame, const Frame& LastFrame, th)         :1350-1476
//   SearchByProjection(Frame& CurrentFrame, kfptr, sAlreadyFound, th, ORBdist)  :1478-1605
// cslam/include/cslam/ORBmatcher.h stays byte-identical.  Compiled against that header and run side by side with the
// reference's ORBmatcher.cpp on stand-in Frame / KeyFrame / MapPoint objects by tests/test_shim_dropin.py.
//
// Every overload has the same three parts.  PRELUDE: the reference's per-point gates up to the GetFeaturesInArea call
// (bad / already-found tests, camera projection, image bounds, scale-invariance distance, viewing angle, PredictScale).  It is
// written with the same cv::Mat expressions the reference uses, so its float rounding is OpenCV's, and it produces one
// (valid, u, v, radius, level) record per point.  SEARCH: one library call (device distances + selection in the reference's
// visiting order).  EPILOGUE: the map surgery, in point order, on the indices that came back.
#include <cslam/ORBmatcher.h>

#include "Sim3Split_shim.h"
#include "ccm_b200.h"

namespace cslam {

namespace {

// the smart-pointer aliases are class-scoped in the reference (cslam/ORBmatcher.h:91-93); the helpers below are free functions
typedef ORBmatcher::kfptr kfptr;
typedef ORBmatcher::mpptr mpptr;

// image side of a search: keypoints + lookup-grid geometry of a Frame or a KeyFrame
template <class ImageLike>
struct GridView {
  std::vector<float> xy, angle;
  std::vector<int32_t> octave;
  ccm_feature_grid g;
  GridView(const ImageLike& im, const std::vector<cv::KeyPoint>& keysUn, const cv::Mat& desc, int cols, int rows, float minx, float miny,
           float maxx, float maxy, float winv, float hinv) {
    const int n = (int)keysUn.size();
    xy.resize(2 * n); angle.resize(n); octave.resize(n);
    for (int i = 0; i < n; i++) { xy[2 * i] = keysUn[i].pt.x; xy[2 * i + 1] = keysUn[i].pt.y; angle[i] = keysUn[i].angle; octave[i] = keysUn[i].octave; }
    g = ccm_feature_grid{n, desc.ptr<uchar>(0), xy.data(), octave.data(), angle.data(), minx, miny, maxx, maxy, winv, hinv, cols, rows};
    (void)im;
  }
};
GridView<Frame> grid_of(const Frame& F) {
  return GridView<Frame>(F, F.mvKeysUn, F.mDescriptors, FRAME_GRID_COLS, FRAME_GRID_ROWS, Frame::mnMinX, Frame::mnMinY, Frame::mnMaxX,
                         Frame::mnMaxY, Frame::mfGridElementWidthInv, Frame::mfGridElementHeightInv);
}
GridView<KeyFrame> grid_of(const kfptr& k) {
  return GridView<KeyFrame>(*k, k->mvKeysUn, k->mDescriptors, k->mnGridCols, k->mnGridRows, (float)k->mnMinX, (float)k->mnMinY,
                            (float)k->mnMaxX, (float)k->mnMaxY, k->mfGridElementWidthInv, k->mfGridElementHeightInv);
}

// query side: one record per candidate point
struct Queries {
  std::vector<uint8_t> valid, desc;
  std::vector<float> uv, radius, angle;
  std::vector<int32_t> level;
  explicit Queries(size_t m) : valid(m, 0), desc(32 * m, 0), uv(2 * m, 0.f), radius(m, 0.f), angle(m, 0.f), level(m, 0) {}
  void set(size_t i, float u, float v, float r, int lvl, const cv::Mat& d, float ang = 0.f) {
    valid[i] = 1; uv[2 * i] = u; uv[2 * i + 1] = v; radius[i] = r; level[i] = lvl; angle[i] = ang;
    memcpy(&desc[32 * i], d.ptr<uchar>(0), 32);
  }
  ccm_proj_queries c() const {
    return ccm_proj_queries{(int32_t)valid.size(), valid.data(), uv.data(), radius.data(), level.data(), desc.data(), angle.data()};
  }
};

inline void must(int rc) { if (rc != CCM_OK) throw estd::infrastructure_ex(); }

// pinhole projection of a camera-frame point; false when behind the camera (the reference's "Depth must be positive")
inline bool project(const cv::Mat& Pc, float fx, float fy, float cx, float cy, float& u, float& v) {
  if (Pc.at<float>(2) < 0.0f) return false;
  const float invz = 1.0f / Pc.at<float>(2);
  u = fx * (Pc.at<float>(0) * invz) + cx;
  v = fy * (Pc.at<float>(1) * invz) + cy;
  return true;
}

// the gates shared by SearchByProjection(kf,Scw), both Fuse overloads: projection into the keyframe, image bounds, distance
// range, 60-degree viewing cone, predicted level (S/ORBmatcher.cpp:344-381, :884-921, :1030-1069)
inline bool gate_into_kf(const kfptr& pKF, const mpptr& pMP, const cv::Mat& Rcw, const cv::Mat& tcw, const cv::Mat& Ow, float th, Queries& q, size_t i) {
  cv::Mat p3Dw = pMP->GetWorldPos();
  cv::Mat p3Dc = Rcw * p3Dw + tcw;
  float u, v;
  if (!project(p3Dc, pKF->fx, pKF->fy, pKF->cx, pKF->cy, u, v)) return false;
  if (!pKF->IsInImage(u, v)) return false;
  const float maxDistance = pMP->GetMaxDistanceInvariance(), minDistance = pMP->GetMinDistanceInvariance();
  cv::Mat PO = p3Dw - Ow;
  const float dist3D = cv::norm(PO);
  if (dist3D < minDistance || dist3D > maxDistance) return false;
  cv::Mat Pn = pMP->GetNormal();
  if (PO.dot(Pn) < 0.5 * dist3D) return false;
  const int lvl = pMP->PredictScale(dist3D, pKF);
  q.set(i, u, v, th * pKF->mvScaleFactors[lvl], lvl, pMP->GetDescriptor());
  return true;
}

}  // namespace

// ---- monocular initialisation -------------------------------------------------------------------------------------------
int ORBmatcher::SearchForInitialization(Frame& F1, Frame& F2, std::vector<cv::Point2f>& vbPrevMatched, std::vector<int>& vnMatches12,
                                        int windowSize) {                                                 // :448-563
  const size_t n1 = F1.mvKeysUn.size();
  Queries q(n1);
  for (size_t i1 = 0; i1 < n1; i1++)   // the library skips octaves > 0 itself (:466-468)
    q.set(i1, vbPrevMatched[i1].x, vbPrevMatched[i1].y, (float)windowSize, F1.mvKeysUn[i1].octave, F1.mDescriptors.row((int)i1),
          F1.mvKeysUn[i1].angle);
  auto G2 = grid_of(F2);
  ccm_proj_queries cq = q.c();
  std::vector<int32_t> m12(n1);
  int32_t n = 0;
  must(ccm_search_for_initialization(&G2.g, &cq, mfNNratio, mbCheckOrientation, m12.data(), &n));
  vnMatches12.assign(m12.begin(), m12.end());
  for (size_t i1 = 0; i1 < n1; i1++)
    if (vnMatches12[i1] >= 0) vbPrevMatched[i1] = F2.mvKeysUn[vnMatches12[i1]].pt;                      // :557-560
  return n;
}

// ---- tracking the local map ---------------------------------------------------------------------------------------------
int ORBmatcher::SearchByProjection(Frame& F, const std::vector<mpptr>& vpMapPoints, const float th) {   // :71-148
  const bool bFactor = th != 1.0;
  Queries q(vpMapPoints.size());
  std::vector<uint8_t> has_obs(vpMapPoints.size(), 0), blocked(F.N, 0);
  for (size_t i = 0; i < vpMapPoints.size(); i++) {
    const mpptr& pMP = vpMapPoints[i];
    if (!pMP->mbTrackInView || pMP->isBad()) continue;
    float r = RadiusByViewingCos(pMP->mTrackViewCos);
    if (bFactor) r *= th;
    q.set(i, pMP->mTrackProjX, pMP->mTrackProjY, r * F.mvScaleFactors[pMP->mnTrackScaleLevel], pMP->mnTrackScaleLevel, pMP->GetDescriptor());
    has_obs[i] = pMP->Observations() > 0;
  }
  for (int j = 0; j < F.N; j++) blocked[j] = F.mvpMapPoints[j] && F.mvpMapPoints[j]->Observations() > 0;
  auto G = grid_of(F);
  ccm_proj_queries cq = q.c();
  std::vector<int32_t> match(F.N);
  int32_t n = 0;
  must(ccm_search_by_projection_track(&G.g, &cq, has_obs.data(), blocked.data(), mfNNratio, match.data(), &n));
  for (int j = 0; j < F.N; j++) if (match[j] >= 0) F.mvpMapPoints[j] = vpMapPoints[match[j]];
  return n;
}

// ---- frame to frame (motion model) and relocalisation ------------------------------------------------------------------
int ORBmatcher::SearchByProjection(Frame& CurrentFrame, const Frame& LastFrame, const float th) {       // :1350-1476
  const cv::Mat Rcw = CurrentFrame.mTcw.rowRange(0, 3).colRange(0, 3), tcw = CurrentFrame.mTcw.rowRange(0, 3).col(3);
  Queries q(LastFrame.N);
  std::vector<uint8_t> has_obs(LastFrame.N, 0), blocked(CurrentFrame.N, 0);
  for (int i = 0; i < LastFrame.N; i++) {
    const mpptr& pMP = LastFrame.mvpMapPoints[i];
    if (!pMP || LastFrame.mvbOutlier[i]) continue;
    cv::Mat x3Dc = Rcw * pMP->GetWorldPos() + tcw;
    const float invzc = 1.0 / x3Dc.at<float>(2);
    if (invzc < 0) continue;
    const float u = CurrentFrame.fx * x3Dc.at<float>(0) * invzc + CurrentFrame.cx;
    const float v = CurrentFrame.fy * x3Dc.at<float>(1) * invzc + CurrentFrame.cy;
    if (u < CurrentFrame.mnMinX || u > CurrentFrame.mnMaxX || v < CurrentFrame.mnMinY || v > CurrentFrame.mnMaxY) continue;
    const int oct = LastFrame.mvKeys[i].octave;
    q.set(i, u, v, th * CurrentFrame.mvScaleFactors[oct], oct, pMP->GetDescriptor(), LastFrame.mvKeysUn[i].angle);
    has_obs[i] = pMP->Observations() > 0;
  }
  for (int j = 0; j < CurrentFrame.N; j++) blocked[j] = CurrentFrame.mvpMapPoints[j] && CurrentFrame.mvpMapPoints[j]->Observations() > 0;
  auto G = grid_of(CurrentFrame);
  ccm_proj_queries cq = q.c();
  std::vector<int32_t> match(CurrentFrame.N);
  int32_t n = 0;
  must(ccm_search_by_projection_frame(&G.g, &cq, has_obs.data(), blocked.data(), /*reloc=*/0, TH_HIGH, mbCheckOrientation, match.data(), &n));
  for (int j = 0; j < CurrentFrame.N; j++) {
    if (match[j] >= 0) CurrentFrame.mvpMapPoints[j] = LastFrame.mvpMapPoints[match[j]];
    else if (match[j] == -2) CurrentFrame.mvpMapPoints[j] = nullptr;           // assigned, then dropped by the rotation histogram
  }
  return n;
}

int ORBmatcher::SearchByProjection(Frame& CurrentFrame, kfptr pKF, const std::set<mpptr>& sAlreadyFound, const float th, const int ORBdist) {  // :1478-1605
  const cv::Mat Rcw = CurrentFrame.mTcw.rowRange(0, 3).colRange(0, 3), tcw = CurrentFrame.mTcw.rowRange(0, 3).col(3);
  const cv::Mat Ow = -Rcw.t() * tcw;
  const std::vector<mpptr> vpMPs = pKF->GetMapPointMatches();
  Queries q(vpMPs.size());
  std::vector<uint8_t> blocked(CurrentFrame.N, 0);
  for (size_t i = 0; i < vpMPs.size(); i++) {
    const mpptr& pMP = vpMPs[i];
    if (!pMP || pMP->isBad() || sAlreadyFound.count(pMP)) continue;
    cv::Mat x3Dw = pMP->GetWorldPos();
    cv::Mat x3Dc = Rcw * x3Dw + tcw;
    const float invzc = 1.0 / x3Dc.at<float>(2);
    const float u = CurrentFrame.fx * x3Dc.at<float>(0) * invzc + CurrentFrame.cx;
    const float v = CurrentFrame.fy * x3Dc.at<float>(1) * invzc + CurrentFrame.cy;
    if (u < CurrentFrame.mnMinX || u > CurrentFrame.mnMaxX || v < CurrentFrame.mnMinY || v > CurrentFrame.mnMaxY) continue;
    cv::Mat PO = x3Dw - Ow;
    const float dist3D = cv::norm(PO);
    if (dist3D < pMP->GetMinDistanceInvariance() || dist3D > pMP->GetMaxDistanceInvariance()) continue;
    const int lvl = pMP->PredictScale(dist3D, CurrentFrame.shared_from_this());
    q.set(i, u, v, th * CurrentFrame.mvScaleFactors[lvl], lvl, pMP->GetDescriptor(), pKF->mvKeysUn[i].angle);
  }
  for (int j = 0; j < CurrentFrame.N; j++) blocked[j] = CurrentFrame.mvpMapPoints[j] ? 1 : 0;
  auto G = grid_of(CurrentFrame);
  ccm_proj_queries cq = q.c();
  std::vector<int32_t> match(CurrentFrame.N);
  int32_t n = 0;
  must(ccm_search_by_projection_frame(&G.g, &cq, nullptr, blocked.data(), /*reloc=*/1, ORBdist, mbCheckOrientation, match.data(), &n));
  for (int j = 0; j < CurrentFrame.N; j++) {
    if (match[j] >= 0) CurrentFrame.mvpMapPoints[j] = vpMPs[match[j]];
    else if (match[j] == -2) CurrentFrame.mvpMapPoints[j] = nullptr;
  }
  return n;
}

// ---- loop closing / map merging ----------------------------------------------------------------------------------------
int ORBmatcher::SearchByProjection(kfptr pKF, cv::Mat Scw, const std::vector<mpptr>& vpPoints, std::vector<mpptr>& vpMatched, int th) {   // :308-446
  const Sim3Split s = split_sim3(Scw);
  std::set<mpptr> spAlreadyFound(vpMatched.begin(), vpMatched.end());
  spAlreadyFound.erase(nullptr);
  Queries q(vpPoints.size());
  std::vector<int32_t> existing(vpPoints.size(), -1);
  for (size_t i = 0; i < vpPoints.size(); i++) {
    const mpptr& pMP = vpPoints[i];
    if (pMP->isBad() || spAlreadyFound.count(pMP)) continue;
    if (gate_into_kf(pKF, pMP, s.Rcw, s.tcw, s.Ow, (float)th, q, i)) existing[i] = pMP->GetIndexInKeyFrame(pKF);
  }
  std::vector<uint8_t> matched(vpMatched.size());
  for (size_t j = 0; j < vpMatched.size(); j++) matched[j] = vpMatched[j] ? 1 : 0;
  auto G = grid_of(pKF);
  ccm_proj_queries cq = q.c();
  std::vector<int32_t> best(vpPoints.size()), mof(G.g.n);
  int32_t n = 0;
  must(ccm_search_by_projection_sim3(&G.g, &cq, matched.data(), existing.data(), best.data(), mof.data(), &n));
  for (size_t i = 0; i < vpPoints.size(); i++) {
    if (best[i] < 0) continue;
    // :418-432.  dist_newplace is the distance to the very keypoint just chosen, so bDoNotReplace never fires: always remapped.
    // The slot is asked for again here: an earlier entry of vpPoints may have been the same point and moved it.
    if (existing[i] != -1) pKF->RemapMapPointMatch(vpPoints[i], vpPoints[i]->GetIndexInKeyFrame(pKF), best[i]);
    else vpMatched[best[i]] = vpPoints[i];
  }
  return n;
}

int ORBmatcher::Fuse(kfptr pKF, const std::vector<mpptr>& vpMapPoints, const float th) {                // :854-993
  const cv::Mat Rcw = pKF->GetRotation(), tcw = pKF->GetTranslation(), Ow = pKF->GetCameraCenter();
  Queries q(vpMapPoints.size());
  for (size_t i = 0; i < vpMapPoints.size(); i++) {
    const mpptr& pMP = vpMapPoints[i];
    if (!pMP || pMP->isBad() || pMP->IsInKeyFrame(pKF) || pMP->mbDoNotReplace) continue;
    gate_into_kf(pKF, pMP, Rcw, tcw, Ow, th, q, i);
  }
  auto G = grid_of(pKF);
  ccm_proj_queries cq = q.c();
  std::vector<int32_t> best(vpMapPoints.size());
  int32_t found = 0;
  must(ccm_fuse_search(&G.g, &cq, pKF->mvInvLevelSigma2.data(), (int)pKF->mvInvLevelSigma2.size(), best.data(), &found));
  int nFused = 0;
  for (size_t i = 0; i < vpMapPoints.size(); i++) {
    if (best[i] < 0) continue;
    const mpptr& pMP = vpMapPoints[i];
    if (pMP->isBad() || pMP->IsInKeyFrame(pKF)) continue;   // a duplicate entry of the list that an earlier iteration already fused
    mpptr pMPinKF = pKF->GetMapPoint(best[i]);
    if (pMPinKF) {
      if (!pMPinKF->isBad() && !pMPinKF->mbDoNotReplace) {
        if (pMPinKF->Observations() > pMP->Observations()) pMP->Replace(pMPinKF);
        else pMPinKF->Replace(pMP);
      }
    } else {
      pMP->AddObservation(pKF, best[i]);
      pKF->AddMapPoint(pMP, best[i]);
    }
    nFused++;
  }
  return nFused;
}

int ORBmatcher::Fuse(kfptr pKF, cv::Mat Scw, const std::vector<mpptr>& vpPoints, float th, std::vector<mpptr>& vpReplacePoint) {   // :995-1122
  const Sim3Split s = split_sim3(Scw);
  const std::set<mpptr> spAlreadyFound = pKF->GetMapPoints();
  Queries q(vpPoints.size());
  for (size_t i = 0; i < vpPoints.size(); i++) {
    const mpptr& pMP = vpPoints[i];
    if (pMP->isBad() || spAlreadyFound.count(pMP)) continue;
    gate_into_kf(pKF, pMP, s.Rcw, s.tcw, s.Ow, th, q, i);
  }
  auto G = grid_of(pKF);
  ccm_proj_queries cq = q.c();
  std::vector<int32_t> best(vpPoints.size());
  int32_t found = 0;
  must(ccm_fuse_search(&G.g, &cq, nullptr, 0, best.data(), &found));
  int nFused = 0;
  for (size_t i = 0; i < vpPoints.size(); i++) {
    if (best[i] < 0) continue;
    mpptr pMPinKF = pKF->GetMapPoint(best[i]);
    if (pMPinKF) {
      if (!pMPinKF->isBad()) vpReplacePoint[i] = pMPinKF;
    } else {
      vpPoints[i]->AddObservation(pKF, best[i]);
      pKF->AddMapPoint(vpPoints[i], best[i]);
    }
    nFused++;
  }
  return nFused;
}

int ORBmatcher::SearchBySim3(kfptr pKF1, kfptr pKF2, std::vector<mpptr>& vpMatches12, const float& s12, const cv::Mat& R12, const cv::Mat& t12,
                             const float th) {                                                          // :1124-1348
  const cv::Mat R1w = pKF1->GetRotation(), t1w = pKF1->GetTranslation(), R2w = pKF2->GetRotation(), t2w = pKF2->GetTranslation();
  const cv::Mat sR12 = s12 * R12, sR21 = (1.0 / s12) * R12.t(), t21 = -sR21 * t12;
  const std::vector<mpptr> vpMapPoints1 = pKF1->GetMapPointMatches(), vpMapPoints2 = pKF2->GetMapPointMatches();
  const int N1 = (int)vpMapPoints1.size(), N2 = (int)vpMapPoints2.size();
  std::vector<bool> done1(N1, false), done2(N2, false);
  for (int i = 0; i < N1; i++) {
    const mpptr& pMP = vpMatches12[i];
    if (!pMP) continue;
    done1[i] = true;
    const int idx2 = pMP->GetIndexInKeyFrame(pKF2);
    if (idx2 >= 0 && idx2 < N2) done2[idx2] = true;
  }
  // one direction: points of `src` carried into the camera of `dst` by (Rsw, tsw) then (sR, t)
  auto carry = [&](const std::vector<mpptr>& pts, const std::vector<bool>& done, const cv::Mat& Rsw, const cv::Mat& tsw, const cv::Mat& sR,
                   const cv::Mat& t, const kfptr& dst, Queries& q) {
    for (size_t i = 0; i < pts.size(); i++) {
      const mpptr& pMP = pts[i];
      if (!pMP || done[i] || pMP->isBad()) continue;
      cv::Mat Pdst = sR * (Rsw * pMP->GetWorldPos() + tsw) + t;
      float u, v;
      if (!project(Pdst, pKF1->fx, pKF1->fy, pKF1->cx, pKF1->cy, u, v)) continue;     // the reference uses pKF1's intrinsics both ways
      if (!dst->IsInImage(u, v)) continue;
      const float dist3D = cv::norm(Pdst);
      if (dist3D < pMP->GetMinDistanceInvariance() || dist3D > pMP->GetMaxDistanceInvariance()) continue;
      const int lvl = pMP->PredictScale(dist3D, dst);
      q.set(i, u, v, th * dst->mvScaleFactors[lvl], lvl, pMP->GetDescriptor());
    }
  };
  Queries q12(N1), q21(N2);
  carry(vpMapPoints1, done1, R1w, t1w, sR21, t21, pKF2, q12);
  carry(vpMapPoints2, done2, R2w, t2w, sR12, t12, pKF1, q21);
  auto G1 = grid_of(pKF1), G2 = grid_of(pKF2);
  ccm_proj_queries c12 = q12.c(), c21 = q21.c();
  std::vector<int32_t> m12(N1);
  int32_t nFound = 0;
  must(ccm_search_by_sim3(&G1.g, &G2.g, &c12, &c21, m12.data(), &nFound));
  for (int i1 = 0; i1 < N1; i1++) if (m12[i1] >= 0) vpMatches12[i1] = vpMapPoints2[m12[i1]];
  return nFound;
}

}  // namespace cslam

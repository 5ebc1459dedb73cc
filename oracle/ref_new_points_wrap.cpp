// ref_new_points_wrap.cpp — TEST INFRASTRUCTURE: shim/NewMapPoints_shim.cpp next to a literal restatement of the body it replaces,
// LocalMapping::CreateNewMapPoints (S/Mapping.cpp:284-469), ComputeF12 and SkewSymmetricMatrix (:549-573), over the stand-in
// LocalMapping / KeyFrame / MapPoint / Map of ref_stub_np/.  Nothing is copied from the reference tree: each block cites the lines it
// restates.  ORBmatcher::SearchForTriangulation, which the body calls, is the oracle's reference-pinned orc_match_triangulation behind a
// stand-in ORBmatcher that forms the epipole as S/ORBmatcher.cpp:707-714 does.  Where OpenCV's MatExpr machinery evaluates an
// expression differently from plain operators (`Mat / double` is convertTo), the restatement calls the step explicitly
// (ref_stub_mp/opencv_matexpr.h).
//
// C interface (oracle/pynp.py): np_scene_create builds a current keyframe and its neighbours from flat arrays; np_run runs the literal
// body (mode 0) or the shim member (mode 1) with CheckNewKeyFrames() forced true at a given poll; np_members dumps what the body
// changed: mvpMapPoints of every keyframe as indices into the map's point list, each point's position, observations, reference
// keyframe and call log, and the recent-points list.
#include <cstdint>
#include <cstring>
#include <vector>

#include <cslam/Mapping.h>
#include <cslam/estd.h>
#include <opencv_matexpr.h>

#include "../shim/NewMapPoints_shim.h"
#include "ccm_b200.h"

extern "C" int orc_match_triangulation(const ccm_tri_view* v1, const ccm_tri_view* v2, const float F12[9], float ex, float ey,
                                       const float* level_sigma2, const float* scale_factors, int check_ori, int* pairs);

namespace cslam {

typedef LocalMapping::kfptr kfptr;
typedef LocalMapping::mpptr mpptr;

// S/Mapping.cpp:549-566
cv::Mat LocalMapping::ComputeF12(kfptr& pKF1, kfptr& pKF2) {
  cv::Mat R1w = pKF1->GetRotation();
  cv::Mat t1w = pKF1->GetTranslation();
  cv::Mat R2w = pKF2->GetRotation();
  cv::Mat t2w = pKF2->GetTranslation();
  cv::Mat R12 = R1w * R2w.t();
  cv::Mat t12 = -R1w * R2w.t() * t2w + t1w;
  cv::Mat t12x = SkewSymmetricMatrix(t12);
  const cv::Mat& K1 = pKF1->mK;
  const cv::Mat& K2 = pKF2->mK;
  return cv::inv3(K1.t()) * t12x * R12 * cv::inv3(K2);
}

// S/Mapping.cpp:568-573
cv::Mat LocalMapping::SkewSymmetricMatrix(const cv::Mat& v) {
  cv::Mat m(3, 3, CV_32F);
  m.at<float>(0, 0) = 0; m.at<float>(0, 1) = -v.at<float>(2); m.at<float>(0, 2) = v.at<float>(1);
  m.at<float>(1, 0) = v.at<float>(2); m.at<float>(1, 1) = 0; m.at<float>(1, 2) = -v.at<float>(0);
  m.at<float>(2, 0) = -v.at<float>(1); m.at<float>(2, 1) = v.at<float>(0); m.at<float>(2, 2) = 0;
  return m;
}

namespace {

// ORBmatcher as CreateNewMapPoints uses it: the epipole of S/ORBmatcher.cpp:707-714, then the pinned matcher of the oracle
struct ORBmatcher {
  bool mbCheckOrientation;
  ORBmatcher(float, bool checkOri) : mbCheckOrientation(checkOri) {}
  struct Flat {
    std::vector<uint8_t> has; std::vector<float> xy, ang; std::vector<int32_t> oct, ptr; std::vector<uint32_t> id, feat;
    ccm_feature_vector fv; ccm_tri_view v;
    explicit Flat(const kfptr& p) {
      for (int i = 0; i < p->N; i++) {
        has.push_back(p->GetMapPoint(i) ? 1 : 0);
        xy.push_back(p->mvKeysUn[i].pt.x); xy.push_back(p->mvKeysUn[i].pt.y); ang.push_back(p->mvKeysUn[i].angle); oct.push_back(p->mvKeysUn[i].octave);
      }
      ptr.push_back(0);
      for (auto& e : p->mFeatVec) { id.push_back(e.first); feat.insert(feat.end(), e.second.begin(), e.second.end()); ptr.push_back((int32_t)feat.size()); }
      fv.n_nodes = (int32_t)id.size(); fv.node_id = id.data(); fv.node_ptr = ptr.data(); fv.feat = feat.data();
      v.desc = p->mDescriptors.ptr(); v.n = p->N; v.has_mp = has.data(); v.kp_xy = xy.data(); v.octave = oct.data(); v.angle = ang.data();
      v.fv = &fv; v.fx = p->fx; v.fy = p->fy; v.cx = p->cx; v.cy = p->cy;
    }
  };
  int SearchForTriangulation(kfptr pKF1, kfptr pKF2, cv::Mat F12, std::vector<std::pair<size_t, size_t> >& vMatchedPairs) {
    cv::Mat Cw = pKF1->GetCameraCenter();
    cv::Mat R2w = pKF2->GetRotation();
    cv::Mat t2w = pKF2->GetTranslation();
    cv::Mat C2 = R2w * Cw + t2w;
    const float invz = 1.0f / C2.at<float>(2);
    const float ex = pKF2->fx * C2.at<float>(0) * invz + pKF2->cx;
    const float ey = pKF2->fy * C2.at<float>(1) * invz + pKF2->cy;
    Flat a(pKF1), b(pKF2);
    float F[9];
    for (int r = 0; r < 3; r++) for (int c = 0; c < 3; c++) F[3 * r + c] = F12.at<float>(r, c);
    std::vector<int> pairs(2 * (size_t)pKF1->N + 2);
    const int n = orc_match_triangulation(&a.v, &b.v, F, ex, ey, pKF2->mvLevelSigma2.data(), pKF2->mvScaleFactors.data(), mbCheckOrientation, pairs.data());
    vMatchedPairs.clear();
    for (int k = 0; k < n; k++) vMatchedPairs.push_back(std::make_pair((size_t)pairs[2 * k], (size_t)pairs[2 * k + 1]));
    return n;
  }
};

cv::Mat vec3(float a, float b, float c) {
  cv::Mat m(3, 1, CV_32F);
  m.at<float>(0) = a; m.at<float>(1) = b; m.at<float>(2) = c;
  return m;
}

// S/Mapping.cpp:284-469, statement for statement; `self` is `this`
void literal_CreateNewMapPoints(LocalMapping& self) {
  kfptr& mpCurrentKeyFrame = self.mpCurrentKeyFrame;
  int nn = 20;                                                                                   // :287-288
  const std::vector<kfptr> vpNeighKFs = mpCurrentKeyFrame->GetBestCovisibilityKeyFrames(nn);
  ORBmatcher matcher(0.6, false);                                                                // :290
  cv::Mat Rcw1 = mpCurrentKeyFrame->GetRotation();                                               // :292-298
  cv::Mat Rwc1 = Rcw1.t();
  cv::Mat tcw1 = mpCurrentKeyFrame->GetTranslation();
  cv::Mat Tcw1(3, 4, CV_32F);
  { cv::Mat d = Tcw1.colRange(0, 3); Rcw1.copyTo(d); }
  { cv::Mat d = Tcw1.col(3); tcw1.copyTo(d); }
  cv::Mat Ow1 = mpCurrentKeyFrame->GetCameraCenter();
  const float& fx1 = mpCurrentKeyFrame->fx;                                                      // :300-305
  const float& fy1 = mpCurrentKeyFrame->fy;
  const float& cx1 = mpCurrentKeyFrame->cx;
  const float& cy1 = mpCurrentKeyFrame->cy;
  const float& invfx1 = mpCurrentKeyFrame->invfx;
  const float& invfy1 = mpCurrentKeyFrame->invfy;
  const float ratioFactor = 1.5f * mpCurrentKeyFrame->mfScaleFactor;                             // :307
  int nnew = 0;
  for (size_t i = 0; i < vpNeighKFs.size(); i++) {                                               // :312
    if (i > 0 && self.CheckNewKeyFrames()) return;                                               // :314-315
    kfptr pKF2 = vpNeighKFs[i];
    cv::Mat Ow2 = pKF2->GetCameraCenter();                                                       // :320-328
    cv::Mat vBaseline = Ow2 - Ow1;
    const float baseline = cv::norm(vBaseline);
    const float medianDepthKF2 = pKF2->ComputeSceneMedianDepth(2);
    const float ratioBaselineDepth = baseline / medianDepthKF2;
    if (ratioBaselineDepth < 0.01) continue;
    cv::Mat F12 = self.ComputeF12(mpCurrentKeyFrame, pKF2);                                      // :331
    std::vector<std::pair<size_t, size_t> > vMatchedIndices;                                     // :334-335
    matcher.SearchForTriangulation(mpCurrentKeyFrame, pKF2, F12, vMatchedIndices);
    cv::Mat Rcw2 = pKF2->GetRotation();                                                          // :337-342
    cv::Mat Rwc2 = Rcw2.t();
    cv::Mat tcw2 = pKF2->GetTranslation();
    cv::Mat Tcw2(3, 4, CV_32F);
    { cv::Mat d = Tcw2.colRange(0, 3); Rcw2.copyTo(d); }
    { cv::Mat d = Tcw2.col(3); tcw2.copyTo(d); }
    const float& fx2 = pKF2->fx;                                                                 // :344-349
    const float& fy2 = pKF2->fy;
    const float& cx2 = pKF2->cx;
    const float& cy2 = pKF2->cy;
    const float& invfx2 = pKF2->invfx;
    const float& invfy2 = pKF2->invfy;
    const int nmatches = vMatchedIndices.size();                                                 // :352
    for (int ikp = 0; ikp < nmatches; ikp++) {
      const int idx1 = vMatchedIndices[ikp].first;
      const int idx2 = vMatchedIndices[ikp].second;
      const cv::KeyPoint& kp1 = mpCurrentKeyFrame->mvKeysUn[idx1];
      const cv::KeyPoint& kp2 = pKF2->mvKeysUn[idx2];
      cv::Mat xn1 = vec3((kp1.pt.x - cx1) * invfx1, (kp1.pt.y - cy1) * invfy1, 1.0);               // :363-364
      cv::Mat xn2 = vec3((kp2.pt.x - cx2) * invfx2, (kp2.pt.y - cy2) * invfy2, 1.0);
      cv::Mat ray1 = Rwc1 * xn1;                                                                 // :366-368
      cv::Mat ray2 = Rwc2 * xn2;
      const float cosParallaxRays = ray1.dot(ray2) / (cv::norm(ray1) * cv::norm(ray2));
      float cosParallaxStereo = cosParallaxRays + 1;                                             // :370
      cv::Mat x3D;
      if (cosParallaxRays < cosParallaxStereo && cosParallaxRays > 0 && (cosParallaxRays < 0.9998)) {   // :373
        cv::Mat A(4, 4, CV_32F);                                                                 // :376-380
        { cv::Mat d = A.row(0); (xn1.at<float>(0) * Tcw1.row(2) - Tcw1.row(0)).copyTo(d); }
        { cv::Mat d = A.row(1); (xn1.at<float>(1) * Tcw1.row(2) - Tcw1.row(1)).copyTo(d); }
        { cv::Mat d = A.row(2); (xn2.at<float>(0) * Tcw2.row(2) - Tcw2.row(0)).copyTo(d); }
        { cv::Mat d = A.row(3); (xn2.at<float>(1) * Tcw2.row(2) - Tcw2.row(1)).copyTo(d); }
        cv::Mat w, u, vt;                                                                        // :382-385
        cv::SVD::compute(A, w, u, vt, cv::SVD::MODIFY_A | cv::SVD::FULL_UV);
        x3D = vt.row(3).t();
        if (x3D.at<float>(3) == 0) continue;                                                     // :387-388
        cv::convertTo(x3D.rowRange(0, 3), x3D, CV_32F, 1.0 / x3D.at<float>(3));                   // :391 `Mat / double`
      } else
        continue;                                                                                // :395
      cv::Mat x3Dt = x3D.t();                                                                    // :397
      float z1 = Rcw1.row(2).dot(x3Dt) + tcw1.at<float>(2);                                      // :400-406
      if (z1 <= 0) continue;
      float z2 = Rcw2.row(2).dot(x3Dt) + tcw2.at<float>(2);
      if (z2 <= 0) continue;
      const float& sigmaSquare1 = mpCurrentKeyFrame->mvLevelSigma2[kp1.octave];                  // :409-419
      const float x1 = Rcw1.row(0).dot(x3Dt) + tcw1.at<float>(0);
      const float y1 = Rcw1.row(1).dot(x3Dt) + tcw1.at<float>(1);
      const float invz1 = 1.0 / z1;
      float u1 = fx1 * x1 * invz1 + cx1;
      float v1 = fy1 * y1 * invz1 + cy1;
      float errX1 = u1 - kp1.pt.x;
      float errY1 = v1 - kp1.pt.y;
      if ((errX1 * errX1 + errY1 * errY1) > 5.991 * sigmaSquare1) continue;
      const float sigmaSquare2 = pKF2->mvLevelSigma2[kp2.octave];                                // :422-432
      const float x2 = Rcw2.row(0).dot(x3Dt) + tcw2.at<float>(0);
      const float y2 = Rcw2.row(1).dot(x3Dt) + tcw2.at<float>(1);
      const float invz2 = 1.0 / z2;
      float u2 = fx2 * x2 * invz2 + cx2;
      float v2 = fy2 * y2 * invz2 + cy2;
      float errX2 = u2 - kp2.pt.x;
      float errY2 = v2 - kp2.pt.y;
      if ((errX2 * errX2 + errY2 * errY2) > 5.991 * sigmaSquare2) continue;
      cv::Mat normal1 = x3D - Ow1;                                                               // :435-448
      float dist1 = cv::norm(normal1);
      cv::Mat normal2 = x3D - Ow2;
      float dist2 = cv::norm(normal2);
      if (dist1 == 0 || dist2 == 0) continue;
      const float ratioDist = dist2 / dist1;
      const float ratioOctave = mpCurrentKeyFrame->mvScaleFactors[kp1.octave] / pKF2->mvScaleFactors[kp2.octave];
      if (ratioDist * ratioFactor < ratioOctave || ratioDist > ratioOctave * ratioFactor) continue;
      mpptr pMP{new MapPoint(x3D, mpCurrentKeyFrame, self.mpMap, self.mClientId, self.mpComm, self.mpCC->mSysState, -1)};   // :451
      pMP->AddObservation(mpCurrentKeyFrame, idx1);                                              // :453-466
      pMP->AddObservation(pKF2, idx2);
      mpCurrentKeyFrame->AddMapPoint(pMP, idx1);
      pKF2->AddMapPoint(pMP, idx2);
      pMP->ComputeDistinctiveDescriptors();
      pMP->UpdateNormalAndDepth();
      self.mpMap->AddMapPoint(pMP);
      self.mlpRecentAddedMapPoints.push_back(pMP);
      nnew++;
    }
  }
}

struct Scene {
  LocalMapping lm;
  std::vector<kfptr> kfs;   // 0 the current keyframe, 1.. its neighbours in covisibility order
  mpptr placeholder;        // the map point that stands for "this feature already carries one"
};

}  // namespace
}  // namespace cslam

using namespace cslam;

extern "C" {

// views: n_kf structs of the library's own layout (the test builds them with api.new_points_structs); median_depth per keyframe
void* np_scene_create(int32_t n_kf, const ccm_newpts_view* const* views, const float* median_depth) {
  Scene* s = new Scene;
  s->lm.mpCC.reset(new CentralControl); s->lm.mpMap.reset(new Map); s->lm.mpComm.reset(new Communicator);
  s->lm.mClientId = 3; s->lm.mpCC->mSysState = 1;
  s->placeholder.reset(new MapPoint(cv::Mat(3, 1, CV_32F), kfptr(), s->lm.mpMap, 0, s->lm.mpComm, 0, 0));
  for (int k = 0; k < n_kf; k++) {
    const ccm_newpts_view* v = views[k];
    kfptr p(new KeyFrame);
    p->N = v->v.n;
    p->fx = v->v.fx; p->fy = v->v.fy; p->cx = v->v.cx; p->cy = v->v.cy; p->invfx = 1.0f / p->fx; p->invfy = 1.0f / p->fy;
    p->mK = cv::Mat::eye(3, 3, CV_32F);
    p->mK.at<float>(0, 0) = p->fx; p->mK.at<float>(1, 1) = p->fy; p->mK.at<float>(0, 2) = p->cx; p->mK.at<float>(1, 2) = p->cy;
    p->mDescriptors = cv::Mat(p->N, 32, CV_8U);
    if (p->N) memcpy(p->mDescriptors.ptr(), v->v.desc, (size_t)p->N * 32);
    for (int i = 0; i < p->N; i++) {
      p->mvKeysUn.push_back(cv::KeyPoint(v->v.kp_xy[2 * i], v->v.kp_xy[2 * i + 1], 31.f, v->v.angle[i], 0, v->v.octave[i]));
      p->mvpMapPoints.push_back(v->v.has_mp[i] ? s->placeholder : mpptr());
    }
    for (int a = 0; a < v->v.fv->n_nodes; a++)
      for (int e = v->v.fv->node_ptr[a]; e < v->v.fv->node_ptr[a + 1]; e++) p->mFeatVec[v->v.fv->node_id[a]].push_back(v->v.fv->feat[e]);
    p->mfScaleFactor = v->scale_factor;
    p->mvScaleFactors.assign(v->scale_factors, v->scale_factors + v->nlevels);
    p->mvLevelSigma2.assign(v->level_sigma2, v->level_sigma2 + v->nlevels);
    p->Tcw = cv::Mat::eye(4, 4, CV_32F);
    for (int r = 0; r < 3; r++) for (int c = 0; c < 4; c++) p->Tcw.at<float>(r, c) = v->Tcw[4 * r + c];
    p->Ow = cv::Mat(3, 1, CV_32F);
    for (int r = 0; r < 3; r++) p->Ow.at<float>(r) = v->Ow[r];
    p->mMedianDepthForTest = median_depth[k];
    s->kfs.push_back(p);
  }
  s->lm.mpCurrentKeyFrame = s->kfs[0];
  s->kfs[0]->mvpOrderedConnectedKeyFrames.assign(s->kfs.begin() + 1, s->kfs.end());
  return s;
}

void np_scene_destroy(void* h) { delete static_cast<Scene*>(h); }

// mode 0 the literal body, 1 the shim member; force_at_poll: the CheckNewKeyFrames() call (1-based) that answers true, -1 never.
// Returns 0, or 1 when the body threw.
int np_run(void* h, int mode, int force_at_poll) {
  Scene* s = static_cast<Scene*>(h);
  s->lm.mPolls = 0; s->lm.mForceAtPoll = force_at_poll;
  try {
    if (mode == 0) literal_CreateNewMapPoints(s->lm);
    else s->lm.CreateNewMapPoints();
  } catch (const estd::infrastructure_ex&) {
    return 1;
  }
  return 0;
}

int32_t np_point_count(void* h) { return (int32_t)static_cast<Scene*>(h)->lm.mpMap->mvpAdded.size(); }
int32_t np_polls(void* h) { return static_cast<Scene*>(h)->lm.mPolls; }

// mvp [sum of N]: per keyframe and feature -1 (none), -2 (the map point it had before) or the index of the new point in the map's list;
// per new point: pos [3], ref (keyframe index), obs [2 x (keyframe index, feature)] in std::map order replaced by (current, neighbour),
// log [8] the members called on it; recent [points]: the recent-points list as indices.  Returns the number of points.
int32_t np_members(void* h, int32_t* mvp, float* pos, int32_t* ref, int32_t* obs, char* log, int32_t* recent, int32_t* n_recent) {
  Scene* s = static_cast<Scene*>(h);
  const std::vector<mpptr>& pts = s->lm.mpMap->mvpAdded;
  auto point_index = [&](const mpptr& p) { for (size_t i = 0; i < pts.size(); i++) if (pts[i] == p) return (int32_t)i; return (int32_t)-3; };
  auto kf_index = [&](const kfptr& p) { for (size_t i = 0; i < s->kfs.size(); i++) if (s->kfs[i] == p) return (int32_t)i; return (int32_t)-1; };
  size_t at = 0;
  for (auto& kf : s->kfs)
    for (int i = 0; i < kf->N; i++) {
      const mpptr& p = kf->mvpMapPoints[i];
      mvp[at++] = !p ? -1 : p == s->placeholder ? -2 : point_index(p);
    }
  for (size_t i = 0; i < pts.size(); i++) {
    for (int r = 0; r < 3; r++) pos[3 * i + r] = pts[i]->mWorldPos.at<float>(r);
    ref[i] = kf_index(pts[i]->mpRefKF);
    int k = 0;
    for (int pass = 0; pass < 2; pass++)   // the current keyframe's observation first, whatever the pointer order of the std::map
      for (auto& o : pts[i]->mObservations)
        if ((kf_index(o.first) == 0) == (pass == 0) && k < 2) { obs[4 * i + 2 * k] = kf_index(o.first); obs[4 * i + 2 * k + 1] = (int32_t)o.second; k++; }
    for (; k < 2; k++) { obs[4 * i + 2 * k] = -1; obs[4 * i + 2 * k + 1] = -1; }
    memset(log + 8 * i, 0, 8);
    strncpy(log + 8 * i, pts[i]->mLog.c_str(), 7);
  }
  *n_recent = 0;
  for (auto& p : s->lm.mlpRecentAddedMapPoints) recent[(*n_recent)++] = point_index(p);
  return (int32_t)pts.size();
}

void np_shim_stats(unsigned long long* c) { ccm_b200_new_map_points_stats(c, c + 1, c + 2); }

}  // extern "C"

// ref_search_and_fuse_wrap.cpp — a literal restatement of LoopFinder::SearchAndFuse (cslam/src/LoopFinder.cpp:709-734),
// MapMerger::SearchAndFuse (cslam/src/MapMerger.cpp:574-598), ORBmatcher::Fuse(pKF, Scw, vpPoints, th, vpReplacePoint)
// (cslam/src/ORBmatcher.cpp:995-1122), MapPoint::Replace (cslam/src/MapPoint.cpp:583-678) and MapPoint::ReplaceAndLock (:680-720),
// over the stand-ins of ref_stub_sf/, next to shim/SearchAndFuse_shim.cpp on the same stand-ins (TEST INFRASTRUCTURE).
//
// sf_scene_create builds keyframes, Sim3s and points from flat arrays; sf_run runs mode 0 (the restatement) or 1 (the shim), at the loop
// site (merge = 0) or the merge site (merge = 1); sf_members reads back what the member changed.
#include <climits>
#include <cstdint>
#include <cstring>
#include <memory>
#include <stdexcept>
#include <vector>

#include <cslam/Converter.h>
#include <cslam/KeyFrame.h>

#include "../shim/SearchAndFuse_shim.h"
#include "ccm_b200.h"

namespace cslam {

static int DescriptorDistance(const cv::Mat& a, const cv::Mat& b) {   // ORBmatcher::DescriptorDistance
  const int* pa = a.ptr<int32_t>();
  const int* pb = b.ptr<int32_t>();
  int dist = 0;
  for (int i = 0; i < 8; i++, pa++, pb++) dist += __builtin_popcount((unsigned)(*pa ^ *pb));
  return dist;
}

// MapPoint::Replace, monocular, statement by statement (cslam/src/MapPoint.cpp:583-678)
void MapPoint::Replace(mpptr pMP, bool bLock) {
  mLog += lock_letter('r', bLock);
  if (pMP->mId == this->mId) return;
  int nvisible, nfound;
  std::map<kfptr, size_t, KfById> obs;
  {
    obs = mObservations;
    mObservations.clear();
    mbBad = true;
    nvisible = mnVisible;
    nfound = mnFound;
    mpReplaced = pMP;
  }
  for (auto mit = obs.begin(), mend = obs.end(); mit != mend; mit++) {
    kfptr pKF = mit->first;
    if (!pMP->IsInKeyFrame(pKF)) {
      pKF->ReplaceMapPointMatch(mit->second, pMP, bLock);
      pMP->AddObservation(pKF, mit->second, bLock);
    } else {
      if ((int)mit->second == pMP->GetIndexInKeyFrame(pKF)) {
        pKF->EraseMapPointMatch(mit->second, bLock);
        pKF->AddMapPoint(pMP, mit->second, bLock);
      } else if (pMP->GetIndexInKeyFrame(pKF) >= 0) {
        mLog += 'i';   // the id-mismatch branch
        pKF->EraseMapPointMatch(mit->second, bLock);
        std::vector<mpptr> mvpMPs = pKF->GetMapPointMatches();
        std::vector<mpptr>::iterator vit = std::find(mvpMPs.begin(), mvpMPs.end(), pMP);
        int id = vit - mvpMPs.begin();
        if (id == pMP->GetIndexInKeyFrame(pKF)) {
        } else if (vit == mvpMPs.end()) {
          const cv::Mat dMP = pMP->GetDescriptor();
          const cv::Mat dKF_pMP_id = pKF->mDescriptors.row(pMP->GetIndexInKeyFrame(pKF));
          const cv::Mat dKF_this_id = pKF->mDescriptors.row(mit->second);
          double dist_pMP_id = DescriptorDistance(dMP, dKF_pMP_id);
          double dist_this_id = DescriptorDistance(dMP, dKF_this_id);
          if (dist_pMP_id <= dist_this_id) {
            pKF->AddMapPoint(pMP, pMP->GetIndexInKeyFrame(pKF), false);
          } else {
            pKF->AddMapPoint(pMP, mit->second, bLock);
            pMP->EraseObservation(pKF, bLock);
            pMP->AddObservation(pKF, mit->second, bLock);
          }
        }
      } else {
        throw std::runtime_error("id mismatch");
      }
    }
  }
  pMP->IncreaseFound(nfound);
  pMP->IncreaseVisible(nvisible);
  pMP->ComputeDistinctiveDescriptors();
  mpMap->EraseMapPoint(self());
}

// MapPoint::ReplaceAndLock, statement by statement (cslam/src/MapPoint.cpp:680-720)
void MapPoint::ReplaceAndLock(mpptr pMP) {
  mLog += 'l';
  if (pMP->mId == this->mId) return;
  int nvisible, nfound;
  std::map<kfptr, size_t, KfById> obs;
  {
    obs = mObservations;
    mObservations.clear();
    mbBad = true;
    nvisible = mnVisible;
    nfound = mnFound;
    mpReplaced = pMP;
  }
  for (auto mit = obs.begin(), mend = obs.end(); mit != mend; mit++) {
    kfptr pKF = mit->first;
    if (pKF->IsEmpty()) continue;
    if (!pMP->IsInKeyFrame(pKF)) {
      pKF->ReplaceMapPointMatch(mit->second, pMP, true);
      pMP->AddObservation(pKF, mit->second, true);
    } else {
      pKF->EraseMapPointMatch(mit->second, true);
    }
  }
  pMP->IncreaseFound(nfound);
  pMP->IncreaseVisible(nvisible);
  pMP->ComputeDistinctiveDescriptors();
  mpMap->EraseMapPoint(self());
}

// what the scene builder may set on a point beyond the public members
struct SfSceneAccess {
  static void distances(MapPoint& m, float mx, float mn) { m.mfMaxDistance = mx; m.mfMinDistance = mn; }
};

namespace {

typedef KeyFrame::kfptr kfptr;
typedef KeyFrame::mpptr mpptr;

// ORBmatcher::Fuse(kfptr pKF, cv::Mat Scw, const vector<mpptr>& vpPoints, float th, vector<mpptr>& vpReplacePoint), statement by statement
int Fuse(kfptr pKF, cv::Mat Scw, const std::vector<mpptr>& vpPoints, float th, std::vector<mpptr>& vpReplacePoint) {
  const int TH_LOW = 50;
  const float& fx = pKF->fx;
  const float& fy = pKF->fy;
  const float& cx = pKF->cx;
  const float& cy = pKF->cy;
  cv::Mat sRcw = Scw.rowRange(0, 3).colRange(0, 3);
  const float scw = sqrt(sRcw.row(0).dot(sRcw.row(0)));
  cv::Mat Rcw = sRcw / scw;
  cv::Mat tcw = Scw.rowRange(0, 3).col(3) / scw;
  cv::Mat Ow = -Rcw.t() * tcw;
  const std::set<mpptr> spAlreadyFound = pKF->GetMapPoints();
  int nFused = 0;
  const int nPoints = vpPoints.size();
  for (int iMP = 0; iMP < nPoints; iMP++) {
    mpptr pMP = vpPoints[iMP];
    if (pMP->isBad() || spAlreadyFound.count(pMP)) continue;
    cv::Mat p3Dw = pMP->GetWorldPos();
    cv::Mat p3Dc = Rcw * p3Dw + tcw;
    if (p3Dc.at<float>(2) < 0.0f) continue;
    const float invz = 1.0 / p3Dc.at<float>(2);
    const float x = p3Dc.at<float>(0) * invz;
    const float y = p3Dc.at<float>(1) * invz;
    const float u = fx * x + cx;
    const float v = fy * y + cy;
    if (!pKF->IsInImage(u, v)) continue;
    const float maxDistance = pMP->GetMaxDistanceInvariance();
    const float minDistance = pMP->GetMinDistanceInvariance();
    cv::Mat PO = p3Dw - Ow;
    const float dist3D = cv::norm(PO);
    if (dist3D < minDistance || dist3D > maxDistance) continue;
    cv::Mat Pn = pMP->GetNormal();
    if (PO.dot(Pn) < 0.5 * dist3D) continue;
    int nPredictedLevel = pMP->PredictScale(dist3D, pKF);
    const float radius = th * pKF->mvScaleFactors[nPredictedLevel];
    const std::vector<size_t> vIndices = pKF->GetFeaturesInArea(u, v, radius);
    if (vIndices.empty()) continue;
    const cv::Mat dMP = pMP->GetDescriptor();
    int bestDist = INT_MAX;
    int bestIdx = -1;
    for (std::vector<size_t>::const_iterator vit = vIndices.begin(); vit != vIndices.end(); vit++) {
      const size_t idx = *vit;
      const int& kpLevel = pKF->mvKeysUn[idx].octave;
      if (kpLevel < nPredictedLevel - 1 || kpLevel > nPredictedLevel) continue;
      const cv::Mat dKF = pKF->mDescriptors.row(idx);
      int dist = DescriptorDistance(dMP, dKF);
      if (dist < bestDist) {
        bestDist = dist;
        bestIdx = idx;
      }
    }
    if (bestDist <= TH_LOW) {
      mpptr pMPinKF = pKF->GetMapPoint(bestIdx);
      if (pMPinKF) {
        if (!pMPinKF->isBad()) vpReplacePoint[iMP] = pMPinKF;
      } else {
        pMP->AddObservation(pKF, bestIdx);
        pKF->AddMapPoint(pMP, bestIdx);
      }
      nFused++;
    }
  }
  return nFused;
}

// LoopFinder::SearchAndFuse (merge = false) and MapMerger::SearchAndFuse (merge = true), statement by statement
void RefSearchAndFuse(const Sim3CorrectionMap& CorrectedPosesMap, std::vector<mpptr> vpLoopMapPoints, bool merge) {
  for (Sim3CorrectionMap::const_iterator mit = CorrectedPosesMap.begin(), mend = CorrectedPosesMap.end(); mit != mend; mit++) {
    kfptr pKF = mit->first;
    g2o::Sim3 g2oScw = mit->second;
    cv::Mat cvScw = Converter::toCvMat(g2oScw);
    std::vector<mpptr> vpReplacePoints(vpLoopMapPoints.size(), nullptr);
    Fuse(pKF, cvScw, vpLoopMapPoints, 4, vpReplacePoints);
    const int nLP = vpLoopMapPoints.size();
    for (int i = 0; i < nLP; i++) {
      mpptr pRep = vpReplacePoints[i];
      if (pRep) {
        if (merge) pRep->ReplaceAndLock(vpLoopMapPoints[i]);
        else pRep->Replace(vpLoopMapPoints[i], true);
      }
    }
  }
}

struct NoDelete { void operator()(KeyFrame*) const {} };

struct Scene {
  // the keyframes live in one array, so that the KeyFrameAndPose's std::less<kfptr> (address) order is the row order in every copy
  // of a scene, and the shim and the restatement walk the same order
  std::unique_ptr<KeyFrame[]> store;
  Sim3CorrectionMap corrected;
  std::vector<kfptr> kfs;
  std::vector<mpptr> pts, loop;
  std::map<MapPoint*, int> row;
  std::map<KeyFrame*, int> kfrow;
};

}  // namespace
}  // namespace cslam

using namespace cslam;

// kfs: the keyframes' grids, intrinsics and scale tables (Tcw / Ow are not read); sim3[k]: qx qy qz qw tx ty tz s of keyframe k's
// corrected Sim3; kf_empty[k]: mbIsEmpty.  Points 0..P-1 (pos, normal, distances, descriptor, bad); slot_ptr / slot: each keyframe's
// mvpMapPoints as point rows (-1 empty), and a point observes (k, j) for every slot that holds it; loop[0..n_loop): vpLoopMapPoints.
extern "C" void* sf_scene_create(int32_t K, const ccm_fuse_kf* kfs, const double* sim3, const uint8_t* kf_empty, const int32_t* slot_ptr,
                                 const int32_t* slot, int32_t P, const float* pos, const float* normal, const float* max_d, const float* min_d,
                                 const uint8_t* desc, const uint8_t* bad, const int32_t* loop, int32_t n_loop) {
  Scene* s = new Scene;
  auto map = boost::shared_ptr<Map>(new Map);
  s->store.reset(new KeyFrame[K]);
  for (int k = 0; k < K; k++) {
    kfptr f(&s->store[k], NoDelete());
    const ccm_fuse_kf& c = kfs[k];
    f->mId = 1000 + k; f->mbIsEmpty = kf_empty[k] != 0;
    f->fx = c.fx; f->fy = c.fy; f->cx = c.cx; f->cy = c.cy; f->N = c.grid.n;
    f->mvKeysUn.resize(c.grid.n);
    for (int i = 0; i < c.grid.n; i++) {
      f->mvKeysUn[i].pt.x = c.grid.kp_xy[2 * i]; f->mvKeysUn[i].pt.y = c.grid.kp_xy[2 * i + 1]; f->mvKeysUn[i].octave = c.grid.octave[i];
    }
    f->mDescriptors = cv::Mat(c.grid.n, 32, CV_8U);
    if (c.grid.n) std::memcpy(f->mDescriptors.ptr(), c.grid.desc, 32 * (size_t)c.grid.n);
    f->mnScaleLevels = c.nlevels; f->mfLogScaleFactor = c.log_scale_factor;
    f->mvScaleFactors.assign(c.scale_factors, c.scale_factors + c.nlevels);
    f->mnMinX = (int)c.grid.min_x; f->mnMinY = (int)c.grid.min_y; f->mnMaxX = (int)c.grid.max_x; f->mnMaxY = (int)c.grid.max_y;
    f->mnGridCols = c.grid.grid_cols; f->mnGridRows = c.grid.grid_rows;
    f->mfGridElementWidthInv = c.grid.grid_w_inv; f->mfGridElementHeightInv = c.grid.grid_h_inv;
    f->AssignFeaturesToGrid();
    f->mvpMapPoints.assign(c.grid.n, nullptr);
    const double* q = sim3 + 8 * k;
    s->corrected[f] = g2o::Sim3(g2o::Quaterniond(q[3], q[0], q[1], q[2]), g2o::Vector3d(q[4], q[5], q[6]), q[7]);
    s->kfrow[f.get()] = k;
    s->kfs.push_back(f);
  }
  for (int p = 0; p < P; p++) {
    mpptr m(new MapPoint);
    m->mSelf = m; m->mpMap = map; m->mId = 1 + p;
    m->mWorldPos = cv::Mat(3, 1, CV_32F); m->mNormalVector = cv::Mat(3, 1, CV_32F); m->mDescriptor = cv::Mat(1, 32, CV_8U);
    for (int r = 0; r < 3; r++) { m->mWorldPos.at<float>(r) = pos[3 * p + r]; m->mNormalVector.at<float>(r) = normal[3 * p + r]; }
    std::memcpy(m->mDescriptor.ptr(), desc + 32 * (size_t)p, 32);
    SfSceneAccess::distances(*m, max_d[p], min_d[p]);
    m->mbBad = bad[p] != 0;
    s->row[m.get()] = p;
    s->pts.push_back(m);
  }
  for (int k = 0; k < K; k++)
    for (int j = 0; j < slot_ptr[k + 1] - slot_ptr[k]; j++) {
      const int r = slot[slot_ptr[k] + j];
      if (r < 0) continue;
      s->kfs[k]->mvpMapPoints[j] = s->pts[r];
      if (!s->pts[r]->mbBad && !s->pts[r]->mObservations.count(s->kfs[k])) { s->pts[r]->mObservations[s->kfs[k]] = j; s->pts[r]->nObs++; }
    }
  for (int i = 0; i < n_loop; i++) s->loop.push_back(s->pts[loop[i]]);
  return s;
}

extern "C" void sf_scene_destroy(void* h) {
  Scene* s = static_cast<Scene*>(h);
  for (auto& p : s->pts) { p->mObservations.clear(); p->mpReplaced.reset(); }
  for (auto& k : s->kfs) k->mvpMapPoints.clear();
  delete s;
}

extern "C" int sf_run(void* h, int mode, int merge) {
  Scene* s = static_cast<Scene*>(h);
  try {
    if (mode == 0) RefSearchAndFuse(s->corrected, s->loop, merge != 0);
    else ccm_b200_search_and_fuse(s->corrected, s->loop, merge != 0);
  } catch (...) {
    return 1;
  }
  return 0;
}

// mvp: every keyframe's slots as point rows; per point: bad, replaced row, descriptor, observations (kf row, idx) in map order
// (obs_ptr / obs), call log (log_ptr / log); per keyframe its call log (klog_ptr / klog)
extern "C" void sf_members(void* h, int32_t* mvp, uint8_t* bad, int32_t* replaced, uint8_t* desc, int32_t* obs_ptr, int32_t* obs, int32_t obs_cap,
                           int32_t* log_ptr, char* log, int32_t log_cap, int32_t* klog_ptr, char* klog, int32_t klog_cap) {
  Scene* s = static_cast<Scene*>(h);
  int at = 0;
  for (auto& k : s->kfs)
    for (auto& m : k->mvpMapPoints) mvp[at++] = m ? s->row[m.get()] : -1;
  int o = 0, l = 0;
  obs_ptr[0] = 0; log_ptr[0] = 0;
  for (size_t p = 0; p < s->pts.size(); p++) {
    const mpptr& m = s->pts[p];
    bad[p] = m->mbBad;
    replaced[p] = m->mpReplaced ? s->row[m->mpReplaced.get()] : -1;
    std::memcpy(desc + 32 * p, m->mDescriptor.ptr(), 32);
    for (auto& ob : m->mObservations)
      if (o + 2 <= obs_cap) { obs[o++] = s->kfrow[ob.first.get()]; obs[o++] = (int32_t)ob.second; }
    obs_ptr[p + 1] = o;
    for (char c : m->mLog)
      if (l < log_cap) log[l++] = c;
    log_ptr[p + 1] = l;
  }
  int kl = 0;
  klog_ptr[0] = 0;
  for (size_t k = 0; k < s->kfs.size(); k++) {
    for (char c : s->kfs[k]->mLog)
      if (kl < klog_cap) klog[kl++] = c;
    klog_ptr[k + 1] = kl;
  }
}

extern "C" void sf_shim_stats(unsigned long long* c) { ccm_b200_search_and_fuse_stats(&c[0], &c[1]); }

// ref_fuse_neighbours_wrap.cpp — a literal restatement of LocalMapping::SearchInNeighbors (cslam/src/Mapping.cpp:471-547), of
// ORBmatcher::Fuse(pKF, vpMapPoints, th) (cslam/src/ORBmatcher.cpp:854-993) and of MapPoint::Replace (cslam/src/MapPoint.cpp:583-678),
// over the stand-ins of ref_stub_fn/, next to shim/FuseNeighbours_shim.cpp on the same stand-ins (TEST INFRASTRUCTURE).
//
// fn_scene_create builds keyframes and points from flat arrays; fn_run runs mode 0 (the restatement) or 1 (the shim); fn_members reads
// back what the member changed.  The shim's batch of the update tail is stood in for here: it marks each point it was handed ('p').
#include <cstdint>
#include <cstring>
#include <iostream>
#include <string>
#include <vector>

#include <cslam/Mapping.h>

#include "../shim/FuseNeighbours_shim.h"
#include "ccm_b200.h"

namespace cslam {

// MapPoint::Replace, monocular client, statement by statement (cslam/src/MapPoint.cpp:583-678); the descriptor distance of the
// remap branch is ORBmatcher::DescriptorDistance
static int DescriptorDistance(const cv::Mat& a, const cv::Mat& b) {
  const int* pa = a.ptr<int32_t>();
  const int* pb = b.ptr<int32_t>();
  int dist = 0;
  for (int i = 0; i < 8; i++, pa++, pb++) dist += __builtin_popcount((unsigned)(*pa ^ *pb));
  return dist;
}

void MapPoint::Replace(mpptr pMP, bool bLock) {
  mLog += 'r';
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

// the batch entry of shim/MapPointDescriptor_shim.cpp as the shim calls it; the parked choices are not modelled
void ccm_b200_prepare_point_updates(const std::vector<boost::shared_ptr<MapPoint> >& points) { for (auto& p : points) p->mLog += 'p'; }
void ccm_b200_clear_descriptors() {}

namespace {

typedef KeyFrame::kfptr kfptr;
typedef KeyFrame::mpptr mpptr;

// ORBmatcher::Fuse(kfptr pKF, const vector<mpptr>& vpMapPoints, const float th=3.0), statement by statement
int Fuse(kfptr pKF, const std::vector<mpptr>& vpMapPoints, const float th = 3.0) {
  const int TH_LOW = 50;
  cv::Mat Rcw = pKF->GetRotation();
  cv::Mat tcw = pKF->GetTranslation();
  const float& fx = pKF->fx;
  const float& fy = pKF->fy;
  const float& cx = pKF->cx;
  const float& cy = pKF->cy;
  cv::Mat Ow = pKF->GetCameraCenter();
  int nFused = 0;
  const int nMPs = vpMapPoints.size();
  for (int i = 0; i < nMPs; i++) {
    mpptr pMP = vpMapPoints[i];
    if (!pMP) continue;
    if (pMP->isBad() || pMP->IsInKeyFrame(pKF)) continue;
    if (pMP->mbDoNotReplace) continue;
    cv::Mat p3Dw = pMP->GetWorldPos();
    cv::Mat p3Dc = Rcw * p3Dw + tcw;
    if (p3Dc.at<float>(2) < 0.0f) continue;
    const float invz = 1 / p3Dc.at<float>(2);
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
    int bestDist = 256;
    int bestIdx = -1;
    for (std::vector<size_t>::const_iterator vit = vIndices.begin(), vend = vIndices.end(); vit != vend; vit++) {
      const size_t idx = *vit;
      const cv::KeyPoint& kp = pKF->mvKeysUn[idx];
      const int& kpLevel = kp.octave;
      if (kpLevel < nPredictedLevel - 1 || kpLevel > nPredictedLevel) continue;
      const float& kpx = kp.pt.x;
      const float& kpy = kp.pt.y;
      const float ex = u - kpx;
      const float ey = v - kpy;
      const float e2 = ex * ex + ey * ey;
      if (e2 * pKF->mvInvLevelSigma2[kpLevel] > 5.99) continue;
      const cv::Mat dKF = pKF->mDescriptors.row(idx);
      const int dist = DescriptorDistance(dMP, dKF);
      if (dist < bestDist) {
        bestDist = dist;
        bestIdx = idx;
      }
    }
    if (bestDist <= TH_LOW) {
      mpptr pMPinKF = pKF->GetMapPoint(bestIdx);
      if (pMPinKF) {
        if (!pMPinKF->isBad() && !pMPinKF->mbDoNotReplace) {
          if (pMPinKF->Observations() > pMP->Observations())
            pMP->Replace(pMPinKF);
          else
            pMPinKF->Replace(pMP);
        }
      } else {
        pMP->AddObservation(pKF, bestIdx);
        pKF->AddMapPoint(pMP, bestIdx);
      }
      nFused++;
    }
  }
  return nFused;
}

// LocalMapping::SearchInNeighbors, statement by statement
void RefSearchInNeighbors(LocalMapping& lm) {
  kfptr& mpCurrentKeyFrame = lm.mpCurrentKeyFrame;
  int nn = 20;
  const std::vector<kfptr> vpNeighKFs = mpCurrentKeyFrame->GetBestCovisibilityKeyFrames(nn);
  std::vector<kfptr> vpTargetKFs;
  for (std::vector<kfptr>::const_iterator vit = vpNeighKFs.begin(), vend = vpNeighKFs.end(); vit != vend; vit++) {
    kfptr pKFi = *vit;
    if (pKFi->isBad() || pKFi->mFuseTargetForKF == mpCurrentKeyFrame->mId) continue;
    vpTargetKFs.push_back(pKFi);
    pKFi->mFuseTargetForKF = mpCurrentKeyFrame->mId;
    const std::vector<kfptr> vpSecondNeighKFs = pKFi->GetBestCovisibilityKeyFrames(5);
    for (std::vector<kfptr>::const_iterator vit2 = vpSecondNeighKFs.begin(), vend2 = vpSecondNeighKFs.end(); vit2 != vend2; vit2++) {
      kfptr pKFi2 = *vit2;
      if (pKFi2->isBad() || pKFi2->mFuseTargetForKF == mpCurrentKeyFrame->mId || pKFi2->mId == mpCurrentKeyFrame->mId) continue;
      vpTargetKFs.push_back(pKFi2);
    }
  }
  std::vector<mpptr> vpMapPointMatches = mpCurrentKeyFrame->GetMapPointMatches();
  for (std::vector<kfptr>::iterator vit = vpTargetKFs.begin(), vend = vpTargetKFs.end(); vit != vend; vit++) {
    kfptr pKFi = *vit;
    Fuse(pKFi, vpMapPointMatches);
  }
  std::vector<mpptr> vpFuseCandidates;
  vpFuseCandidates.reserve(vpTargetKFs.size() * vpMapPointMatches.size());
  for (std::vector<kfptr>::iterator vitKF = vpTargetKFs.begin(), vendKF = vpTargetKFs.end(); vitKF != vendKF; vitKF++) {
    kfptr pKFi = *vitKF;
    std::vector<mpptr> vpMapPointsKFi = pKFi->GetMapPointMatches();
    for (std::vector<mpptr>::iterator vitMP = vpMapPointsKFi.begin(), vendMP = vpMapPointsKFi.end(); vitMP != vendMP; vitMP++) {
      mpptr pMP = *vitMP;
      if (!pMP) continue;
      if (pMP->isBad() || pMP->mFuseCandidateForKF == mpCurrentKeyFrame->mId) continue;
      pMP->mFuseCandidateForKF = mpCurrentKeyFrame->mId;
      vpFuseCandidates.push_back(pMP);
    }
  }
  Fuse(mpCurrentKeyFrame, vpFuseCandidates);
  vpMapPointMatches = mpCurrentKeyFrame->GetMapPointMatches();
  std::vector<mpptr> vpUpdate;   // the shim hands these to its batch; the same marks here keep the call logs comparable
  for (const mpptr& pMP : vpMapPointMatches)
    if (pMP && !pMP->isBad()) vpUpdate.push_back(pMP);
  ccm_b200_prepare_point_updates(vpUpdate);
  for (size_t i = 0, iend = vpMapPointMatches.size(); i < iend; i++) {
    mpptr pMP = vpMapPointMatches[i];
    if (pMP) {
      if (!pMP->isBad()) {
        pMP->ComputeDistinctiveDescriptors();
        pMP->UpdateNormalAndDepth();
      }
    }
  }
  mpCurrentKeyFrame->UpdateConnections();
}

struct Scene {
  LocalMapping lm;
  std::vector<kfptr> kfs;
  std::vector<mpptr> pts;
  std::map<MapPoint*, int> row;
  std::map<KeyFrame*, int> kfrow;
};

}  // namespace
}  // namespace cslam

using namespace cslam;

// kfs[0] the current keyframe; conn_ptr / conn: each keyframe's ordered connections as keyframe rows; slot_ptr / slot: each keyframe's
// mvpMapPoints as point rows (-1 empty); a point observes (k, j) for every slot that holds it.
extern "C" void* fn_scene_create(int32_t K, const ccm_fuse_kf* kfs, const uint8_t* kf_bad, const int32_t* conn_ptr, const int32_t* conn,
                                 const int32_t* slot_ptr, const int32_t* slot, int32_t P, const float* pos, const float* normal,
                                 const float* max_d, const float* min_d, const uint8_t* desc, const uint8_t* dnr, const uint8_t* bad) {
  Scene* s = new Scene;
  auto map = boost::shared_ptr<Map>(new Map);
  for (int k = 0; k < K; k++) {
    kfptr f(new KeyFrame);
    const ccm_fuse_kf& c = kfs[k];
    f->mId = 1000 + k; f->mbBad = kf_bad[k] != 0;
    f->fx = c.fx; f->fy = c.fy; f->cx = c.cx; f->cy = c.cy; f->N = c.grid.n;
    f->mvKeysUn.resize(c.grid.n);
    for (int i = 0; i < c.grid.n; i++) {
      f->mvKeysUn[i].pt.x = c.grid.kp_xy[2 * i]; f->mvKeysUn[i].pt.y = c.grid.kp_xy[2 * i + 1]; f->mvKeysUn[i].octave = c.grid.octave[i];
    }
    f->mDescriptors = cv::Mat(c.grid.n, 32, CV_8U);
    if (c.grid.n) std::memcpy(f->mDescriptors.ptr(), c.grid.desc, 32 * (size_t)c.grid.n);
    f->mnScaleLevels = c.nlevels; f->mfLogScaleFactor = c.log_scale_factor;
    f->mvScaleFactors.assign(c.scale_factors, c.scale_factors + c.nlevels);
    f->mvInvLevelSigma2.assign(c.inv_level_sigma2, c.inv_level_sigma2 + c.nlevels);
    f->mnMinX = (int)c.grid.min_x; f->mnMinY = (int)c.grid.min_y; f->mnMaxX = (int)c.grid.max_x; f->mnMaxY = (int)c.grid.max_y;
    f->mnGridCols = c.grid.grid_cols; f->mnGridRows = c.grid.grid_rows;
    f->mfGridElementWidthInv = c.grid.grid_w_inv; f->mfGridElementHeightInv = c.grid.grid_h_inv;
    f->Tcw = cv::Mat(3, 4, CV_32F); f->Ow = cv::Mat(3, 1, CV_32F);
    for (int r = 0; r < 3; r++) { for (int q = 0; q < 4; q++) f->Tcw.at<float>(r, q) = c.Tcw[4 * r + q]; f->Ow.at<float>(r) = c.Ow[r]; }
    f->AssignFeaturesToGrid();
    f->mvpMapPoints.assign(c.grid.n, nullptr);
    s->kfrow[f.get()] = k;
    s->kfs.push_back(f);
  }
  for (int p = 0; p < P; p++) {
    mpptr m(new MapPoint);
    m->mSelf = m; m->mpMap = map; m->mId = 1 + p;
    m->mWorldPos = cv::Mat(3, 1, CV_32F); m->mNormalVector = cv::Mat(3, 1, CV_32F); m->mDescriptor = cv::Mat(1, 32, CV_8U);
    for (int r = 0; r < 3; r++) { m->mWorldPos.at<float>(r) = pos[3 * p + r]; m->mNormalVector.at<float>(r) = normal[3 * p + r]; }
    std::memcpy(m->mDescriptor.ptr(), desc + 32 * (size_t)p, 32);
    m->mfMaxDistance = max_d[p]; m->mfMinDistance = min_d[p]; m->mbDoNotReplace = dnr[p] != 0; m->mbBad = bad[p] != 0;
    s->row[m.get()] = p;
    s->pts.push_back(m);
  }
  for (int k = 0; k < K; k++) {
    for (int j = conn_ptr[k]; j < conn_ptr[k + 1]; j++) s->kfs[k]->mvpOrderedConnectedKeyFrames.push_back(s->kfs[conn[j]]);
    for (int j = 0; j < slot_ptr[k + 1] - slot_ptr[k]; j++) {
      const int r = slot[slot_ptr[k] + j];
      if (r < 0) continue;
      s->kfs[k]->mvpMapPoints[j] = s->pts[r];
      if (!s->pts[r]->mbBad && !s->pts[r]->mObservations.count(s->kfs[k])) { s->pts[r]->mObservations[s->kfs[k]] = j; s->pts[r]->nObs++; }
    }
  }
  s->lm.mpCurrentKeyFrame = s->kfs[0];
  return s;
}

extern "C" void fn_scene_destroy(void* h) {
  Scene* s = static_cast<Scene*>(h);
  for (auto& p : s->pts) { p->mObservations.clear(); p->mpReplaced.reset(); }
  for (auto& k : s->kfs) { k->mvpMapPoints.clear(); k->mvpOrderedConnectedKeyFrames.clear(); }
  delete s;
}

extern "C" int fn_run(void* h, int mode) {
  Scene* s = static_cast<Scene*>(h);
  try {
    if (mode == 0) RefSearchInNeighbors(s->lm);
    else s->lm.SearchInNeighbors();
  } catch (...) {
    return 1;
  }
  return 0;
}

// mvp: every keyframe's slots as point rows; per point: bad, replaced row, descriptor, candidate mark, observations (kf row, idx) in map
// order (obs_ptr / obs), call log (log_ptr / log); per keyframe: fuse-target mark and UpdateConnections count
extern "C" void fn_members(void* h, int32_t* mvp, uint8_t* bad, int32_t* replaced, uint8_t* desc, int64_t* cand_mark, int32_t* obs_ptr,
                           int32_t* obs, int32_t obs_cap, int32_t* log_ptr, char* log, int32_t log_cap, int64_t* target_mark, int32_t* conn_updates) {
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
    cand_mark[p] = (int64_t)m->mFuseCandidateForKF;
    for (auto& ob : m->mObservations)
      if (o + 2 <= obs_cap) { obs[o++] = s->kfrow[ob.first.get()]; obs[o++] = (int32_t)ob.second; }
    obs_ptr[p + 1] = o;
    for (char c : m->mLog)
      if (l < log_cap) log[l++] = c;
    log_ptr[p + 1] = l;
  }
  for (size_t k = 0; k < s->kfs.size(); k++) { target_mark[k] = (int64_t)s->kfs[k]->mFuseTargetForKF; conn_updates[k] = s->kfs[k]->mnConnectionUpdates; }
}

extern "C" void fn_shim_stats(unsigned long long* c) { ccm_b200_fuse_neighbours_stats(&c[0], &c[1]); }

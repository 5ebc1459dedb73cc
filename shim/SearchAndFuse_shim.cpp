// SearchAndFuse_shim.cpp — LoopFinder::SearchAndFuse / MapMerger::SearchAndFuse over one ccm_search_and_fuse call (INTEGRATION.md §4i).
//
// What stays the reference's own, in its order: the walk over CorrectedPosesMap, spAlreadyFound = pKF->GetMapPoints() taken at each
// keyframe, the live isBad() skip, Fuse(Scw)'s surgery (cslam/src/ORBmatcher.cpp:1103-1118) and the replacements of the member body.
// What the library does in one call: the prelude and window search of every (keyframe, loop point) pair, over the split of each Scw
// (Sim3Split_shim.h) and the points as they are at the start.
//
// Why one call before the walk is enough (DESIGN.md §5): of the state the member changes, a search reads only the point's descriptor
// (Replace and ReplaceAndLock end with ComputeDistinctiveDescriptors on the survivor); isBad() and GetMapPoints() are checked here live.
// Before each keyframe's walk, the points it will search whose descriptor no longer equals the bytes passed in are searched again,
// all in one ccm_search_and_fuse_host call for that keyframe, and counted as repairs.
#include "SearchAndFuse_shim.h"

#include <atomic>
#include <cstring>
#include <memory>
#include <set>
#include <vector>

#include <cslam/Converter.h>
#include <cslam/KeyFrame.h>
#include <cslam/MapPoint.h>
#include <cslam/estd.h>

#include "Sim3Split_shim.h"
#include "ccm_b200.h"

namespace cslam {

namespace {
std::atomic<unsigned long long> g_calls(0), g_repairs(0);

typedef boost::shared_ptr<KeyFrame> kfptr;
typedef boost::shared_ptr<MapPoint> mpptr;

// mfMaxDistance / mfMinDistance are protected in MapPoint; PredictScale needs the former itself, not GetMaxDistanceInvariance()
struct DistancePeek : MapPoint {
  static float MapPoint::*max_d() { return &DistancePeek::mfMaxDistance; }
  static float MapPoint::*min_d() { return &DistancePeek::mfMinDistance; }
};

struct FlatKf {   // keeps the arrays a ccm_fuse_kf points to; the camera is Fuse(Scw)'s split of Scw
  std::vector<float> xy, angle;
  std::vector<int32_t> octave;
  ccm_fuse_kf k;
  FlatKf(const kfptr& pKF, const cv::Mat& Scw) {
    const int N = pKF->N;
    xy.resize(2 * (size_t)N); angle.resize(N); octave.resize(N);
    for (int i = 0; i < N; i++) {
      const cv::KeyPoint& kp = pKF->mvKeysUn[i];
      xy[2 * i] = kp.pt.x; xy[2 * i + 1] = kp.pt.y; angle[i] = kp.angle; octave[i] = kp.octave;
    }
    std::memset(&k, 0, sizeof k);
    k.grid = ccm_feature_grid{N, pKF->mDescriptors.ptr(), xy.data(), octave.data(), angle.data(), (float)pKF->mnMinX, (float)pKF->mnMinY,
                              (float)pKF->mnMaxX, (float)pKF->mnMaxY, pKF->mfGridElementWidthInv, pKF->mfGridElementHeightInv,
                              pKF->mnGridCols, pKF->mnGridRows};
    const Sim3Split s = split_sim3(Scw);
    for (int r = 0; r < 3; r++) {
      for (int c = 0; c < 3; c++) k.Tcw[4 * r + c] = s.Rcw.at<float>(r, c);
      k.Tcw[4 * r + 3] = s.tcw.at<float>(r);
      k.Ow[r] = s.Ow.at<float>(r);
    }
    k.fx = pKF->fx; k.fy = pKF->fy; k.cx = pKF->cx; k.cy = pKF->cy;
    k.scale_factors = pKF->mvScaleFactors.data(); k.inv_level_sigma2 = nullptr;   // Fuse(Scw) has no chi-square gate
    k.nlevels = pKF->mnScaleLevels; k.log_scale_factor = pKF->mfLogScaleFactor;
  }
};

// one row per entry of a point list, its state as the library reads it (skip = isBad())
struct FlatPoints {
  std::vector<float> pos, normal, max_d, min_d;
  std::vector<uint8_t> desc, skip;
  void add(const mpptr& pMP) {
    const cv::Mat P = pMP->GetWorldPos(), Nv = pMP->GetNormal(), D = pMP->GetDescriptor();
    for (int k = 0; k < 3; k++) { pos.push_back(P.at<float>(k)); normal.push_back(Nv.at<float>(k)); }
    max_d.push_back((*pMP).*DistancePeek::max_d()); min_d.push_back((*pMP).*DistancePeek::min_d());
    desc.insert(desc.end(), D.ptr(), D.ptr() + 32);
    skip.push_back(pMP->isBad());
  }
  ccm_fuse_points c() const {
    return ccm_fuse_points{(int32_t)skip.size(), pos.data(), normal.data(), max_d.data(), min_d.data(), desc.data(), skip.data()};
  }
  bool same_descriptor(size_t r, const mpptr& pMP) const {
    const cv::Mat D = pMP->GetDescriptor();
    return std::memcmp(D.ptr(), &desc[32 * r], 32) == 0;
  }
};

inline void must(int rc) { if (rc != CCM_OK) throw estd::infrastructure_ex(); }
}  // namespace

void ccm_b200_search_and_fuse_stats(unsigned long long* calls, unsigned long long* repairs) {
  if (calls) *calls = g_calls.load();
  if (repairs) *repairs = g_repairs.load();
}

void ccm_b200_search_and_fuse(const Sim3CorrectionMap& CorrectedPosesMap, const std::vector<mpptr>& vpLoopMapPoints, bool merge) {
  const size_t nLP = vpLoopMapPoints.size();
  std::vector<kfptr> kfs;
  std::vector<std::unique_ptr<FlatKf> > flat;
  std::vector<ccm_fuse_kf> K;
  for (Sim3CorrectionMap::const_iterator mit = CorrectedPosesMap.begin(), mend = CorrectedPosesMap.end(); mit != mend; mit++) {
    kfs.push_back(mit->first);
    flat.emplace_back(new FlatKf(mit->first, Converter::toCvMat(mit->second)));
    K.push_back(flat.back()->k);
  }
  FlatPoints P;
  for (const mpptr& pMP : vpLoopMapPoints) P.add(pMP);
  const ccm_fuse_points pts = P.c();
  std::vector<int32_t> best(kfs.size() * nLP, -1);
  g_calls++;
  must(ccm_search_and_fuse(K.data(), (int32_t)kfs.size(), &pts, best.data(), nullptr));

  for (size_t k = 0; k < kfs.size(); k++) {
    const kfptr& pKF = kfs[k];
    int32_t* found = best.data() + k * nLP;
    // Fuse(pKF, cvScw, vpLoopMapPoints, 4, vpReplacePoints), ORBmatcher.cpp:995-1122
    const std::set<mpptr> spAlreadyFound = pKF->GetMapPoints();
    std::vector<size_t> stale;
    for (size_t i = 0; i < nLP; i++) {
      const mpptr& pMP = vpLoopMapPoints[i];
      if (!pMP->isBad() && !spAlreadyFound.count(pMP) && !P.same_descriptor(i, pMP)) stale.push_back(i);
    }
    if (!stale.empty()) {   // the points an earlier keyframe's replacement changed: searched again over their state now
      FlatPoints S;
      for (size_t i : stale) S.add(vpLoopMapPoints[i]);
      const ccm_fuse_points sp = S.c();
      std::vector<int32_t> again(stale.size(), -1);
      must(ccm_search_and_fuse_host(&K[k], 1, &sp, again.data(), nullptr));
      for (size_t s = 0; s < stale.size(); s++) found[stale[s]] = again[s];
      g_repairs += stale.size();
    }
    std::vector<mpptr> vpReplacePoints(nLP, nullptr);
    for (size_t iMP = 0; iMP < nLP; iMP++) {
      mpptr pMP = vpLoopMapPoints[iMP];
      if (pMP->isBad() || spAlreadyFound.count(pMP)) continue;
      const int bestIdx = found[iMP];
      if (bestIdx < 0) continue;
      mpptr pMPinKF = pKF->GetMapPoint(bestIdx);
      if(pMPinKF)
      {
          if(!pMPinKF->isBad())
              vpReplacePoints[iMP] = pMPinKF;
      }
      else
      {
          pMP->AddObservation(pKF,bestIdx);
          pKF->AddMapPoint(pMP,bestIdx);
      }
    }
    // the member body after Fuse (LoopFinder.cpp:724-732, MapMerger.cpp:588-596)
    for (size_t i = 0; i < nLP; i++) {
      mpptr pRep = vpReplacePoints[i];
      if (pRep) {
        if (merge) pRep->ReplaceAndLock(vpLoopMapPoints[i]);
        else pRep->Replace(vpLoopMapPoints[i], true);
      }
    }
  }
}

}  // namespace cslam

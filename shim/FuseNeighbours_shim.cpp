// FuseNeighbours_shim.cpp — LocalMapping::SearchInNeighbors (cslam/src/Mapping.cpp:471-547) over one ccm_fuse_neighbours call.
//
// Replace the member's body in Mapping.cpp by this translation unit (INTEGRATION.md §4g).  What stays the reference's own, verbatim:
// the target list with its mFuseTargetForKF marks, the candidate list with its mFuseCandidateForKF marks, the skips of Fuse
// (cslam/src/ORBmatcher.cpp:872-882), the surgery that follows each search (:955-990), and the tail that refreshes the current points
// and the covisibility graph (:531-546).  What the library does in one call: the prelude and window search of every Fuse pair.
//
// Why one call before the walk is enough (DESIGN.md §5): the search of a pair reads, of all the state the surgery changes, only
// isBad(), IsInKeyFrame() and the point's descriptor (MapPoint::Replace ends with ComputeDistinctiveDescriptors on the survivor).  The
// first two are checked here live, in the reference's order.  A pair whose point's descriptor no longer equals the bytes uploaded is
// searched again on the host (ccm_fuse_neighbours_host for that one pair: the same prelude and window search) and counted as a repair.
// The backward candidates are built after the forward walk, as the reference builds them; every one of them is a target's point at
// the start of the member (a point the forward walk adds to a target is a current point, which the backward Fuse skips), so the call
// searches every target's point at the start against the current keyframe, and a candidate outside that set is searched on the host.
#include "FuseNeighbours_shim.h"

#include <atomic>
#include <cstring>
#include <map>
#include <vector>

#include <cslam/Mapping.h>
#include <cslam/estd.h>

#include "MapPointDescriptor_shim.h"
#include "ccm_b200.h"

namespace cslam {

namespace {
std::atomic<unsigned long long> g_calls(0), g_repairs(0);

typedef LocalMapping::kfptr kfptr;
typedef LocalMapping::mpptr mpptr;

// mfMaxDistance / mfMinDistance are protected in MapPoint; PredictScale needs the former itself, not GetMaxDistanceInvariance()
struct DistancePeek : MapPoint {
  static float MapPoint::*max_d() { return &DistancePeek::mfMaxDistance; }
  static float MapPoint::*min_d() { return &DistancePeek::mfMinDistance; }
};

struct FlatKf {   // keeps the arrays a ccm_fuse_kf points to
  std::vector<float> xy, angle;
  std::vector<int32_t> octave;
  ccm_fuse_kf k;
  explicit FlatKf(const kfptr& pKF) {
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
    const cv::Mat R = pKF->GetRotation(), t = pKF->GetTranslation(), O = pKF->GetCameraCenter();
    for (int r = 0; r < 3; r++) {
      for (int c = 0; c < 3; c++) k.Tcw[4 * r + c] = R.at<float>(r, c);
      k.Tcw[4 * r + 3] = t.at<float>(r);
      k.Ow[r] = O.at<float>(r);
    }
    k.fx = pKF->fx; k.fy = pKF->fy; k.cx = pKF->cx; k.cy = pKF->cy;
    k.scale_factors = pKF->mvScaleFactors.data(); k.inv_level_sigma2 = pKF->mvInvLevelSigma2.data();
    k.nlevels = pKF->mnScaleLevels; k.log_scale_factor = pKF->mfLogScaleFactor;
  }
};

// the point table: one row per distinct point, its state as the library reads it
struct FlatPoints {
  std::map<MapPoint*, int> row;
  std::vector<float> pos, normal, max_d, min_d;
  std::vector<uint8_t> desc, skip;
  int add(const mpptr& pMP) {
    if (!pMP) return -1;
    const auto it = row.find(pMP.get());
    if (it != row.end()) return it->second;
    const int r = (int)skip.size();
    row[pMP.get()] = r;
    const cv::Mat P = pMP->GetWorldPos(), Nv = pMP->GetNormal(), D = pMP->GetDescriptor();
    for (int k = 0; k < 3; k++) { pos.push_back(P.at<float>(k)); normal.push_back(Nv.at<float>(k)); }
    max_d.push_back((*pMP).*DistancePeek::max_d()); min_d.push_back((*pMP).*DistancePeek::min_d());
    desc.insert(desc.end(), D.ptr(), D.ptr() + 32);
    skip.push_back(pMP->mbDoNotReplace || pMP->isBad());
    return r;
  }
  ccm_fuse_points c() const {
    return ccm_fuse_points{(int32_t)skip.size(), pos.data(), normal.data(), max_d.data(), min_d.data(), desc.data(), skip.data()};
  }
  bool same_descriptor(int r, const mpptr& pMP) const {
    const cv::Mat D = pMP->GetDescriptor();
    return std::memcmp(D.ptr(), &desc[32 * (size_t)r], 32) == 0;
  }
};

inline void must(int rc) { if (rc != CCM_OK) throw estd::infrastructure_ex(); }

// one pair on the host, over the point's current state: Fuse's prelude and window search into pKF
int repair(const kfptr& pKF, const mpptr& pMP) {
  g_repairs++;
  FlatKf K(pKF);
  FlatPoints P;
  P.add(pMP);
  const ccm_fuse_points pts = P.c();
  const std::vector<int32_t> none((size_t)pKF->N, -1);
  const int32_t cand = 0;
  int32_t best = -1;
  must(ccm_fuse_neighbours_host(&K.k, nullptr, 0, &pts, none.data(), &cand, 1, nullptr, &best, nullptr));
  return best;
}

// the surgery of Fuse(pKF, vpMapPoints) for one point and its best keypoint (cslam/src/ORBmatcher.cpp:955-990)
void fuse_one(const kfptr& pKF, const mpptr& pMP, int bestIdx) {
  mpptr pMPinKF = pKF->GetMapPoint(bestIdx);
  if(pMPinKF)
  {
      if(!pMPinKF->isBad() && !pMPinKF->mbDoNotReplace)
      {
          if(pMPinKF->Observations()>pMP->Observations())
              pMP->Replace(pMPinKF);
          else
              pMPinKF->Replace(pMP);
      }
  }
  else
  {
      pMP->AddObservation(pKF,bestIdx);
      pKF->AddMapPoint(pMP,bestIdx);
  }
}

// Fuse's skips (:872-882)
bool skipped(const mpptr& pMP, const kfptr& pKF) { return !pMP || pMP->isBad() || pMP->IsInKeyFrame(pKF) || pMP->mbDoNotReplace; }
}  // namespace

void ccm_b200_fuse_neighbours_stats(unsigned long long* calls, unsigned long long* repairs) {
  if (calls) *calls = g_calls.load();
  if (repairs) *repairs = g_repairs.load();
}

void LocalMapping::SearchInNeighbors()
{
    // Retrieve neighbor keyframes
    int nn=20;
    const std::vector<kfptr> vpNeighKFs = mpCurrentKeyFrame->GetBestCovisibilityKeyFrames(nn);
    std::vector<kfptr> vpTargetKFs;
    for(std::vector<kfptr>::const_iterator vit=vpNeighKFs.begin(), vend=vpNeighKFs.end(); vit!=vend; vit++)
    {
        kfptr pKFi = *vit;
        if(pKFi->isBad() || pKFi->mFuseTargetForKF == mpCurrentKeyFrame->mId)
            continue;
        vpTargetKFs.push_back(pKFi);
        pKFi->mFuseTargetForKF = mpCurrentKeyFrame->mId;

        // Extend to some second neighbors
        const std::vector<kfptr> vpSecondNeighKFs = pKFi->GetBestCovisibilityKeyFrames(5);
        for(std::vector<kfptr>::const_iterator vit2=vpSecondNeighKFs.begin(), vend2=vpSecondNeighKFs.end(); vit2!=vend2; vit2++)
        {
            kfptr pKFi2 = *vit2;
            if(pKFi2->isBad() || pKFi2->mFuseTargetForKF==mpCurrentKeyFrame->mId || pKFi2->mId==mpCurrentKeyFrame->mId)
                continue;
            vpTargetKFs.push_back(pKFi2);
        }
    }

    std::vector<mpptr> vpMapPointMatches = mpCurrentKeyFrame->GetMapPointMatches();

    // one upload: each distinct target once, the current slots' points, every target's point at the start as the backward superset
    std::map<KeyFrame*, int> targetRow;
    std::vector<FlatKf> vFlat;
    vFlat.reserve(vpTargetKFs.size() + 1);
    vFlat.emplace_back(mpCurrentKeyFrame);
    std::vector<ccm_fuse_kf> vTargets;
    for (const kfptr& pKF : vpTargetKFs)
        if (targetRow.emplace(pKF.get(), (int)vTargets.size()).second) {
            vFlat.emplace_back(pKF);
            vTargets.push_back(vFlat.back().k);
        }
    FlatPoints P;
    const int n = mpCurrentKeyFrame->N;
    std::vector<int32_t> curPoint(n);
    for (int i = 0; i < n; i++) curPoint[i] = P.add(vpMapPointMatches[i]);
    std::vector<int32_t> super;
    std::map<MapPoint*, int> superAt;
    for (const kfptr& pKF : vpTargetKFs)
        for (const mpptr& pMP : pKF->GetMapPointMatches())
            if (pMP && superAt.emplace(pMP.get(), (int)super.size()).second) super.push_back(P.add(pMP));
    const ccm_fuse_points pts = P.c();
    std::vector<int32_t> fwd((size_t)n * vTargets.size() + 1), bwd(super.size() + 1);
    g_calls++;
    must(ccm_fuse_neighbours(&vFlat[0].k, vTargets.data(), (int32_t)vTargets.size(), &pts, curPoint.data(), super.data(),
                             (int32_t)super.size(), fwd.data(), bwd.data(), nullptr));

    // Search matches by projection from current KF in target KFs
    for(std::vector<kfptr>::iterator vit=vpTargetKFs.begin(), vend=vpTargetKFs.end(); vit!=vend; vit++)
    {
        kfptr pKFi = *vit;
        const int t = targetRow[pKFi.get()];
        for (int i = 0; i < n; i++)
        {
            mpptr pMP = vpMapPointMatches[i];
            if (skipped(pMP, pKFi))
                continue;
            const int best = P.same_descriptor(curPoint[i], pMP) ? fwd[(size_t)t * n + i] : repair(pKFi, pMP);
            if (best >= 0)
                fuse_one(pKFi, pMP, best);
        }
    }

    // Search matches by projection from target KFs in current KF
    std::vector<mpptr> vpFuseCandidates;
    vpFuseCandidates.reserve(vpTargetKFs.size()*vpMapPointMatches.size());

    for(std::vector<kfptr>::iterator vitKF=vpTargetKFs.begin(), vendKF=vpTargetKFs.end(); vitKF!=vendKF; vitKF++)
    {
        kfptr pKFi = *vitKF;

        std::vector<mpptr> vpMapPointsKFi = pKFi->GetMapPointMatches();

        for(std::vector<mpptr>::iterator vitMP=vpMapPointsKFi.begin(), vendMP=vpMapPointsKFi.end(); vitMP!=vendMP; vitMP++)
        {
            mpptr pMP = *vitMP;
            if(!pMP)
                continue;
            if(pMP->isBad() || pMP->mFuseCandidateForKF == mpCurrentKeyFrame->mId)
                continue;
            pMP->mFuseCandidateForKF = mpCurrentKeyFrame->mId;
            vpFuseCandidates.push_back(pMP);
        }
    }

    for (const mpptr& pMP : vpFuseCandidates)
    {
        if (skipped(pMP, mpCurrentKeyFrame))
            continue;
        const auto it = superAt.find(pMP.get());
        const bool uploaded = it != superAt.end() && P.same_descriptor(super[it->second], pMP);
        const int best = uploaded ? bwd[it->second] : repair(mpCurrentKeyFrame, pMP);
        if (best >= 0)
            fuse_one(mpCurrentKeyFrame, pMP, best);
    }

    // Update points: both members for every current point in one batch each, parked for the loop below (INTEGRATION.md §4d)
    vpMapPointMatches = mpCurrentKeyFrame->GetMapPointMatches();
    std::vector<mpptr> vpUpdate;
    for (const mpptr& pMP : vpMapPointMatches)
        if (pMP && !pMP->isBad())
            vpUpdate.push_back(pMP);
    ccm_b200_prepare_point_updates(vpUpdate);
    ParkedDescriptorsGuard parked;
    for(size_t i=0, iend=vpMapPointMatches.size(); i<iend; i++)
    {
        mpptr pMP=vpMapPointMatches[i];
        if(pMP)
        {
            if(!pMP->isBad())
            {
                pMP->ComputeDistinctiveDescriptors();
                pMP->UpdateNormalAndDepth();
            }
        }
    }

    // Update connections in covisibility graph
    mpCurrentKeyFrame->UpdateConnections();
}

}  // namespace cslam

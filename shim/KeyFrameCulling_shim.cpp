// KeyFrameCulling_shim.cpp — LocalMapping::KeyFrameCullingV3 (cslam/src/Mapping.cpp:771-863) over one ccm_keyframe_culling call.
//
// Replace the member's body in Mapping.cpp by this translation unit (INTEGRATION.md §4j).  What stays the reference's own, verbatim: the
// random pick with its second try, the mlpRecentAddedKFs checks, mspKFsCheckedForCulling, the skips of mId.first 0 / 1, and the
// SetBadFlag / ++mCulledKfs of each culled keyframe, in covisibility order.  What the library does in one call: every candidate's
// nMPs / nRedundant count and verdict, earlier culls included (include/ccm_b200.h: the counts over the state at the start, then a host
// settle that applies each effective cull and counts again the candidates it reached).  So the SetBadFlag calls below, made in the
// reference's order, leave the map as the reference leaves it.
#include "KeyFrameCulling_shim.h"

#include <algorithm>
#include <atomic>
#include <map>
#include <vector>

#include <cslam/Mapping.h>
#include <cslam/estd.h>

#include "ccm_b200.h"

namespace cslam {

namespace {
std::atomic<unsigned long long> g_calls(0), g_settled(0);

typedef LocalMapping::kfptr kfptr;
typedef LocalMapping::mpptr mpptr;

// mbNotErase is protected in KeyFrame; SetBadFlag's server branch reads it
struct NotErasePeek : KeyFrame {
  static bool KeyFrame::*flag() { return &NotErasePeek::mbNotErase; }
};

inline void must(int rc) { if (rc != CCM_OK) throw estd::infrastructure_ex(); }

// the flat arrays of ccm_keyframe_culling for the candidates, in order: keyframe rows (candidates and observers), point rows
struct Flat {
  std::map<KeyFrame*, int32_t> kfRow;
  std::map<MapPoint*, int32_t> mpRow;
  std::vector<uint8_t> kf_bad, cand_not_erase, mp_bad;
  std::vector<int32_t> cand_kf, slot_mp, slot_octave, mp_nobs, mp_ref, obs_kf, obs_octave;
  std::vector<int64_t> slot_ptr{0}, obs_ptr{0};
  std::vector<mpptr> points;

  int32_t kf(const kfptr& pKF) {
    const auto it = kfRow.find(pKF.get());
    if (it != kfRow.end()) return it->second;
    const int32_t r = (int32_t)kf_bad.size();
    kfRow[pKF.get()] = r;
    kf_bad.push_back(pKF->isBad());
    return r;
  }
  int32_t mp(const mpptr& pMP) {
    if (!pMP) return -1;
    const auto it = mpRow.find(pMP.get());
    if (it != mpRow.end()) return it->second;
    const int32_t r = (int32_t)points.size();
    mpRow[pMP.get()] = r;
    points.push_back(pMP);
    return r;
  }
  void candidate(const kfptr& pKF) {
    cand_kf.push_back(kf(pKF));
    cand_not_erase.push_back((*pKF).*NotErasePeek::flag());
    const std::vector<mpptr> vpMapPoints = pKF->GetMapPointMatches();
    for (size_t i = 0; i < vpMapPoints.size(); i++) {
      slot_mp.push_back(mp(vpMapPoints[i]));
      slot_octave.push_back(pKF->mvKeysUn[i].octave);
    }
    slot_ptr.push_back((int64_t)slot_mp.size());
  }
  // each point's state, after every candidate is in (observers get rows as they appear)
  void finish() {
    for (size_t r = 0; r < points.size(); r++) {
      const mpptr& pMP = points[r];
      const bool bad = pMP->isBad();
      mp_bad.push_back(bad);
      mp_nobs.push_back(pMP->Observations());
      const kfptr pRef = pMP->GetReferenceKeyFrame();
      mp_ref.push_back(pRef ? kf(pRef) : -1);
      if (!bad) {
        const auto observations = pMP->GetObservations();
        for (const auto& o : observations) {
          obs_kf.push_back(kf(o.first));
          obs_octave.push_back(o.first->mvKeysUn[o.second].octave);
        }
      }
      obs_ptr.push_back((int64_t)obs_kf.size());
    }
  }
};
}  // namespace

void ccm_b200_keyframe_culling_stats(unsigned long long* calls, unsigned long long* settled) {
  if (calls) *calls = g_calls.load();
  if (settled) *settled = g_settled.load();
}

void LocalMapping::KeyFrameCullingV3()
{
    //This version: randomly pick a KF and check for redundancy
    kfptr pKFc = mpMap->GetRandKfPtr();
    if(!pKFc)
        return; //safety check

    //we don't check KFs in mlpRecentAddedKFs, since the neighbors will probably not be allowed for culling.
    std::list<kfptr>::iterator lit1 = std::find(mlpRecentAddedKFs.begin(),mlpRecentAddedKFs.end(),pKFc);
    if(lit1 != mlpRecentAddedKFs.end())
    {
        //give it a second try -- if not successful return to not spend ages in this method.

        pKFc = mpMap->GetRandKfPtr();
            if(!pKFc)
                return; //safety check

        lit1 = std::find(mlpRecentAddedKFs.begin(),mlpRecentAddedKFs.end(),pKFc);
        if(lit1 != mlpRecentAddedKFs.end())
            return;
    }

    if(mspKFsCheckedForCulling.count(pKFc))
        return;
    else
        mspKFsCheckedForCulling.insert(pKFc);

    std::vector<kfptr> vpLocalKeyFrames = pKFc->GetVectorCovisibleKeyFrames();

    // the candidates, as the member's loop skips them (:799-805), flattened in covisibility order
    std::vector<kfptr> vpCandidates;
    Flat F;
    for(std::vector<kfptr>::iterator vit=vpLocalKeyFrames.begin(), vend=vpLocalKeyFrames.end(); vit!=vend; vit++)
    {
        kfptr pKF = *vit;
        if(pKF->mId.first==0 || pKF->mId.first==1)
            continue;
        std::list<kfptr>::iterator lit2 = std::find(mlpRecentAddedKFs.begin(),mlpRecentAddedKFs.end(),pKF);
        if(lit2 != mlpRecentAddedKFs.end())
            continue;
        vpCandidates.push_back(pKF);
        F.candidate(pKF);
    }
    if (vpCandidates.empty())
        return;
    F.finish();

    const int32_t n_c = (int32_t)vpCandidates.size();
    std::vector<uint8_t> cull(n_c);
    std::vector<int32_t> n_mps(n_c), n_red(n_c);
    int32_t n_settled = 0;
    const int thObs=3;
    g_calls++;
    must(ccm_keyframe_culling((int32_t)F.kf_bad.size(), F.kf_bad.data(), n_c, F.cand_kf.data(), F.cand_not_erase.data(), F.slot_ptr.data(),
                              F.slot_mp.data(), F.slot_octave.data(), (int32_t)F.points.size(), F.mp_bad.data(), F.mp_nobs.data(),
                              F.mp_ref.data(), F.obs_ptr.data(), F.obs_kf.data(), F.obs_octave.data(), thObs,
                              params::mapping::mfRedundancyThres, cull.data(), n_mps.data(), n_red.data(), &n_settled));
    g_settled += (unsigned long long)n_settled;

    for (int32_t c = 0; c < n_c; c++)
    {
        if (cull[c])
        {
            vpCandidates[c]->SetBadFlag();
            ++mCulledKfs;
        }
    }
}

}  // namespace cslam

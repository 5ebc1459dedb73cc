// ref_keyframe_culling_wrap.cpp — a literal restatement of LocalMapping::KeyFrameCullingV3 (cslam/src/Mapping.cpp:771-863) and of the
// paths its SetBadFlag calls reach on the server — KeyFrame::SetBadFlag (cslam/src/KeyFrame.cpp:936-990, up to the connection and
// spanning-tree surgery, which the member does not read), MapPoint::EraseObservation (cslam/src/MapPoint.cpp:442-509) and
// MapPoint::SetBadFlag (:520-548, up to the map bookkeeping) — over the stand-ins of ref_stub_kc/, next to shim/KeyFrameCulling_shim.cpp
// on the same stand-ins (TEST INFRASTRUCTURE).
//
// kc_scene_create builds keyframes and points from flat arrays; kc_run runs mode 0 (the restatement) or 1 (the shim); kc_members reads
// back what the member left.
#include <algorithm>
#include <cstdint>
#include <iostream>
#include <vector>

#include <cslam/Mapping.h>

#include "../shim/KeyFrameCulling_shim.h"

namespace cslam {

namespace params { namespace mapping { fptype mfRedundancyThres = 0.98; } }

void KeyFrame::SetBadFlag(bool bSuppressMapAction, bool bNoParent)
{
    {
        if(mbBad)
            return;
    }
    {
        if(mId.first==0)
            return;
        else if(mbNotErase)
        {
            mbToBeErased = true;
            return;
        }
    }
    for(size_t i=0; i<mvpMapPoints.size(); i++)
    {
        if(mvpMapPoints[i])
        {
                mpptr pMPx = mvpMapPoints[i];
                pMPx->EraseObservation(this->shared_from_this(),false,true);
        }
    }
    mbBad = true;
}

void MapPoint::EraseObservation(kfptr pKF, bool bLock, bool bSuppressMapAction)
{
    bool bBad=false;
    {
        if(mObservations.count(pKF))
        {
            nObs--;

            mObservations.erase(pKF);

            if(mpRefKF==pKF)
            {
                if(nObs > 0)
                {
                    mpRefKF = nullptr;
                    std::map<kfptr,size_t,KfById>::const_iterator mitRef = mObservations.begin();
                    while(!mpRefKF)
                    {
                        if(mitRef == mObservations.end()) break;
                        if(!(mitRef->first->isBad()))
                            mpRefKF=mitRef->first;
                        else
                            ++mitRef;
                    }
                }
                else
                    mpRefKF=nullptr;
            }

            // If only 2 observations or less, discard point
            if(nObs<=2)
                bBad=true;
        }
    }

    if(bBad)
        SetBadFlag(bSuppressMapAction);

    if(!mpRefKF)
    {
        if(!mbBad)
        {
            SetBadFlag(bSuppressMapAction);
        }
    }
}

void MapPoint::SetBadFlag(bool bSuppressMapAction)
{
    {
        if(mbBad)
            return;
    }
    std::map<kfptr,size_t,KfById> obs;
    {
        mbBad=true;
        obs = mObservations;
        mObservations.clear();
    }
    for(std::map<kfptr,size_t,KfById>::iterator mit=obs.begin(), mend=obs.end(); mit!=mend; mit++)
    {
        kfptr pKF = mit->first;
        pKF->EraseMapPointMatch(mit->second);
    }
}

struct KcScene {
  typedef LocalMapping::kfptr kfptr;
  typedef LocalMapping::mpptr mpptr;
  std::vector<kfptr> kfs;
  std::vector<mpptr> pts;
  boost::shared_ptr<Map> map;
  LocalMapping lm;

  static void* create(int32_t K, const uint8_t* kf_bad, const uint8_t* kf_not_erase, const int64_t* kf_id, const int64_t* slot_ptr,
                                 const int32_t* slot_mp, const int32_t* slot_octave, int32_t P, const uint8_t* mp_bad, const int32_t* nobs,
                                 const int32_t* ref, const int64_t* obs_ptr, const int32_t* obs_kf, const int32_t* obs_idx, int32_t query,
                                 const int32_t* covis, int32_t n_covis, const int32_t* recent, int32_t n_recent, const int32_t* picks,
                                 int32_t n_picks, const int32_t* checked, int32_t n_checked);
  static void members(void* h, uint8_t* kf_bad, uint8_t* to_be_erased, int32_t* slots, uint8_t* mp_bad, int32_t* nobs, int32_t* ref,
                           int64_t* obs_ptr, int32_t* obs, int64_t* culled, uint8_t* checked);
  static void destroy(void* h);
  void shim() { lm.KeyFrameCullingV3(); }

  // the member as cslam/src/Mapping.cpp:771-863 writes it
  void reference()
  {
    LocalMapping* self = &lm;
    std::list<kfptr>& mlpRecentAddedKFs = self->mlpRecentAddedKFs;
    std::set<kfptr>& mspKFsCheckedForCulling = self->mspKFsCheckedForCulling;
    size_t& mCulledKfs = self->mCulledKfs;
    boost::shared_ptr<Map>& mpMap = self->mpMap;

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

    for(std::vector<kfptr>::iterator vit=vpLocalKeyFrames.begin(), vend=vpLocalKeyFrames.end(); vit!=vend; vit++)
    {
        kfptr pKF = *vit;
        if(pKF->mId.first==0 || pKF->mId.first==1)
            continue;

        std::list<kfptr>::iterator lit2 = std::find(mlpRecentAddedKFs.begin(),mlpRecentAddedKFs.end(),pKF);
        if(lit2 != mlpRecentAddedKFs.end())
            continue;
        const std::vector<mpptr> vpMapPoints = pKF->GetMapPointMatches();

        const int thObs=3;
        int nRedundantObservations=0;
        int nMPs=0;
        for(size_t i=0, iend=vpMapPoints.size(); i<iend; i++)
        {
            mpptr pMP = vpMapPoints[i];
            if(pMP)
            {
                if(!pMP->isBad())
                {
                    nMPs++;
                    if(pMP->Observations()>thObs)
                    {
                        const int &scaleLevel = pKF->mvKeysUn[i].octave;
                        const std::map<kfptr, size_t, KfById> observations = pMP->GetObservations();
                        int nObs=0;
                        for(std::map<kfptr, size_t, KfById>::const_iterator mit=observations.begin(), mend=observations.end(); mit!=mend; mit++)
                        {
                            kfptr pKFi = mit->first;

                            if(pKFi->isBad()) continue;

                            if(pKFi==pKF)
                                continue;
                            const int &scaleLeveli = pKFi->mvKeysUn[mit->second].octave;

                            if(scaleLeveli<=scaleLevel+1)
                            {
                                nObs++;
                                if(nObs>=thObs)
                                    break;
                            }
                        }
                        if(nObs>=thObs)
                        {
                            nRedundantObservations++;
                        }
                    }
                }
            }
        }

        if(nRedundantObservations>params::mapping::mfRedundancyThres*nMPs)
        {
            pKF->SetBadFlag();
            ++mCulledKfs;
        }
    }
  }
};

}  // namespace cslam

using namespace cslam;

void* KcScene::create(int32_t K, const uint8_t* kf_bad, const uint8_t* kf_not_erase, const int64_t* kf_id, const int64_t* slot_ptr,
                                 const int32_t* slot_mp, const int32_t* slot_octave, int32_t P, const uint8_t* mp_bad, const int32_t* nobs,
                                 const int32_t* ref, const int64_t* obs_ptr, const int32_t* obs_kf, const int32_t* obs_idx, int32_t query,
                                 const int32_t* covis, int32_t n_covis, const int32_t* recent, int32_t n_recent, const int32_t* picks,
                                 int32_t n_picks, const int32_t* checked, int32_t n_checked) {
  KcScene* s = new KcScene;
  for (int32_t k = 0; k < K; k++) {
    KcScene::kfptr f(new KeyFrame);
    f->mId = idpair((size_t)kf_id[k], 0);
    f->mbBad = kf_bad[k]; f->mbNotErase = kf_not_erase[k];
    f->mvKeysUn.resize((size_t)(slot_ptr[k + 1] - slot_ptr[k]));
    for (int64_t j = slot_ptr[k]; j < slot_ptr[k + 1]; j++) f->mvKeysUn[j - slot_ptr[k]].octave = slot_octave[j];
    s->kfs.push_back(f);
  }
  for (int32_t p = 0; p < P; p++) {
    KcScene::mpptr m(new MapPoint);
    m->mbBad = mp_bad[p]; m->nObs = nobs[p];
    if (ref[p] >= 0) m->mpRefKF = s->kfs[ref[p]];
    for (int64_t j = obs_ptr[p]; j < obs_ptr[p + 1]; j++) m->mObservations[s->kfs[obs_kf[j]]] = (size_t)obs_idx[j];
    s->pts.push_back(m);
  }
  for (int32_t k = 0; k < K; k++)
    for (int64_t j = slot_ptr[k]; j < slot_ptr[k + 1]; j++)
      s->kfs[k]->mvpMapPoints.push_back(slot_mp[j] >= 0 ? s->pts[slot_mp[j]] : KcScene::mpptr());
  for (int32_t i = 0; i < n_covis; i++) s->kfs[query]->mvpOrderedConnectedKeyFrames.push_back(s->kfs[covis[i]]);
  s->map.reset(new Map);
  for (int32_t i = 0; i < n_picks; i++) s->map->mvScript.push_back(picks[i] >= 0 ? s->kfs[picks[i]] : KcScene::kfptr());
  s->lm.mpMap = s->map;
  for (int32_t i = 0; i < n_recent; i++) s->lm.mlpRecentAddedKFs.push_back(s->kfs[recent[i]]);
  for (int32_t i = 0; i < n_checked; i++) s->lm.mspKFsCheckedForCulling.insert(s->kfs[checked[i]]);
  return s;
}

void KcScene::destroy(void* h) {
  KcScene* s = static_cast<KcScene*>(h);
  for (auto& p : s->pts) { p->mObservations.clear(); p->mpRefKF.reset(); }
  for (auto& k : s->kfs) { k->mvpMapPoints.clear(); k->mvpOrderedConnectedKeyFrames.clear(); }
  delete s;
}

extern "C" void* kc_scene_create(int32_t K, const uint8_t* kf_bad, const uint8_t* kf_not_erase, const int64_t* kf_id, const int64_t* slot_ptr,
                                 const int32_t* slot_mp, const int32_t* slot_octave, int32_t P, const uint8_t* mp_bad, const int32_t* nobs,
                                 const int32_t* ref, const int64_t* obs_ptr, const int32_t* obs_kf, const int32_t* obs_idx, int32_t query,
                                 const int32_t* covis, int32_t n_covis, const int32_t* recent, int32_t n_recent, const int32_t* picks,
                                 int32_t n_picks, const int32_t* checked, int32_t n_checked) {
  return KcScene::create(K, kf_bad, kf_not_erase, kf_id, slot_ptr, slot_mp, slot_octave, P, mp_bad, nobs, ref, obs_ptr, obs_kf, obs_idx, query, covis, n_covis, recent, n_recent, picks, n_picks, checked, n_checked);
}

extern "C" void kc_scene_destroy(void* h) { KcScene::destroy(h); }

extern "C" void kc_members(void* h, uint8_t* kf_bad, uint8_t* to_be_erased, int32_t* slots, uint8_t* mp_bad, int32_t* nobs, int32_t* ref,
                           int64_t* obs_ptr, int32_t* obs, int64_t* culled, uint8_t* checked) {
  KcScene::members(h, kf_bad, to_be_erased, slots, mp_bad, nobs, ref, obs_ptr, obs, culled, checked);
}

extern "C" int kc_run(void* h, int mode) {
  KcScene* s = static_cast<KcScene*>(h);
  try {
    if (mode == 0) s->reference();
    else s->shim();
  } catch (const std::exception& e) {
    std::cerr << "kc_run: " << e.what() << std::endl;
    return 1;
  }
  return 0;
}

void KcScene::members(void* h, uint8_t* kf_bad, uint8_t* to_be_erased, int32_t* slots, uint8_t* mp_bad, int32_t* nobs, int32_t* ref,
                           int64_t* obs_ptr, int32_t* obs, int64_t* culled, uint8_t* checked) {
  KcScene* s = static_cast<KcScene*>(h);
  std::map<KeyFrame*, int32_t> kr;
  std::map<MapPoint*, int32_t> pr;
  for (size_t k = 0; k < s->kfs.size(); k++) kr[s->kfs[k].get()] = (int32_t)k;
  for (size_t p = 0; p < s->pts.size(); p++) pr[s->pts[p].get()] = (int32_t)p;
  int64_t at = 0;
  for (size_t k = 0; k < s->kfs.size(); k++) {
    const KcScene::kfptr& f = s->kfs[k];
    kf_bad[k] = f->mbBad; to_be_erased[k] = f->mbToBeErased; checked[k] = s->lm.mspKFsCheckedForCulling.count(f) > 0;
    for (const auto& m : f->mvpMapPoints) slots[at++] = m ? pr[m.get()] : -1;
  }
  obs_ptr[0] = 0;
  for (size_t p = 0; p < s->pts.size(); p++) {
    const KcScene::mpptr& m = s->pts[p];
    mp_bad[p] = m->mbBad; nobs[p] = m->nObs; ref[p] = m->mpRefKF ? kr[m->mpRefKF.get()] : -1;
    int64_t n = obs_ptr[p];
    for (const auto& o : m->mObservations) { obs[2 * n] = kr[o.first.get()]; obs[2 * n + 1] = (int32_t)o.second; n++; }
    obs_ptr[p + 1] = n;
  }
  *culled = (int64_t)s->lm.mCulledKfs;
}

extern "C" void kc_set_threshold(double t) { params::mapping::mfRedundancyThres = t; }

extern "C" void kc_shim_stats(unsigned long long* c) { ccm_b200_keyframe_culling_stats(&c[0], &c[1]); }

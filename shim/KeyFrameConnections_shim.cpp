// KeyFrameConnections_shim.cpp — reference-side translation unit for KeyFrame::UpdateConnections (cslam/src/KeyFrame.cpp:629-852).
//
// The member is deleted from KeyFrame.cpp and defined here.  Only its first part changes: how KFcounter, the number of this
// keyframe's map points each other keyframe observes, is filled.
//   * batched: a loop over many keyframes calls ccm_b200_prepare_connections once before it starts.  It flattens the keyframes (each
//     distinct map point's observations copied once), makes one ccm_covisibility call on the GPU, and parks each keyframe's counter
//     per thread with a snapshot: its mvpMapPoints element for element, and each point's isBad() and Observations().  The member
//     uses the parked counter when its own copy of mvpMapPoints matches and every point still has the flag and count it had;
//   * single keyframe: every other caller (ingest, a keyframe whose snapshot went stale) flattens itself and counts through
//     ccm_covisibility_host, the same rule.
// Either way the counter arrives as (keyframe, weight) pairs in std::map<kfptr,int>'s own order: the shim ranks the keyframes with
// std::less<kfptr>, the map's comparator, so the order holds under any allocator and for any shared_ptr ordering.  The map is then
// filled by hinted inserts at its end.  Everything after the counter (the threshold, the AddConnection calls in map order, the
// ordered lists, the parent choice and the client's bSetBad path) is the reference's logic, unchanged in order and effect.
// In this repository it is compiled against the stand-in KeyFrame / MapPoint of oracle/ref_stub_cv and run next to a literal
// restatement of the reference body by tests/test_shim_covisibility.py.
#include <cslam/KeyFrame.h>
#include <cslam/MapPoint.h>
#include <cslam/estd.h>

#include <algorithm>
#include <atomic>
#include <functional>
#include <iostream>
#include <list>
#include <memory>
#include <unordered_map>
#include <utility>
#include <vector>

#include "KeyFrameConnections_shim.h"
#include "ccm_b200.h"

namespace cslam {

namespace {

typedef boost::shared_ptr<KeyFrame> kfptr;
typedef boost::shared_ptr<MapPoint> mpptr;

struct PointState {
  bool bad;
  int nobs;
};

// keyframes and points of one preparation, shared by the counters parked from it
struct Batch {
  std::vector<kfptr> rows;
  std::unordered_map<const MapPoint*, PointState> points;
};

struct Parked {
  std::shared_ptr<const Batch> batch;
  std::vector<const MapPoint*> mvp;                       // mvpMapPoints when counted
  std::vector<std::pair<int32_t, int32_t> > counter;      // (row, weight), std::map<kfptr,int>'s order
};

std::unordered_map<const KeyFrame*, Parked>& parked() {
  static thread_local std::unordered_map<const KeyFrame*, Parked> table;
  return table;
}

std::atomic<unsigned long long> g_hits(0), g_stale(0), g_host(0);

void check(int rc, const char* fn) {
  if (rc != CCM_OK) { std::cerr << "libccm_b200: " << fn << ": " << ccm_last_error() << std::endl; throw estd::infrastructure_ex(); }
}

// the flat arrays of include/ccm_b200.h's ccm_covisibility
struct Flat {
  std::shared_ptr<Batch> batch_state = std::make_shared<Batch>();
  std::unordered_map<const KeyFrame*, int32_t> row_of;
  std::map<idpair, uint64_t> id_code;
  std::vector<uint64_t> kf_id;
  std::vector<int32_t> batch, mp, obs;
  std::vector<int64_t> mptr{0}, optr{0};
  std::vector<uint8_t> mp_bad;
  std::unordered_map<const MapPoint*, int32_t> point_of;
  std::vector<int64_t> out_ptr;
  std::vector<int32_t> out_kf, out_w;

  int32_t add_kf(const kfptr& pKF) {
    std::unordered_map<const KeyFrame*, int32_t>::const_iterator it = row_of.find(pKF.get());
    if (it != row_of.end()) return it->second;
    const int32_t r = (int32_t)kf_id.size();
    row_of[pKF.get()] = r;
    batch_state->rows.push_back(pKF);
    std::map<idpair, uint64_t>::iterator c = id_code.insert(std::make_pair(pKF->mId, (uint64_t)id_code.size())).first;
    kf_id.push_back(c->second);
    return r;
  }
  // the count is read before the observations are copied: a later change moves it, except an observer replaced at equal count
  int32_t add_point(const mpptr& pMP) {
    std::unordered_map<const MapPoint*, int32_t>::const_iterator it = point_of.find(pMP.get());
    if (it != point_of.end()) return it->second;
    const int32_t p = (int32_t)mp_bad.size();
    point_of[pMP.get()] = p;
    PointState st;
    st.bad = pMP->isBad();
    st.nobs = pMP->Observations();
    batch_state->points[pMP.get()] = st;
    mp_bad.push_back(st.bad ? 1 : 0);
    if (!st.bad) {
      const std::map<kfptr, size_t> observations = pMP->GetObservations();
      for (std::map<kfptr, size_t>::const_iterator o = observations.begin(); o != observations.end(); ++o) obs.push_back(add_kf(o->first));
    }
    optr.push_back((int64_t)obs.size());
    return p;
  }
  void add_keyframe(const kfptr& pKF, const std::vector<mpptr>& vpMP) {
    batch.push_back(add_kf(pKF));
    for (size_t i = 0; i < vpMP.size(); i++) mp.push_back(vpMP[i] ? add_point(vpMP[i]) : -1);
    mptr.push_back((int64_t)mp.size());
  }
  // one ccm_covisibility(_host) call, ranks from std::less<kfptr>; a first capacity guess, then the exact total if it was short
  void run(bool device) {
    const std::vector<kfptr>& rows = batch_state->rows;
    std::vector<int32_t> order(rows.size());
    for (size_t i = 0; i < order.size(); i++) order[i] = (int32_t)i;
    std::sort(order.begin(), order.end(), [&](int32_t a, int32_t b) { return std::less<kfptr>()(rows[a], rows[b]); });
    std::vector<uint32_t> rank(rows.size());
    for (size_t i = 0; i < order.size(); i++) rank[order[i]] = (uint32_t)i;
    const int32_t n_b = (int32_t)batch.size();
    int64_t cap = std::min<int64_t>((int64_t)obs.size() + 1, 64 * (int64_t)n_b + 1024), total = 0;
    std::vector<int32_t> n_sel(n_b), sel_kf, sel_w;
    std::vector<uint8_t> status(n_b);
    out_ptr.assign(n_b + 1, 0);
    for (int attempt = 0; attempt < 2; attempt++) {
      out_kf.resize(cap); out_w.resize(cap); sel_kf.resize(cap); sel_w.resize(cap);
      const int rc = (device ? ccm_covisibility : ccm_covisibility_host)(
          (int32_t)rows.size(), kf_id.data(), rank.data(), n_b, batch.data(), mptr.data(), mp.data(), (int32_t)mp_bad.size(), mp_bad.data(),
          optr.data(), obs.data(), 15, cap, out_ptr.data(), out_kf.data(), out_w.data(), n_sel.data(), sel_kf.data(), sel_w.data(),
          status.data(), &total);
      if (rc != CCM_OK && attempt == 0 && total > cap) { cap = total; continue; }
      check(rc, device ? "ccm_covisibility" : "ccm_covisibility_host");
      break;
    }
  }
};

// the parked counter of this keyframe when its snapshot still holds
bool take_parked(const KeyFrame* self, const std::vector<mpptr>& vpMP, std::map<kfptr, int>& KFcounter) {
  std::unordered_map<const KeyFrame*, Parked>& t = parked();
  std::unordered_map<const KeyFrame*, Parked>::iterator it = t.empty() ? t.end() : t.find(self);
  if (it == t.end()) return false;
  const Parked& p = it->second;
  bool same = p.mvp.size() == vpMP.size();
  for (size_t i = 0; same && i < vpMP.size(); i++) {
    same = p.mvp[i] == vpMP[i].get();
    if (!same || !vpMP[i]) continue;
    std::unordered_map<const MapPoint*, PointState>::const_iterator s = p.batch->points.find(vpMP[i].get());
    same = s != p.batch->points.end() && s->second.bad == vpMP[i]->isBad() && s->second.nobs == vpMP[i]->Observations();
  }
  if (same) {
    for (size_t i = 0; i < p.counter.size(); i++)
      KFcounter.insert(KFcounter.end(), std::make_pair(p.batch->rows[p.counter[i].first], (int)p.counter[i].second));
    g_hits++;
  } else {
    g_stale++;
  }
  t.erase(it);
  return same;
}

void fill(const Flat& f, int32_t b, std::map<kfptr, int>& KFcounter) {
  for (int64_t e = f.out_ptr[b]; e < f.out_ptr[b + 1]; e++)
    KFcounter.insert(KFcounter.end(), std::make_pair(f.batch_state->rows[f.out_kf[e]], (int)f.out_w[e]));
}

}  // namespace

void ccm_b200_prepare_connections(const std::vector<kfptr>& keyframes) {
  Flat f;
  std::vector<const KeyFrame*> who;
  std::vector<std::vector<const MapPoint*> > snap;
  std::unordered_map<const KeyFrame*, int> seen;
  for (size_t i = 0; i < keyframes.size(); i++) {
    const kfptr& pKF = keyframes[i];
    if (!pKF || seen.count(pKF.get())) continue;
    seen[pKF.get()] = 1;
    std::vector<mpptr> vpMP;
    {
      std::unique_lock<std::mutex> lock(pKF->mMutexFeatures);
      vpMP = pKF->mvpMapPoints;
    }
    f.add_keyframe(pKF, vpMP);
    who.push_back(pKF.get());
    std::vector<const MapPoint*> s(vpMP.size());
    for (size_t j = 0; j < vpMP.size(); j++) s[j] = vpMP[j].get();
    snap.push_back(s);
  }
  if (who.empty()) return;
  f.run(true);
  std::shared_ptr<const Batch> shared = f.batch_state;
  std::unordered_map<const KeyFrame*, Parked>& t = parked();
  for (size_t b = 0; b < who.size(); b++) {
    Parked& p = t[who[b]];
    p.batch = shared;
    p.mvp.swap(snap[b]);
    p.counter.clear();
    for (int64_t e = f.out_ptr[b]; e < f.out_ptr[b + 1]; e++) p.counter.push_back(std::make_pair(f.out_kf[e], f.out_w[e]));
  }
}

void ccm_b200_clear_connections() { parked().clear(); }

void ccm_b200_connections_stats(unsigned long long* hits, unsigned long long* stale, unsigned long long* host) {
  if (hits) *hits = g_hits.load();
  if (stale) *stale = g_stale.load();
  if (host) *host = g_host.load();
}

void KeyFrame::UpdateConnections(bool bIgnoreMutex) {
  (void)bIgnoreMutex;
  bool bSetBad = false;
  std::map<kfptr, int> KFcounter;
  std::vector<mpptr> vpMP;
  {
    std::unique_lock<std::mutex> lockMPs(mMutexFeatures);
    vpMP = mvpMapPoints;
  }
  if (!take_parked(this, vpMP, KFcounter)) {                      // this keyframe alone, on the host
    g_host++;
    Flat f;
    f.add_keyframe(this->shared_from_this(), vpMP);
    f.run(false);
    fill(f, 0, KFcounter);
  }

  if (KFcounter.empty()) return;

  // from here on the reference's own logic: threshold and AddConnection in map order, the fallback maximum, the ordered lists
  int nmax = 0;
  kfptr pKFmax = nullptr;
  const int th = 15;
  std::vector<std::pair<int, kfptr> > vPairs;
  vPairs.reserve(KFcounter.size());
  for (std::map<kfptr, int>::iterator mit = KFcounter.begin(), mend = KFcounter.end(); mit != mend; mit++) {
    if (mit->second > nmax) {
      nmax = mit->second;
      pKFmax = mit->first;
    }
    if (mit->second >= th) {
      vPairs.push_back(std::make_pair(mit->second, mit->first));
      (mit->first)->AddConnection(this->shared_from_this(), mit->second);
    }
  }
  if (vPairs.empty()) {
    vPairs.push_back(std::make_pair(nmax, pKFmax));
    pKFmax->AddConnection(this->shared_from_this(), nmax);
  }
  std::sort(vPairs.begin(), vPairs.end());
  std::list<kfptr> lKFs;
  std::list<int> lWs;
  for (size_t i = 0; i < vPairs.size(); i++) {
    lKFs.push_front(vPairs[i].second);
    lWs.push_front(vPairs[i].first);
  }

  {
    std::unique_lock<std::mutex> lockCon(mMutexConnections);
    mConnectedKeyFrameWeights = KFcounter;
    mvpOrderedConnectedKeyFrames = std::vector<kfptr>(lKFs.begin(), lKFs.end());
    mvOrderedWeights = std::vector<int>(lWs.begin(), lWs.end());

    if (mbFirstConnection && mId.first != 0) {
      if (mSysState == eSystemState::CLIENT) {
        // the first ordered connection that is neither a child of this keyframe nor sent from the server
        mpParent = mvpOrderedConnectedKeyFrames.front();
        std::vector<kfptr>::iterator vit = mvpOrderedConnectedKeyFrames.begin();
        while (mspChildrens.count(mpParent) || mpParent->mbFromServer) {
          ++vit;
          if (vit == mvpOrderedConnectedKeyFrames.end()) {
            if (this->mId.second == mpMap->mMapId) bSetBad = true;
            else mpParent = nullptr;
            break;
          }
          mpParent = *vit;
        }
      } else if (mSysState == eSystemState::SERVER) {
        // the first ordered connection with a smaller mId.first, else the nearest of the nine predecessors in the map
        std::vector<kfptr>::iterator vit = mvpOrderedConnectedKeyFrames.begin();
        kfptr pPC = *vit;
        while (!(pPC->mId.first < this->mId.first)) {
          ++vit;
          if (vit == mvpOrderedConnectedKeyFrames.end()) {
            for (int itid = 1; itid < 10; itid++) {
              pPC = mpMap->GetKfPtr(mId.first - itid, mId.second);
              if (pPC) break;
            }
            if (!pPC) {
              std::cout << "No predecessor" << std::endl;
              throw estd::infrastructure_ex();
            }
            break;
          }
          pPC = *vit;
        }
        mpParent = pPC;
      }
      if (!bSetBad) {
        if (mpParent) {
          mpParent->AddChild(this->shared_from_this());
          mbFirstConnection = false;
        } else if (!(mSysState == eSystemState::CLIENT && this->mId.second != mpMap->mMapId)) {
          std::cout << "UpdateConnections: cannot find parent" << std::endl;
          throw infrastructure_ex();
        } else {
          // a client keyframe of another client's map without a parent: drop it
          for (std::map<kfptr, int>::iterator mit = mConnectedKeyFrameWeights.begin(), mend = mConnectedKeyFrameWeights.end(); mit != mend; mit++)
            mit->first->EraseConnection(this->shared_from_this());
          for (size_t i = 0; i < mvpMapPoints.size(); i++)
            if (mvpMapPoints[i]) mvpMapPoints[i]->EraseObservation(this->shared_from_this(), false, true);
          {
            std::unique_lock<std::mutex> lock1(mMutexFeatures);
            mConnectedKeyFrameWeights.clear();
            mvpOrderedConnectedKeyFrames.clear();
            if (!mspChildrens.empty()) std::cout << "UpdateConnections: mspChildrens assumed to be empty at this point" << std::endl;
            mbBad = true;
          }
          mpMap->EraseKeyFrame(this->shared_from_this());
          mpKeyFrameDB->erase(this->shared_from_this());
        }
      }
    }
  }

  if (!bSetBad && mpParent && mpParent->mId == this->mId) {
    std::cout << "UpdateConnections: child->mId == this->mId (" << mId.first << "|" << mId.second << ")" << std::endl;
    throw infrastructure_ex();
  }
  if (bSetBad) this->SetBadFlag(false, true);
}

}  // namespace cslam

// ref_covis_wrap.cpp — TEST INFRASTRUCTURE: stand-in KeyFrame / MapPoint scenes (oracle/ref_stub_cv) built from the flat arrays of
// synth.make_covisibility, the reference members UpdateConnections calls, and the ways to run it:
//   AddConnection, UpdateBestCovisibles, AddChild, EraseConnection   cslam/src/KeyFrame.cpp:392-426, 858-863, 458-470, restated
//   literal_update_connections   the reference body (KeyFrame.cpp:629-852) restated on the stand-ins, server branch (the server's
//                                keyframes are the ones batched); a std::map<kfptr,int> counter filled one observation at a time
//   cv_merge         MapMerger::MergeMaps' CorrectedSim3All loop shape (MapMerger.cpp:349-395): per keyframe SetPose + UpdateConnections,
//                    through the literal body, the shim member alone, or the shim after ccm_b200_prepare_connections
//   cv_merge_stale   prepare, change the scene (a map point index, an observation count, a point set bad), then the shim loop
//   cv_load_map      Map::LoadMap's keyframe loop (Map.cpp:596-618), as the reference runs it (AddMapPoint then the literal body per
//                    keyframe) or split as INTEGRATION.md §4e describes (every AddMapPoint, one prepare, every UpdateConnections)
//   cv_literal_flat  the literal counter and ordered list of each batch keyframe, read without touching the scene's members
// Keyframe row k lives at slot kf_rank[k] of one array, so its address rank is kf_rank[k] and every std::map<kfptr,...> iterates in
// ascending kf_rank.  All keyframes are server keyframes of one Map per mId.second.
#include <cslam/KeyFrame.h>
#include <cslam/MapPoint.h>

#include <algorithm>
#include <cstdint>
#include <cstring>
#include <list>
#include <map>
#include <vector>

#include "../shim/KeyFrameConnections_shim.h"

using namespace cslam;
typedef boost::shared_ptr<KeyFrame> kfptr;
typedef boost::shared_ptr<MapPoint> mpptr;

// ---- the reference members UpdateConnections calls --------------------------------------------------------------------------------
void KeyFrame::AddConnection(kfptr pKF, const int& weight) {
  {
    std::unique_lock<std::mutex> lock(mMutexConnections);
    if (!mConnectedKeyFrameWeights.count(pKF)) mConnectedKeyFrameWeights[pKF] = weight;
    else if (mConnectedKeyFrameWeights[pKF] != weight) mConnectedKeyFrameWeights[pKF] = weight;
    else return;
  }
  UpdateBestCovisibles();
}

void KeyFrame::UpdateBestCovisibles() {
  std::unique_lock<std::mutex> lock(mMutexConnections);
  std::vector<std::pair<int, kfptr> > vPairs;
  vPairs.reserve(mConnectedKeyFrameWeights.size());
  for (std::map<kfptr, int>::iterator mit = mConnectedKeyFrameWeights.begin(); mit != mConnectedKeyFrameWeights.end(); mit++)
    vPairs.push_back(std::make_pair(mit->second, mit->first));
  std::sort(vPairs.begin(), vPairs.end());
  std::list<kfptr> lKFs;
  std::list<int> lWs;
  for (size_t i = 0; i < vPairs.size(); i++) { lKFs.push_front(vPairs[i].second); lWs.push_front(vPairs[i].first); }
  mvpOrderedConnectedKeyFrames = std::vector<kfptr>(lKFs.begin(), lKFs.end());
  mvOrderedWeights = std::vector<int>(lWs.begin(), lWs.end());
}

void KeyFrame::AddChild(kfptr pKF) {
  std::unique_lock<std::mutex> lockCon(mMutexConnections);
  mspChildrens.insert(pKF);
}

void KeyFrame::EraseConnection(kfptr pKF) {
  bool bUpdate = false;
  {
    std::unique_lock<std::mutex> lock(mMutexConnections);
    if (mConnectedKeyFrameWeights.count(pKF)) { mConnectedKeyFrameWeights.erase(pKF); bUpdate = true; }
  }
  if (bUpdate) UpdateBestCovisibles();
}

void KeyFrame::SetBadFlag(bool, bool) { std::unique_lock<std::mutex> lock(mMutexConnections); mbBad = true; }

// ---- the literal body ---------------------------------------------------------------------------------------------------------
// KeyFrame.cpp:629-852, server branch.  out_counter: a copy of KFcounter (bookkeeping for the flat comparison, not part of the body);
// apply = false stops before the first write (AddConnection and the members).
static void literal_update_connections(KeyFrame* self, bool apply, std::map<kfptr, int>* out_counter = nullptr,
                                       std::vector<std::pair<int, kfptr> >* out_pairs = nullptr) {
  std::map<kfptr, int> KFcounter;
  std::vector<mpptr> vpMP;
  {
    std::unique_lock<std::mutex> lockMPs(self->mMutexFeatures);
    vpMP = self->mvpMapPoints;
  }
  for (std::vector<mpptr>::iterator vit = vpMP.begin(), vend = vpMP.end(); vit != vend; vit++) {
    mpptr pMP = *vit;
    if (!pMP) continue;
    if (pMP->isBad()) continue;
    std::map<kfptr, size_t> observations = pMP->GetObservations();
    for (std::map<kfptr, size_t>::iterator mit = observations.begin(), mend = observations.end(); mit != mend; mit++) {
      if (mit->first->mId == self->mId) continue;
      KFcounter[mit->first]++;
    }
  }
  if (out_counter) *out_counter = KFcounter;
  if (KFcounter.empty()) return;
  int nmax = 0;
  kfptr pKFmax = nullptr;
  int th = 15;
  std::vector<std::pair<int, kfptr> > vPairs;
  vPairs.reserve(KFcounter.size());
  for (std::map<kfptr, int>::iterator mit = KFcounter.begin(), mend = KFcounter.end(); mit != mend; mit++) {
    if (mit->second > nmax) { nmax = mit->second; pKFmax = mit->first; }
    if (mit->second >= th) {
      vPairs.push_back(std::make_pair(mit->second, mit->first));
      if (apply) (mit->first)->AddConnection(self->shared_from_this(), mit->second);
    }
  }
  if (vPairs.empty()) {
    vPairs.push_back(std::make_pair(nmax, pKFmax));
    if (apply) pKFmax->AddConnection(self->shared_from_this(), nmax);
  }
  std::sort(vPairs.begin(), vPairs.end());
  std::list<kfptr> lKFs;
  std::list<int> lWs;
  for (size_t i = 0; i < vPairs.size(); i++) { lKFs.push_front(vPairs[i].second); lWs.push_front(vPairs[i].first); }
  if (out_pairs) {
    out_pairs->clear();
    std::list<int>::iterator w = lWs.begin();
    for (std::list<kfptr>::iterator k = lKFs.begin(); k != lKFs.end(); ++k, ++w) out_pairs->push_back(std::make_pair(*w, *k));
  }
  if (!apply) return;
  {
    std::unique_lock<std::mutex> lockCon(self->mMutexConnections);
    self->mConnectedKeyFrameWeights = KFcounter;
    self->mvpOrderedConnectedKeyFrames = std::vector<kfptr>(lKFs.begin(), lKFs.end());
    self->mvOrderedWeights = std::vector<int>(lWs.begin(), lWs.end());
    if (self->mbFirstConnection && self->mId.first != 0) {
      std::vector<kfptr>::iterator vit = self->mvpOrderedConnectedKeyFrames.begin();
      kfptr pPC = *vit;
      while (!(pPC->mId.first < self->mId.first)) {
        ++vit;
        if (vit == self->mvpOrderedConnectedKeyFrames.end()) {
          for (int itid = 1; itid < 10; itid++) {
            pPC = self->mpMap->GetKfPtr(self->mId.first - itid, self->mId.second);
            if (pPC) break;
          }
          if (!pPC) throw estd::infrastructure_ex();
          break;
        }
        pPC = *vit;
      }
      self->mpParent = pPC;
      self->mpParent->AddChild(self->shared_from_this());
      self->mbFirstConnection = false;
    }
  }
  if (self->mpParent && self->mpParent->mId == self->mId) throw estd::infrastructure_ex();
}

// ---- scenes -------------------------------------------------------------------------------------------------------------------
struct Scene {
  std::vector<KeyFrame> kf_store;                     // row k at slot rank[k]
  std::vector<kfptr> kfs;                             // by row
  std::vector<mpptr> mps;
  std::vector<std::vector<int32_t> > mvp;             // each row's point list, for AddMapPoint
  std::vector<int32_t> batch;
  std::map<size_t, boost::shared_ptr<Map> > maps;
};

extern "C" void* cv_scene_create(int32_t K, const uint64_t* kf_id, const uint32_t* kf_rank, const uint8_t* kf_bad, const uint8_t* first_conn,
                                 const int64_t* mvp_ptr, const int32_t* mvp, int32_t P, const uint8_t* mp_bad, const int64_t* obs_ptr,
                                 const int32_t* obs_kf, const int32_t* obs_idx, int32_t n_b, const int32_t* batch, int fill_mvp) {
  Scene* s = new Scene();
  s->kf_store = std::vector<KeyFrame>(K);
  for (int32_t k = 0; k < K; k++) {
    KeyFrame& kf = s->kf_store[kf_rank[k]];
    kf.mId = std::make_pair((size_t)(kf_id[k] & 0xffffffffu), (size_t)(kf_id[k] >> 32));
    kf.mbBad = kf_bad[k] != 0;
    kf.mbFirstConnection = first_conn[k] != 0;
    kf.mnRowForTest = k;
    kf.mvpMapPoints.resize(mvp_ptr[k + 1] - mvp_ptr[k]);
    boost::shared_ptr<Map>& m = s->maps[kf.mId.second];
    if (!m) { m.reset(new Map()); m->mMapId = kf.mId.second; }
    kf.mpMap = m;
    kf.mpKeyFrameDB.reset(new KeyFrameDatabase());
    s->kfs.push_back(kfptr(&kf, [](KeyFrame*) {}));
    s->mvp.push_back(std::vector<int32_t>(mvp + mvp_ptr[k], mvp + mvp_ptr[k + 1]));
  }
  for (int32_t k = 0; k < K; k++) {
    Map& m = *s->kfs[k]->mpMap;
    if (!m.mmpKeyFrames.count(s->kfs[k]->mId)) m.mmpKeyFrames[s->kfs[k]->mId] = s->kfs[k];
  }
  for (int32_t i = 0; i < P; i++) {
    mpptr m(new MapPoint());
    for (int64_t e = obs_ptr[i]; e < obs_ptr[i + 1]; e++) m->AddObservationForTest(s->kfs[obs_kf[e]], (size_t)obs_idx[e]);
    m->SetBadForTest(mp_bad[i] != 0);
    s->mps.push_back(m);
  }
  if (fill_mvp)
    for (int32_t k = 0; k < K; k++)
      for (size_t j = 0; j < s->mvp[k].size(); j++) s->kfs[k]->mvpMapPoints[j] = s->mvp[k][j] >= 0 ? s->mps[s->mvp[k][j]] : mpptr();
  s->batch.assign(batch, batch + n_b);
  return s;
}

extern "C" void cv_scene_destroy(void* h) {
  Scene* s = static_cast<Scene*>(h);
  for (size_t k = 0; k < s->kfs.size(); k++) {          // break the kfptr cycles through parents, children and connections
    KeyFrame& kf = *s->kfs[k];
    kf.mConnectedKeyFrameWeights.clear(); kf.mvpOrderedConnectedKeyFrames.clear(); kf.mspChildrens.clear(); kf.mpParent.reset();
  }
  delete s;
}

extern "C" void cv_stats(unsigned long long* c) { ccm_b200_connections_stats(&c[0], &c[1], &c[2]); }

// mode 0: the literal body; 1: the shim member alone; 2: ccm_b200_prepare_connections over the batch, then the shim member.
// Returns 0, or -1 when something threw.
static int run_loop(Scene* s, int mode) {
  try {
    ParkedConnectionsGuard guard;
    std::vector<kfptr> keys;
    for (size_t i = 0; i < s->batch.size(); i++) keys.push_back(s->kfs[s->batch[i]]);
    if (mode == 2) ccm_b200_prepare_connections(keys);
    cv::Mat T = cv::Mat::eye(4, 4, CV_32F);
    for (size_t i = 0; i < keys.size(); i++) {
      keys[i]->SetPose(T, true);
      if (mode == 0) literal_update_connections(keys[i].get(), true);
      else keys[i]->UpdateConnections();
    }
  } catch (...) {
    return -1;
  }
  return 0;
}

extern "C" int cv_merge(void* h, int mode) { return run_loop(static_cast<Scene*>(h), mode); }

// kind 1: the first map point index of every third batch keyframe set to null (or to a point when null); kind 2: one observation
// added to the first point of every third batch keyframe (count changes); kind 3: that point set bad; kind 4: one observer of that
// point replaced by another keyframe (count unchanged: the snapshot does not see it).  Then the shim loop; literal = 1: no prepare,
// the same changes, then the literal body (the members the reference leaves on the changed scene).
extern "C" int cv_merge_stale(void* h, int kind, int32_t extra_row, int literal) {
  Scene* s = static_cast<Scene*>(h);
  try {
    ParkedConnectionsGuard guard;
    std::vector<kfptr> keys;
    for (size_t i = 0; i < s->batch.size(); i++) keys.push_back(s->kfs[s->batch[i]]);
    if (!literal) ccm_b200_prepare_connections(keys);
    for (size_t i = 0; i < keys.size(); i += 3) {
      KeyFrame& kf = *keys[i];
      if (kf.mvpMapPoints.empty()) continue;
      size_t j = 0;
      while (j < kf.mvpMapPoints.size() && !kf.mvpMapPoints[j]) j++;
      if (kind == 1) { kf.mvpMapPoints[0] = kf.mvpMapPoints[0] ? mpptr() : s->mps[0]; continue; }
      if (j == kf.mvpMapPoints.size()) continue;
      MapPoint& m = *kf.mvpMapPoints[j];
      const std::map<kfptr, size_t> obs = m.GetObservations();
      if (kind == 2) m.AddObservationForTest(s->kfs[extra_row], 0);
      if (kind == 3) m.SetBadForTest(true);
      if (kind == 4 && !obs.empty() && !obs.count(s->kfs[extra_row])) m.ReplaceObserverForTest(obs.rbegin()->first, s->kfs[extra_row]);
    }
    for (size_t i = 0; i < keys.size(); i++) {
      if (literal) literal_update_connections(keys[i].get(), true);
      else keys[i]->UpdateConnections();
    }
  } catch (...) {
    return -1;
  }
  return 0;
}

// Map::LoadMap's keyframe loop over the batch (the scene was created with empty mvpMapPoints).  split 0: per keyframe every
// AddMapPoint, then the literal body; split 1: every AddMapPoint of every keyframe, one prepare, then the shim member per keyframe.
extern "C" int cv_load_map(void* h, int split) {
  Scene* s = static_cast<Scene*>(h);
  try {
    ParkedConnectionsGuard guard;
    std::vector<kfptr> keys;
    for (size_t i = 0; i < s->batch.size(); i++) keys.push_back(s->kfs[s->batch[i]]);
    for (size_t i = 0; i < keys.size(); i++) {
      const std::vector<int32_t>& l = s->mvp[keys[i]->mnRowForTest];
      for (size_t j = 0; j < l.size(); j++)
        if (l[j] >= 0) keys[i]->AddMapPoint(s->mps[l[j]], j);
      if (!split) literal_update_connections(keys[i].get(), true);
    }
    if (split) {
      ccm_b200_prepare_connections(keys);
      for (size_t i = 0; i < keys.size(); i++) keys[i]->UpdateConnections();
    }
  } catch (...) {
    return -1;
  }
  return 0;
}

// the members of every keyframe row as CSR arrays of room `cap` each; sizes[4] = entries written to each (weights, ordered,
// children) and -1 if cap was short.  parent[k]: the parent's row, -1 none.
extern "C" int cv_members(void* h, int64_t cap, int64_t* w_ptr, int32_t* w_kf, int32_t* w_w, int64_t* o_ptr, int32_t* o_kf, int32_t* o_w,
                          int64_t* c_ptr, int32_t* c_kf, int32_t* parent, uint8_t* first_conn) {
  Scene* s = static_cast<Scene*>(h);
  int64_t a = 0, b = 0, c = 0;
  w_ptr[0] = o_ptr[0] = c_ptr[0] = 0;
  for (size_t k = 0; k < s->kfs.size(); k++) {
    KeyFrame& kf = *s->kfs[k];
    for (std::map<kfptr, int>::iterator it = kf.mConnectedKeyFrameWeights.begin(); it != kf.mConnectedKeyFrameWeights.end(); ++it, ++a) {
      if (a >= cap) return -1;
      w_kf[a] = it->first->mnRowForTest; w_w[a] = it->second;
    }
    if (kf.mvpOrderedConnectedKeyFrames.size() != kf.mvOrderedWeights.size()) return -2;
    for (size_t i = 0; i < kf.mvpOrderedConnectedKeyFrames.size(); i++, b++) {
      if (b >= cap) return -1;
      o_kf[b] = kf.mvpOrderedConnectedKeyFrames[i]->mnRowForTest; o_w[b] = kf.mvOrderedWeights[i];
    }
    for (std::set<kfptr>::iterator it = kf.mspChildrens.begin(); it != kf.mspChildrens.end(); ++it, ++c) {
      if (c >= cap) return -1;
      c_kf[c] = (*it)->mnRowForTest;
    }
    w_ptr[k + 1] = a; o_ptr[k + 1] = b; c_ptr[k + 1] = c;
    parent[k] = kf.mpParent ? kf.mpParent->mnRowForTest : -1;
    first_conn[k] = kf.mbFirstConnection ? 1 : 0;
  }
  return 0;
}

// the literal counter and selection of each batch keyframe (the flat outputs of ccm_covisibility), members untouched
extern "C" int cv_literal_flat(void* h, int64_t cap, int64_t* conn_ptr, int32_t* conn_kf, int32_t* conn_w, int32_t* n_sel, int32_t* sel_kf,
                               int32_t* sel_w, uint8_t* status) {
  Scene* s = static_cast<Scene*>(h);
  int64_t at = 0;
  conn_ptr[0] = 0;
  for (size_t b = 0; b < s->batch.size(); b++) {
    std::map<kfptr, int> counter;
    std::vector<std::pair<int, kfptr> > pairs;
    literal_update_connections(s->kfs[s->batch[b]].get(), false, &counter, &pairs);
    if (at + (int64_t)counter.size() > cap) return -1;
    const int64_t base = at;
    for (std::map<kfptr, int>::iterator it = counter.begin(); it != counter.end(); ++it, ++at) {
      conn_kf[at] = it->first->mnRowForTest; conn_w[at] = it->second; sel_kf[at] = -1; sel_w[at] = 0;
    }
    for (size_t i = 0; i < pairs.size(); i++) { sel_kf[base + i] = pairs[i].second->mnRowForTest; sel_w[base + i] = pairs[i].first; }
    conn_ptr[b + 1] = at;
    n_sel[b] = (int32_t)pairs.size();
    status[b] = counter.empty() ? 0 : 1;
  }
  return 0;
}

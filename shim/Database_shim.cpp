// Database_shim.cpp — cslam::KeyFrameDatabase on top of libccm_b200.so (ccm_kfdb_*).  Replaces cslam/src/Database.cpp; compiled
// against the reference's own cslam/Database.h, which stays byte-identical.
//
//   add / erase / clear                   Database.cpp:37-70   -> ccm_kfdb_add / erase / clear (uid = mUniqueId, client = mId.second)
//   DetectLoopCandidates                  Database.cpp:72-202  -> visibility from the objects the reference reads, ccm_kfdb_query,
//   DetectMapMatchCandidates              Database.cpp:204-327    GetBestCovisibilityKeyFrames(10) of the scored candidates only,
//   DetectRelocalizationCandidates        Database.cpp:329-439    ccm_kfdb_select
//   AddMP / AddDirectBad / Find* / ResetMPs  Database.cpp:441-485 (the debug maps, host containers as before)
//
// The header declares no destructor, so the device database lives in a side table keyed by the KeyFrameDatabase object
// (ORBVocabulary_shim.cpp keeps its vocabularies the same way); a new database at the same address replaces the entry.  The side table
// also holds the keyframe pointers in the database, as the reference's inverted file does, to turn the returned uids into kfptr.
//
// Visibility (DESIGN.md §5): a loop query sees the database keyframes of the query map's clients that are in GetMmpKeyFrames(), minus the
// query keyframe and GetConnectedKeyFrames(); a keyframe in the database but not in the map is passed as an explicit exclusion.  A
// map-match query sees the keyframes of every client not in pMap->msuAssClients; relocalisation sees all.  The marker members
// (mLoopQuery / mMatchQuery / mRelocQuery, mnLoopWords / mnRelocWords, mLoopScore / mRelocScore) are written for the scored candidates;
// the counts of keyframes that were not scored and the mnLoopWords = 1 the reference leaves on connected keyframes are not.
// A keyframe added twice keeps its first place (the reference would list it twice).
#include <cslam/Database.h>

#include <map>
#include <memory>
#include <mutex>
#include <stdexcept>
#include <string>
#include <unordered_map>
#include <vector>

#include "ccm_b200.h"

namespace cslam {

namespace {

struct DeviceDb {
  ccm_kfdb* h = nullptr;
  std::mutex mu;                                                     // guards kfs (the device handle has its own lock)
  std::unordered_map<size_t, KeyFrameDatabase::kfptr> kfs;           // mUniqueId -> keyframe in the database
  ~DeviceDb() { if (h) ccm_kfdb_destroy(h); }
};

std::mutex g_mu;
std::map<const KeyFrameDatabase*, std::shared_ptr<DeviceDb>> g_db;

std::shared_ptr<DeviceDb> db_of(const KeyFrameDatabase* d) {
  std::lock_guard<std::mutex> lk(g_mu);
  auto it = g_db.find(d);
  if (it == g_db.end()) throw std::runtime_error("KeyFrameDatabase: no device database (constructor not run through the shim)");
  return it->second;
}

void check(int rc) {
  if (rc != CCM_OK) throw std::runtime_error(std::string("libccm_b200: ") + ccm_last_error());
}

void flatten(const DBoW2::BowVector& b, std::vector<uint32_t>& w, std::vector<double>& v) {
  w.clear(); v.clear();
  for (DBoW2::BowVector::const_iterator it = b.begin(); it != b.end(); ++it) { w.push_back(it->first); v.push_back(it->second); }
}

uint64_t client_bit(size_t c) { return c < 64 ? (1ull << c) : 0ull; }

enum Kind { LOOP, MAP_MATCH, RELOC };

// the device query, the markers of the scored candidates, the covisibility lists of the scored candidates, the selection
std::vector<KeyFrameDatabase::kfptr> detect(DeviceDb& D, const DBoW2::BowVector& bow, uint64_t mask, const std::vector<uint64_t>& exclude,
                                            Kind kind, const idpair& qid, float minScore) {
  typedef KeyFrameDatabase::kfptr kfptr;
  std::vector<uint32_t> w; std::vector<double> v;
  flatten(bow, w, v);
  std::vector<ccm_kfdb_candidate> cand;
  {
    std::lock_guard<std::mutex> lk(D.mu);
    cand.resize(D.kfs.size() + 1);
  }
  ccm_kfdb_request q;
  q.n = (int32_t)w.size(); q.word = w.data(); q.value = v.data(); q.client_mask = mask;
  q.n_exclude = (int32_t)exclude.size(); q.exclude_uid = exclude.data();
  ccm_kfdb_result r;
  for (;;) {                                                         // another thread may add keyframes: grow to what the query needs
    r.cand = cand.data(); r.cap = (int32_t)cand.size(); r.n = 0;
    const int rc = ccm_kfdb_query(D.h, &q, &r);
    if (rc == CCM_ERR_INVALID && r.n > r.cap) { cand.resize(r.n + 16); continue; }
    check(rc);
    break;
  }
  std::vector<kfptr> scored(r.n);
  {
    std::lock_guard<std::mutex> lk(D.mu);
    for (int i = 0; i < r.n; i++) {
      auto it = D.kfs.find((size_t)cand[i].uid);
      if (it == D.kfs.end()) throw std::runtime_error("KeyFrameDatabase: device returned an unknown keyframe");
      scored[i] = it->second;
    }
  }
  for (int i = 0; i < r.n; i++) {
    kfptr k = scored[i];
    if (kind == LOOP) { k->mLoopQuery = qid; k->mnLoopWords = cand[i].n_words; k->mLoopScore = cand[i].score; }
    else if (kind == MAP_MATCH) { k->mMatchQuery = qid; k->mnLoopWords = cand[i].n_words; k->mLoopScore = cand[i].score; }
    else { k->mRelocQuery = qid; k->mnRelocWords = cand[i].n_words; k->mRelocScore = cand[i].score; }
  }
  std::vector<int32_t> ptr(1, 0);
  std::vector<uint64_t> covis;
  for (int i = 0; i < r.n; i++) {
    if (kind == RELOC || cand[i].score >= minScore) {               // the selection reads the lists of these candidates only
      std::vector<kfptr> nb = scored[i]->GetBestCovisibilityKeyFrames(10);
      for (size_t j = 0; j < nb.size(); j++) covis.push_back(nb[j]->mUniqueId);
    }
    ptr.push_back((int32_t)covis.size());
  }
  std::vector<uint64_t> out(r.n + 1);
  int32_t n_out = 0;
  check(ccm_kfdb_select(&r, ptr.data(), covis.data(), kind == RELOC, minScore, out.data(), &n_out));
  std::vector<kfptr> res;
  res.reserve(n_out);
  std::lock_guard<std::mutex> lk(D.mu);
  for (int i = 0; i < n_out; i++) res.push_back(D.kfs.at((size_t)out[i]));
  return res;
}

}  // namespace

KeyFrameDatabase::KeyFrameDatabase(const vocptr pVoc) : mpVoc(pVoc) {
  std::shared_ptr<DeviceDb> d(new DeviceDb);
  check(ccm_kfdb_create((int32_t)pVoc->size(), (int32_t)pVoc->getScoringType(), &d->h));
  std::lock_guard<std::mutex> lk(g_mu);
  g_db[this] = d;
}

void KeyFrameDatabase::add(kfptr pKF) {
  std::shared_ptr<DeviceDb> D = db_of(this);
  {
    std::lock_guard<std::mutex> lk(D->mu);
    if (D->kfs.count(pKF->mUniqueId)) return;
    D->kfs[pKF->mUniqueId] = pKF;
  }
  std::vector<uint32_t> w; std::vector<double> v;
  flatten(pKF->mBowVec, w, v);
  check(ccm_kfdb_add(D->h, pKF->mUniqueId, (uint32_t)pKF->mId.second, (int32_t)w.size(), w.data(), v.data()));
}

void KeyFrameDatabase::erase(kfptr pKF) {
  std::shared_ptr<DeviceDb> D = db_of(this);
  check(ccm_kfdb_erase(D->h, pKF->mUniqueId));
  std::lock_guard<std::mutex> lk(D->mu);
  D->kfs.erase(pKF->mUniqueId);
}

void KeyFrameDatabase::clear() {
  std::shared_ptr<DeviceDb> D = db_of(this);
  check(ccm_kfdb_clear(D->h));
  std::lock_guard<std::mutex> lk(D->mu);
  D->kfs.clear();
}

vector<KeyFrameDatabase::kfptr> KeyFrameDatabase::DetectLoopCandidates(kfptr pKF, float minScore) {
  std::shared_ptr<DeviceDb> D = db_of(this);
  set<kfptr> spConnectedKeyFrames = pKF->GetConnectedKeyFrames();
  std::map<idpair, kfptr> mpAllKfsInMap = pKF->GetMapptr()->GetMmpKeyFrames();
  uint64_t mask = 0;
  for (std::map<idpair, kfptr>::const_iterator it = mpAllKfsInMap.begin(); it != mpAllKfsInMap.end(); ++it) mask |= client_bit(it->first.second);
  std::vector<uint64_t> exclude(1, pKF->mUniqueId);
  for (set<kfptr>::const_iterator it = spConnectedKeyFrames.begin(); it != spConnectedKeyFrames.end(); ++it) exclude.push_back((*it)->mUniqueId);
  {
    std::lock_guard<std::mutex> lk(D->mu);
    for (auto& kv : D->kfs)                                          // in the database and of a visible client, but not in the map
      if ((mask & client_bit(kv.second->mId.second)) && !mpAllKfsInMap.count(kv.second->mId)) exclude.push_back(kv.first);
  }
  return detect(*D, pKF->mBowVec, mask, exclude, LOOP, pKF->mId, minScore);
}

vector<KeyFrameDatabase::kfptr> KeyFrameDatabase::DetectMapMatchCandidates(kfptr pKF, float minScore, mapptr pMap) {
  std::shared_ptr<DeviceDb> D = db_of(this);
  uint64_t mask = ~0ull;
  for (set<size_t>::const_iterator it = pMap->msuAssClients.begin(); it != pMap->msuAssClients.end(); ++it) mask &= ~client_bit(*it);
  return detect(*D, pKF->mBowVec, mask, std::vector<uint64_t>(), MAP_MATCH, pKF->mId, minScore);
}

std::vector<KeyFrameDatabase::kfptr> KeyFrameDatabase::DetectRelocalizationCandidates(Frame& F) {
  std::shared_ptr<DeviceDb> D = db_of(this);
  return detect(*D, F.mBowVec, ~0ull, std::vector<uint64_t>(), RELOC, F.mId, 0.f);
}

void KeyFrameDatabase::AddMP(mpptr pMP) {
  if (!pMP) return;
  unique_lock<mutex> lock(mMutexMPs);
  mmpMPs[pMP->mId] = pMP;
}

void KeyFrameDatabase::AddDirectBad(size_t id, size_t cid) {
  unique_lock<mutex> lock(mMutexMPs);
  mmbDirectBad[make_pair(id, cid)] = true;
}

bool KeyFrameDatabase::FindMP(size_t id, size_t cid) {
  unique_lock<mutex> lock(mMutexMPs);
  return mmpMPs.count(make_pair(id, cid)) > 0;
}

bool KeyFrameDatabase::FindDirectBad(size_t id, size_t cid) {
  unique_lock<mutex> lock(mMutexMPs);
  return mmbDirectBad.count(make_pair(id, cid)) > 0;
}

void KeyFrameDatabase::ResetMPs() {
  unique_lock<mutex> lock(mMutexMPs);
  mmbDirectBad.clear();
  mmpMPs.clear();
}

}  // namespace cslam

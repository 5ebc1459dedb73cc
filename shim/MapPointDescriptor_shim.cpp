// MapPointDescriptor_shim.cpp — reference-side translation unit for MapPoint::ComputeDistinctiveDescriptors
// (cslam/src/MapPoint.cpp:929-994).
//
// The body is deleted from MapPoint.cpp and defined here (mDescriptor is protected and has no setter; a member body keeps MapPoint.h
// unchanged).  Two paths leave the same member, byte for byte:
//   * batched: a loop over many points calls ccm_b200_prepare_descriptors (or ccm_b200_prepare_point_updates) once before it starts.
//     It flattens the points (observers in mObservations order, each keyframe's isBad() read once), makes one ccm_distinctive_descriptors
//     call on the GPU, or ccm_kfstore_distinctive_descriptors when a keyframe store is registered, and parks the chosen position per
//     thread with a snapshot of the observation list it was chosen from: the (KeyFrame*, idx) pairs in order.  The member then clones
//     that keyframe's mDescriptors.row(idx) when its own copy of mObservations equals the snapshot;
//   * single point: every other caller (Replace, ReplaceAndLock, the MapMerger / LoopFinder fusion loops) and any point whose snapshot
//     went stale chooses on the host through ccm_distinctive_descriptors_host, the same rule.
// Either way the bytes are cloned from pKF->mDescriptors.row(idx), where the reference takes them from.
// In this repository it is compiled against the stand-in MapPoint / KeyFrame of oracle/ref_stub_dd and run next to a literal
// restatement of the reference body by tests/test_shim_distinctive.py.
#include <cslam/KeyFrame.h>
#include <cslam/MapPoint.h>
#include <cslam/estd.h>

#include <atomic>
#include <cstring>
#include <iostream>
#include <unordered_map>
#include <utility>
#include <vector>

#include "MapPointDescriptor_shim.h"
#include "MapPoint_shim.h"
#include "ccm_b200.h"

namespace cslam {

namespace {

typedef boost::shared_ptr<KeyFrame> kfptr;
typedef boost::shared_ptr<MapPoint> mpptr;
typedef std::vector<std::pair<const KeyFrame*, size_t> > ObsList;

struct Parked {
  ObsList obs;      // the observation list the choice was made from, in mObservations order
  int32_t best;     // position of the chosen observer in it; -1: every observer was bad
};

std::unordered_map<const MapPoint*, Parked>& parked() {
  static thread_local std::unordered_map<const MapPoint*, Parked> table;
  return table;
}

std::atomic<ccm_kf_store*> g_store(nullptr);

// the flat arrays of include/ccm_b200.h's ccm_distinctive_descriptors / ccm_kfstore_distinctive_descriptors
struct FlatDescriptors {
  bool store;                       // rows named by (uid, idx) instead of copied
  std::vector<uint8_t> bad, desc;
  std::vector<uint64_t> uid;
  std::vector<int64_t> ptr{0};
  std::vector<int32_t> obs, feat;
  std::unordered_map<const KeyFrame*, int32_t> row;

  explicit FlatDescriptors(bool by_uid) : store(by_uid) {}
  int32_t add_kf(const kfptr& pKF) {
    std::unordered_map<const KeyFrame*, int32_t>::const_iterator it = row.find(pKF.get());
    if (it != row.end()) return it->second;
    const int32_t r = (int32_t)bad.size();
    row[pKF.get()] = r;
    bad.push_back(pKF->isBad() ? 1 : 0);
    if (store) uid.push_back((uint64_t)pKF->mUniqueId);
    return r;
  }
  // one point: observers in map order; a bad observer's row is not read
  void add_point(const std::map<kfptr, size_t>& observations) {
    for (std::map<kfptr, size_t>::const_iterator it = observations.begin(); it != observations.end(); ++it) {
      const int32_t r = add_kf(it->first);
      obs.push_back(r);
      if (store) {
        feat.push_back((int32_t)it->second);
      } else {
        const size_t at = desc.size();
        desc.resize(at + 32, 0);
        if (!bad[r]) std::memcpy(&desc[at], it->first->mDescriptors.ptr((int)it->second), 32);
      }
    }
    ptr.push_back((int64_t)obs.size());
  }
  int32_t n_points() const { return (int32_t)ptr.size() - 1; }
};

// as MapPoint_shim.cpp's check(): the reference's callers handle estd::infrastructure_ex
void check(int rc, const char* fn) {
  if (rc != CCM_OK) { std::cerr << "libccm_b200: " << fn << ": " << ccm_last_error() << std::endl; throw estd::infrastructure_ex(); }
}

ObsList snapshot(const std::map<kfptr, size_t>& observations) {
  ObsList s;
  s.reserve(observations.size());
  for (std::map<kfptr, size_t>::const_iterator it = observations.begin(); it != observations.end(); ++it) s.push_back(std::make_pair(it->first.get(), it->second));
  return s;
}

bool same_list(const ObsList& s, const std::map<kfptr, size_t>& observations) {
  if (s.size() != observations.size()) return false;
  size_t i = 0;
  for (std::map<kfptr, size_t>::const_iterator it = observations.begin(); it != observations.end(); ++it, ++i)
    if (s[i].first != it->first.get() || s[i].second != it->second) return false;
  return true;
}

// member calls by outcome, process-wide: a parked choice written / a parked choice found stale / chosen on the host
std::atomic<unsigned long long> g_hits(0), g_stale(0), g_host(0);

}  // namespace

void ccm_b200_register_kfstore(ccm_kf_store* store) { g_store.store(store); }

void ccm_b200_prepare_descriptors(const std::vector<mpptr>& points) {
  ccm_kf_store* store = g_store.load();
  FlatDescriptors f(store != nullptr);
  std::vector<const MapPoint*> who;
  std::vector<ObsList> snap;
  for (size_t i = 0; i < points.size(); i++) {
    const mpptr& pMP = points[i];
    if (!pMP || pMP->isBad()) continue;
    const std::map<kfptr, size_t> observations = pMP->GetObservations();
    if (observations.empty()) continue;                            // the member returns before writing there
    f.add_point(observations);
    who.push_back(pMP.get());
    snap.push_back(snapshot(observations));
  }
  const int32_t P = f.n_points();
  if (P == 0) return;
  std::vector<int32_t> best(P);
  if (store)
    check(ccm_kfstore_distinctive_descriptors(store, (int32_t)f.bad.size(), f.uid.data(), f.bad.data(), P, f.ptr.data(), f.obs.data(),
                                              f.feat.data(), best.data(), nullptr, nullptr),
          "ccm_kfstore_distinctive_descriptors");
  else
    check(ccm_distinctive_descriptors((int32_t)f.bad.size(), f.bad.data(), P, f.ptr.data(), f.obs.data(), f.desc.data(), best.data(), nullptr,
                                      nullptr),
          "ccm_distinctive_descriptors");
  std::unordered_map<const MapPoint*, Parked>& t = parked();
  for (int32_t i = 0; i < P; i++) {
    Parked& p = t[who[i]];
    p.obs.swap(snap[i]);
    p.best = best[i];
  }
}

void ccm_b200_prepare_point_updates(const std::vector<mpptr>& points) {
  ccm_b200_prepare_normals(points, nullptr);
  ccm_b200_prepare_descriptors(points);
}

void ccm_b200_clear_descriptors() { parked().clear(); }

void ccm_b200_descriptors_stats(unsigned long long* hits, unsigned long long* stale, unsigned long long* host) {
  if (hits) *hits = g_hits.load();
  if (stale) *stale = g_stale.load();
  if (host) *host = g_host.load();
}

void MapPoint::ComputeDistinctiveDescriptors() {
  std::map<kfptr, size_t> observations;
  {
    std::unique_lock<std::mutex> lock1(mMutexFeatures);
    if (mbBad) return;
    observations = mObservations;
  }
  if (observations.empty()) return;
  int32_t best = -1;
  bool have = false;
  std::unordered_map<const MapPoint*, Parked>& t = parked();
  std::unordered_map<const MapPoint*, Parked>::iterator it = t.empty() ? t.end() : t.find(this);
  if (it != t.end()) {
    have = same_list(it->second.obs, observations);
    if (have) { best = it->second.best; g_hits++; }
    else g_stale++;
    t.erase(it);
  }
  if (!have) {                                                     // the reference's own reads, one point on the host
    g_host++;
    FlatDescriptors f(false);
    f.add_point(observations);
    check(ccm_distinctive_descriptors_host((int32_t)f.bad.size(), f.bad.data(), 1, f.ptr.data(), f.obs.data(), f.desc.data(), &best, nullptr,
                                           nullptr),
          "ccm_distinctive_descriptors_host");
  }
  if (best < 0) return;                                            // every observer bad: vDescriptors empty, nothing written
  std::map<kfptr, size_t>::const_iterator o = observations.begin();
  std::advance(o, best);
  cv::Mat d = o->first->mDescriptors.row((int)o->second).clone();
  {
    std::unique_lock<std::mutex> lock(mMutexFeatures);
    mDescriptor = d;
  }
}

}  // namespace cslam

// MapPoint_shim.cpp — reference-side translation unit for MapPoint::UpdateNormalAndDepth (cslam/src/MapPoint.cpp:779-823).
//
// The body is deleted from MapPoint.cpp and defined here (the members it writes are protected and have no setter; a member body keeps
// MapPoint.h unchanged).  Two paths give the same members bit for bit:
//   * batched: the write-back loops of Optimizer_shim.cpp call ccm_b200_prepare_normals once before they start.  It flattens the
//     points (observers in mObservations order, each keyframe's centre and isBad() read once), makes one ccm_normal_depth call on the
//     GPU and parks the results per thread, with a snapshot of what they were computed from: position, observation count, pRefKF.
//     The member then writes the parked values when the snapshot still matches;
//   * parked by another batch: shim/Sim3Correction_shim.cpp computes the normals of the points a loop or merge correction moves in its
//     own device call and parks them through ccm_b200_park_normals, under the same snapshot rule;
//   * single point: every other caller (tracking, mapping, the communicator) and any
//     point whose snapshot went stale computes on the host through ccm_normal_depth_host, the same arithmetic.
// In this repository it is compiled against the stand-in MapPoint / KeyFrame of oracle/ref_stub_mp and run next to a literal
// restatement of the reference body by tests/test_normal_depth.py.
#include <cslam/KeyFrame.h>
#include <cslam/MapPoint.h>
#include <cslam/estd.h>

#include <atomic>
#include <iostream>
#include <unordered_map>
#include <vector>

#include "MapPoint_shim.h"
#include "ccm_b200.h"

namespace cslam {

namespace {

typedef boost::shared_ptr<KeyFrame> kfptr;
typedef boost::shared_ptr<MapPoint> mpptr;

struct Parked {
  float pos[3];
  size_t n_obs;
  const KeyFrame* ref;
  float normal[3], max_dist, min_dist;
};

std::unordered_map<const MapPoint*, Parked>& parked() {
  static thread_local std::unordered_map<const MapPoint*, Parked> table;
  return table;
}

// the flat arrays of include/ccm_b200.h's ccm_normal_depth
struct FlatNormals {
  std::vector<float> centre, pos, scale_ref, scale_last;
  std::vector<uint8_t> bad;
  std::vector<int64_t> ptr{0};
  std::vector<int32_t> obs, ref;
  std::unordered_map<const KeyFrame*, int32_t> row;

  int32_t add_kf(const kfptr& pKF) {
    std::unordered_map<const KeyFrame*, int32_t>::const_iterator it = row.find(pKF.get());
    if (it != row.end()) return it->second;
    const int32_t r = (int32_t)bad.size();
    row[pKF.get()] = r;
    const cv::Mat O = pKF->GetCameraCenter();
    for (int i = 0; i < 3; i++) centre.push_back(O.at<float>(i));
    bad.push_back(pKF->isBad() ? 1 : 0);
    return r;
  }
  // one point: observers in map order; the reference keyframe's octave from its own observation, or from keypoint 0 when it does not
  // observe the point (observations[pRefKF] inserts 0, MapPoint.cpp:813)
  void add_point(const std::map<kfptr, size_t>& observations, const kfptr& pRefKF, const float* X) {
    for (std::map<kfptr, size_t>::const_iterator it = observations.begin(); it != observations.end(); ++it) obs.push_back(add_kf(it->first));
    ptr.push_back((int64_t)obs.size());
    pos.insert(pos.end(), X, X + 3);
    ref.push_back(add_kf(pRefKF));
    std::map<kfptr, size_t>::const_iterator f = observations.find(pRefKF);
    const size_t idx = f == observations.end() ? 0 : f->second;
    scale_ref.push_back(pRefKF->mvScaleFactors[pRefKF->mvKeysUn[idx].octave]);
    scale_last.push_back(pRefKF->mvScaleFactors[pRefKF->mnScaleLevels - 1]);
  }
  int32_t n_points() const { return (int32_t)ref.size(); }
};

// as Optimizer_shim.cpp's check(): the reference's callers handle estd::infrastructure_ex
void check(int rc, const char* fn) {
  if (rc != CCM_OK) { std::cerr << "libccm_b200: " << fn << ": " << ccm_last_error() << std::endl; throw estd::infrastructure_ex(); }
}

// member calls by outcome, process-wide: a parked value written / a parked value found stale / computed on the host
std::atomic<unsigned long long> g_hits(0), g_stale(0), g_host(0);

// parks the values of point i (status[i] != 0) with the snapshot snap[i] (observation count, pRefKF) and the position pos[i]
void park(const std::vector<const MapPoint*>& who, const float* pos, std::vector<Parked>& snap, const float* normal, const float* dmax,
          const float* dmin, const uint8_t* status) {
  std::unordered_map<const MapPoint*, Parked>& t = parked();
  for (size_t i = 0; i < who.size(); i++) {
    if (!status[i]) continue;
    Parked& p = snap[i];
    for (int j = 0; j < 3; j++) { p.pos[j] = pos[3 * i + j]; p.normal[j] = normal[3 * i + j]; }
    p.max_dist = dmax[i]; p.min_dist = dmin[i];
    t[who[i]] = p;
  }
}

}  // namespace

void ccm_b200_prepare_normals(const std::vector<mpptr>& points, const float* new_pos) {
  FlatNormals f;
  std::vector<const MapPoint*> who;
  std::vector<Parked> snap;
  for (size_t i = 0; i < points.size(); i++) {
    const mpptr& pMP = points[i];
    if (!pMP || pMP->isBad()) continue;
    const std::map<kfptr, size_t> observations = pMP->GetObservations();
    const kfptr pRefKF = pMP->GetReferenceKeyFrame();
    if (observations.empty() || !pRefKF) continue;                 // the member returns before writing (or would fault) there
    Parked p;
    if (new_pos) for (int j = 0; j < 3; j++) p.pos[j] = new_pos[3 * i + j];
    else { const cv::Mat X = pMP->GetWorldPos(); for (int j = 0; j < 3; j++) p.pos[j] = X.at<float>(j); }
    p.n_obs = observations.size();
    p.ref = pRefKF.get();
    f.add_point(observations, pRefKF, p.pos);
    who.push_back(pMP.get());
    snap.push_back(p);
  }
  const int32_t P = f.n_points();
  if (P == 0) return;
  std::vector<float> normal((size_t)P * 3), dmax(P), dmin(P);
  std::vector<uint8_t> status(P);
  check(ccm_normal_depth((int32_t)f.bad.size(), f.centre.data(), f.bad.data(), P, f.pos.data(), f.ptr.data(), f.obs.data(), f.ref.data(),
                         f.scale_ref.data(), f.scale_last.data(), normal.data(), dmax.data(), dmin.data(), status.data()),
        "ccm_normal_depth");
  park(who, f.pos.data(), snap, normal.data(), dmax.data(), dmin.data(), status.data());
}

void ccm_b200_park_normals(const std::vector<mpptr>& points, const float* pos, const float* normal, const float* max_dist,
                           const float* min_dist, const uint8_t* status) {
  std::vector<const MapPoint*> who;
  std::vector<Parked> snap;
  std::vector<float> p_pos, p_normal, p_max, p_min;
  std::vector<uint8_t> p_status;
  for (size_t i = 0; i < points.size(); i++) {
    const mpptr& pMP = points[i];
    if (!pMP || !status[i]) continue;
    Parked p;
    p.n_obs = pMP->GetObservations().size();
    p.ref = pMP->GetReferenceKeyFrame().get();
    who.push_back(pMP.get());
    snap.push_back(p);
    p_pos.insert(p_pos.end(), pos + 3 * i, pos + 3 * i + 3);
    p_normal.insert(p_normal.end(), normal + 3 * i, normal + 3 * i + 3);
    p_max.push_back(max_dist[i]); p_min.push_back(min_dist[i]); p_status.push_back(1);
  }
  park(who, p_pos.data(), snap, p_normal.data(), p_max.data(), p_min.data(), p_status.data());
}

void ccm_b200_clear_normals() { parked().clear(); }

void ccm_b200_normals_stats(unsigned long long* hits, unsigned long long* stale, unsigned long long* host) {
  if (hits) *hits = g_hits.load();
  if (stale) *stale = g_stale.load();
  if (host) *host = g_host.load();
}

void MapPoint::UpdateNormalAndDepth() {
  float X[3];
  size_t n_obs;
  kfptr pRefKF;
  {
    std::unique_lock<std::mutex> lock1(mMutexFeatures);
    std::unique_lock<std::mutex> lock2(mMutexPos);
    if (mbBad) return;
    if (mObservations.empty()) return;
    n_obs = mObservations.size();
    pRefKF = mpRefKF;
    for (int j = 0; j < 3; j++) X[j] = mWorldPos.at<float>(j);
  }
  float normal[3], max_dist, min_dist;
  std::unordered_map<const MapPoint*, Parked>& t = parked();
  std::unordered_map<const MapPoint*, Parked>::iterator it = t.empty() ? t.end() : t.find(this);
  bool have = false;
  if (it != t.end()) {
    const Parked& p = it->second;
    have = p.pos[0] == X[0] && p.pos[1] == X[1] && p.pos[2] == X[2] && p.n_obs == n_obs && p.ref == pRefKF.get();
    if (have) {
      for (int j = 0; j < 3; j++) normal[j] = p.normal[j];
      max_dist = p.max_dist; min_dist = p.min_dist;
      g_hits++;
    } else {
      g_stale++;
    }
    t.erase(it);
  }
  if (!have) {                                                     // the reference's own reads, one point on the host
    std::map<kfptr, size_t> observations;
    {
      std::unique_lock<std::mutex> lock1(mMutexFeatures);
      std::unique_lock<std::mutex> lock2(mMutexPos);
      if (mbBad) return;
      observations = mObservations;
      pRefKF = mpRefKF;
      for (int j = 0; j < 3; j++) X[j] = mWorldPos.at<float>(j);
    }
    if (observations.empty()) return;
    g_host++;
    FlatNormals f;
    f.add_point(observations, pRefKF, X);
    uint8_t status = 0;
    check(ccm_normal_depth_host((int32_t)f.bad.size(), f.centre.data(), f.bad.data(), 1, f.pos.data(), f.ptr.data(), f.obs.data(), f.ref.data(),
                                f.scale_ref.data(), f.scale_last.data(), normal, &max_dist, &min_dist, &status),
          "ccm_normal_depth_host");
    if (!status) return;
  }
  std::unique_lock<std::mutex> lock3(mMutexPos);
  mfMaxDistance = max_dist;
  mfMinDistance = min_dist;
  mNormalVector.create(3, 1, CV_32F);
  for (int j = 0; j < 3; j++) mNormalVector.at<float>(j) = normal[j];
}

}  // namespace cslam

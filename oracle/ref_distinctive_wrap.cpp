// ref_distinctive_wrap.cpp — TEST INFRASTRUCTURE: stand-in MapPoint / KeyFrame scenes (oracle/ref_stub_dd) built from the flat arrays
// of synth.make_distinctive, and the ways to choose their descriptors:
//   dd_literal        the reference body (cslam/src/MapPoint.cpp:929-994) restated on the stand-ins, with its stack array, its
//                     vector<cv::Mat>, std::sort and vDists[0.5*(N-1)] as written; results go to arrays, the objects are not touched
//                     (the array takes 4 N^2 bytes of stack: N in the low thousands at most)
//   dd_shim           shim/MapPointDescriptor_shim.cpp's member on every point, optionally after the batched preparation
//   dd_shim_stale     prepare, then change every other point (observation replaced / observation added / point set bad), then the members
//   dd_search_in_neighbors, dd_establish   the loops of LocalMapping::SearchInNeighbors (cslam/src/Mapping.cpp:531-542) and
//                     KeyFrame::EstablishInitialConnectionsServer (cslam/src/KeyFrame.cpp:146-170), the latter as the reference runs it
//                     (literal body) or split as INTEGRATION.md §4d describes (shim)
// Keyframes live in one array in row order (with room for SPARE appended ones), so every std::map<kfptr> iterates its observers in
// ascending row (map_order scenes).  Every
// point also gets a position and a reference keyframe, so that shim/MapPoint_shim.cpp's member can run next to it.
#include <cslam/KeyFrame.h>
#include <cslam/MapPoint.h>

#include <algorithm>
#include <climits>
#include <cstdint>
#include <cstring>
#include <map>
#include <vector>

#include "../shim/MapPointDescriptor_shim.h"
#include "../shim/MapPoint_shim.h"

using namespace cslam;
using std::map;
using std::vector;
typedef boost::shared_ptr<KeyFrame> kfptr;
typedef boost::shared_ptr<MapPoint> mpptr;

static const int SPARE = 8;

struct Scene {
  std::vector<KeyFrame> kf_store;
  std::vector<kfptr> kfs;
  std::vector<mpptr> mps;
};

static void noop(KeyFrame*) {}

static int32_t add_keyframe(Scene* s, uint64_t uid, uint8_t bad, int32_t n, const uint8_t* desc) {
  const int32_t k = (int32_t)s->kfs.size();
  if ((size_t)k >= s->kf_store.size()) return -1;
  KeyFrame& kf = s->kf_store[k];
  kf.mUniqueId = (size_t)uid;
  kf.mbBad = bad != 0;
  kf.mDescriptors = cv::Mat(n, 32, CV_8U);
  if (n) std::memcpy(kf.mDescriptors.data, desc, 32 * (size_t)n);
  kf.Ow = cv::Mat(3, 1, CV_32F);
  for (int j = 0; j < 3; j++) kf.Ow.at<float>(j) = (float)((k * 7 + j * 3) % 11) - 5.f;
  kf.mvScaleFactors.assign(8, 1.f);
  for (int l = 1; l < 8; l++) kf.mvScaleFactors[l] = kf.mvScaleFactors[l - 1] * 1.2f;
  for (int i = 0; i < std::max(n, 1); i++) kf.mvKeysUn.push_back(cv::KeyPoint(0.f, 0.f, 7.f, -1.f, 0.f, (k + i) % 8));
  s->kfs.push_back(kfptr(&kf, noop));
  return k;
}

extern "C" void* dd_scene_create(int32_t K, const uint8_t* kf_bad, const uint64_t* kf_uid, const int64_t* kf_desc_ptr, const uint8_t* kf_desc,
                                 int32_t P, const uint8_t* mp_bad, const int64_t* obs_ptr, const int32_t* obs_kf, const int32_t* obs_feat) {
  Scene* s = new Scene();
  s->kf_store = std::vector<KeyFrame>(K + SPARE);
  for (int k = 0; k < K; k++)
    add_keyframe(s, kf_uid[k], kf_bad[k], (int32_t)(kf_desc_ptr[k + 1] - kf_desc_ptr[k]), kf_desc + 32 * kf_desc_ptr[k]);
  for (int i = 0; i < P; i++) {
    mpptr m(new MapPoint());
    cv::Mat X(3, 1, CV_32F);
    for (int j = 0; j < 3; j++) X.at<float>(j) = 20.f + (float)((i * 13 + j * 5) % 17);
    m->SetWorldPos(X, true);
    for (int64_t e = obs_ptr[i]; e < obs_ptr[i + 1]; e++) m->AddObservationForTest(s->kfs[obs_kf[e]], (size_t)obs_feat[e]);
    if (obs_ptr[i + 1] > obs_ptr[i]) m->SetReferenceForTest(s->kfs[obs_kf[obs_ptr[i]]]);
    else if (K) m->SetReferenceForTest(s->kfs[0]);               // the reference sets mpRefKF at construction
    m->SetBadForTest(mp_bad[i] != 0);
    s->mps.push_back(m);
  }
  return s;
}

extern "C" void dd_scene_destroy(void* h) { delete static_cast<Scene*>(h); }

// a keyframe appended to the scene (row returned, -1 past SPARE); it observes nothing until a test makes it
extern "C" int32_t dd_add_keyframe(void* h, uint64_t uid, uint8_t bad, int32_t n, const uint8_t* desc) {
  return add_keyframe(static_cast<Scene*>(h), uid, bad, n, desc);
}

extern "C" void dd_stats(unsigned long long* c) { ccm_b200_descriptors_stats(&c[0], &c[1], &c[2]); }
extern "C" void dd_nd_stats(unsigned long long* c) { ccm_b200_normals_stats(&c[0], &c[1], &c[2]); }
extern "C" void dd_register_store(void* store) { ccm_b200_register_kfstore(static_cast<ccm_kf_store*>(store)); }

// ORBmatcher::DescriptorDistance (cslam/src/ORBmatcher.cpp:1653-1669), the bit-parallel popcount of each 32-bit word
static int DescriptorDistance(const cv::Mat& a, const cv::Mat& b) {
  const int32_t* pa = a.ptr<int32_t>();
  const int32_t* pb = b.ptr<int32_t>();
  int dist = 0;
  for (int i = 0; i < 8; i++, pa++, pb++) {
    unsigned int v = *pa ^ *pb;
    v = v - ((v >> 1) & 0x55555555);
    v = (v & 0x33333333) + ((v >> 2) & 0x33333333);
    dist += (((v + (v >> 4)) & 0xF0F0F0F) * 0x1010101) >> 24;
  }
  return dist;
}

// MapPoint.cpp:929-994 on one stand-in point; false where the body returns before writing.  pos: the chosen observer's position in
// the observation list (bookkeeping for the comparison, not part of the body)
static bool literal_one(MapPoint* self, uint8_t* out, int32_t* out_pos, int32_t* out_median) {
  vector<cv::Mat> vDescriptors;
  vector<int32_t> vPos;
  map<kfptr, size_t> observations;
  {
    if (self->isBad()) return false;
    observations = self->GetObservations();
  }
  if (observations.empty()) return false;
  vDescriptors.reserve(observations.size());
  int32_t at = 0;
  for (map<kfptr, size_t>::iterator mit = observations.begin(), mend = observations.end(); mit != mend; mit++, at++) {
    kfptr pKF = mit->first;
    if (!pKF->isBad()) { vDescriptors.push_back(pKF->mDescriptors.row(mit->second)); vPos.push_back(at); }
  }
  if (vDescriptors.empty()) return false;
  const size_t N = vDescriptors.size();
  float Distances[N][N];
  for (size_t i = 0; i < N; i++) {
    Distances[i][i] = 0;
    for (size_t j = i + 1; j < N; j++) {
      int distij = DescriptorDistance(vDescriptors[i], vDescriptors[j]);
      Distances[i][j] = distij;
      Distances[j][i] = distij;
    }
  }
  int BestMedian = INT_MAX;
  int BestIdx = 0;
  for (size_t i = 0; i < N; i++) {
    vector<int> vDists(Distances[i], Distances[i] + N);
    std::sort(vDists.begin(), vDists.end());
    int median = vDists[0.5 * (N - 1)];
    if (median < BestMedian) {
      BestMedian = median;
      BestIdx = i;
    }
  }
  cv::Mat mDescriptor = vDescriptors[BestIdx].clone();
  std::memcpy(out, mDescriptor.data, 32);
  *out_pos = vPos[BestIdx];
  *out_median = BestMedian;
  return true;
}

extern "C" void dd_literal(void* h, int32_t* best, int32_t* median, uint8_t* desc) {
  Scene* s = static_cast<Scene*>(h);
  for (size_t i = 0; i < s->mps.size(); i++) {
    std::memset(desc + 32 * i, 0, 32);
    best[i] = -1; median[i] = 0;
    literal_one(s->mps[i].get(), desc + 32 * i, best + i, median + i);
  }
}

// mDescriptor as GetDescriptor() returns it: written 0 empty, 1 a continuous 1 x 32 CV_8U matrix, 2 anything else
static void read_members(Scene* s, uint8_t* desc, uint8_t* written) {
  for (size_t i = 0; i < s->mps.size(); i++) {
    const cv::Mat d = s->mps[i]->GetDescriptor();
    std::memset(desc + 32 * i, 0, 32);
    if (d.empty()) { written[i] = 0; continue; }
    written[i] = d.rows == 1 && d.cols == 32 && d.type() == CV_8U && d.isContinuous() ? 1 : 2;
    if (written[i] == 1) std::memcpy(desc + 32 * i, d.data, 32);
  }
}

// prepare: 0 member only (host path), 1 ccm_b200_prepare_descriptors first, 2 ccm_b200_prepare_point_updates first (both members then
// run, descriptors first, as the reference's loops call them); returns 0 or -1 on an exception
extern "C" int dd_shim(void* h, int prepare, uint8_t* desc, uint8_t* written) {
  Scene* s = static_cast<Scene*>(h);
  try {
    ParkedDescriptorsGuard guard;
    ParkedNormalsGuard nguard;
    if (prepare == 1) ccm_b200_prepare_descriptors(s->mps);
    if (prepare == 2) ccm_b200_prepare_point_updates(s->mps);
    for (size_t i = 0; i < s->mps.size(); i++) {
      s->mps[i]->ComputeDistinctiveDescriptors();
      if (prepare == 2) s->mps[i]->UpdateNormalAndDepth();
    }
  } catch (...) {
    return -1;
  }
  read_members(s, desc, written);
  return 0;
}

// prepare, then on every other point: kind 1 replace its first observation by feature (i % n) of keyframe row `kf` (same count),
// kind 2 add that observation, kind 3 set the point bad.  Then the members, as dd_shim.
extern "C" int dd_shim_stale(void* h, int kind, int32_t kf, uint8_t* desc, uint8_t* written) {
  Scene* s = static_cast<Scene*>(h);
  try {
    ParkedDescriptorsGuard guard;
    ccm_b200_prepare_descriptors(s->mps);
    const int n = s->kf_store[kf].mDescriptors.rows;
    for (size_t i = 0; i < s->mps.size(); i += 2) {
      MapPoint& m = *s->mps[i];
      const std::map<kfptr, size_t> obs = m.GetObservations();
      if (kind == 1 && !obs.empty()) { m.EraseObservationForTest(obs.begin()->first); m.AddObservationForTest(s->kfs[kf], i % n); }
      else if (kind == 2) m.AddObservationForTest(s->kfs[kf], i % n);
      else if (kind == 3) m.SetBadForTest(true);
    }
    for (size_t i = 0; i < s->mps.size(); i++) s->mps[i]->ComputeDistinctiveDescriptors();
  } catch (...) {
    return -1;
  }
  read_members(s, desc, written);
  return 0;
}

// SearchInNeighbors' update loop over the points pts[0..n) (repeats and bad points allowed), after one ccm_b200_prepare_point_updates
extern "C" int dd_search_in_neighbors(void* h, int32_t n, const int32_t* pts, uint8_t* desc, uint8_t* written) {
  Scene* s = static_cast<Scene*>(h);
  try {
    ParkedDescriptorsGuard guard;
    ParkedNormalsGuard nguard;
    std::vector<mpptr> vpMapPointMatches;
    for (int32_t i = 0; i < n; i++) vpMapPointMatches.push_back(s->mps[pts[i]]);
    ccm_b200_prepare_point_updates(vpMapPointMatches);
    for (size_t i = 0, iend = vpMapPointMatches.size(); i < iend; i++) {
      mpptr pMP = vpMapPointMatches[i];
      if (pMP && !pMP->isBad()) {
        pMP->ComputeDistinctiveDescriptors();
        pMP->UpdateNormalAndDepth();
      }
    }
  } catch (...) {
    return -1;
  }
  read_members(s, desc, written);
  return 0;
}

// EstablishInitialConnectionsServer for keyframe row `kf` whose mvpMapPoints[idx] is point mp_of_idx[idx] (-1: none).
// split 0: the reference's loop (AddObservation, then the literal body, per index); the chosen bytes of each point touched go to desc
// (the last call wins).  split 1: every AddObservation, one ccm_b200_prepare_point_updates, then both members per index; desc is
// each point's mDescriptor afterwards.  written[i] = 1 for the points touched.
extern "C" int dd_establish(void* h, int32_t kf, int32_t n_idx, const int32_t* mp_of_idx, int split, uint8_t* desc, uint8_t* written) {
  Scene* s = static_cast<Scene*>(h);
  const kfptr self = s->kfs[kf];
  std::vector<uint8_t> touched(s->mps.size(), 0);
  try {
    if (!split) {
      for (int32_t idx = 0; idx < n_idx; idx++) {
        if (mp_of_idx[idx] < 0) continue;
        MapPoint* pMPi = s->mps[mp_of_idx[idx]].get();
        pMPi->AddObservation(self, idx);
        int32_t pos, med;
        uint8_t d[32];
        if (literal_one(pMPi, d, &pos, &med)) std::memcpy(desc + 32 * (size_t)mp_of_idx[idx], d, 32);
        touched[mp_of_idx[idx]] = 1;
      }
      for (size_t i = 0; i < touched.size(); i++) written[i] = touched[i];
      return 0;
    }
    ParkedDescriptorsGuard guard;
    ParkedNormalsGuard nguard;
    std::vector<mpptr> batch;
    for (int32_t idx = 0; idx < n_idx; idx++) {
      if (mp_of_idx[idx] < 0) continue;
      s->mps[mp_of_idx[idx]]->AddObservation(self, idx);
      batch.push_back(s->mps[mp_of_idx[idx]]);
    }
    ccm_b200_prepare_point_updates(batch);
    for (int32_t idx = 0; idx < n_idx; idx++) {
      if (mp_of_idx[idx] < 0) continue;
      mpptr pMPi = s->mps[mp_of_idx[idx]];
      pMPi->ComputeDistinctiveDescriptors();
      pMPi->UpdateNormalAndDepth();
      touched[mp_of_idx[idx]] = 1;
    }
  } catch (...) {
    return -1;
  }
  std::vector<uint8_t> w(s->mps.size());
  read_members(s, desc, w.data());
  for (size_t i = 0; i < touched.size(); i++) written[i] = touched[i];
  return 0;
}

// kf_store.cu — device-resident keyframe features behind ccm_kfstore_* (include/ccm_b200.h); SURVEY.md §8(f) rank 4.
//
// On the server every keyframe arrives as a ccmslam_msgs::KF (cslam_msgs/msg/KF.msg) through Communicator::ProcessKfInServer
// (S/Communicator.cpp:815-1140); KeyFrame::WriteMembersFromMessage (S/KeyFrame.cpp:1662-1726) copies mvKeysUn and mDescriptors out of
// the message element by element, runs the vocabulary transform on them, and every later place-recognition / map-fusion matcher call
// reads the descriptors again from host memory.  Here the descriptors are uploaded ONCE, when the message arrives, straight from the
// message's own storage (ccmslam_msgs/Descriptor[] is n contiguous 32-byte records; ccmslam_msgs/CvKeyPoint[] is n packed 15-byte
// records on the wire), the BoW transform runs over the resident copy, and the server-side matchers name their operands by mUniqueId:
// no per-call host-to-device copy of either descriptor set.
//
// Device memory: slabs of 2^20 descriptors (32 MB), bump allocation inside a slab, first-fit reuse of erased ranges.  Tens of GB of HBM
// hold the descriptors of millions of keyframes; the store never moves a keyframe once placed (matchers may be running on it).
// Keypoints stay on the host (decoded once, as Converter::fromCvKeyPointMsg does, S/Converter.cc:180-192): the order-dependent
// selection halves of the matchers read angles / octaves there.
#include <memory>
#include <mutex>
#include <unordered_map>

#include "common.cuh"

namespace ccm {
const uint16_t* hamming_matrix_mixed(const uint8_t* A, const void* dA, int nA, const uint8_t* B, const void* dB, int nB);  // match.cu
int voc_transform_resident(ccm_voc_handle* h, const void* d_desc, int32_t n, int32_t levelsup, uint32_t* word_of_feat, uint32_t* node_of_feat,
                           double* weight_of_feat, uint32_t* bow_id, double* bow_val, int32_t* bow_n, uint32_t* fv_node_id,
                           int32_t* fv_node_ptr, uint32_t* fv_feat, int32_t* fv_n_nodes);                                  // voc.cu
}  // namespace ccm

using namespace ccm;

struct ccm_kf_store {
  static constexpr size_t SLAB = (size_t)1 << 20;  // descriptors per slab
  struct Range { int slab; size_t off, n; };
  struct Entry { Range r; std::vector<ccm_keypoint> kp; std::vector<float> angle; };
  std::vector<uint4*> slabs;       // cudaMalloc'ed, SLAB * 32 bytes each
  std::vector<size_t> slab_used;
  std::vector<Range> free_list;
  std::unordered_map<uint64_t, Entry> kf;
  cudaStream_t stream = nullptr;
  int device = 0;
  std::mutex mu;
  int64_t h2d_bytes = 0;

  ~ccm_kf_store() {
    for (uint4* p : slabs) cudaFree(p);
    if (stream) cudaStreamDestroy(stream);
  }
  const uint4* ptr(const Range& r) const { return slabs[r.slab] + r.off * 2; }
  Range take(size_t n) {
    for (size_t i = 0; i < free_list.size(); i++)
      if (free_list[i].n >= n) {
        Range r = free_list[i];
        if (r.n == n) free_list.erase(free_list.begin() + i);
        else { free_list[i].off += n; free_list[i].n -= n; }
        r.n = n;
        return r;
      }
    CCM_REQUIRE(n <= SLAB, "ccm_kfstore_put: more than 2^20 features in one keyframe");
    if (slabs.empty() || slab_used.back() + n > SLAB) {
      uint4* p = nullptr;
      CCM_CUDA(cudaMalloc((void**)&p, SLAB * 32));
      slabs.push_back(p); slab_used.push_back(0);
    }
    Range r{(int)slabs.size() - 1, slab_used.back(), n};
    slab_used.back() += n;
    return r;
  }
};

namespace ccm {
// the device address of each uid's first descriptor and its feature count (nullptr / -1: not in the store), for
// ccm_kfstore_distinctive_descriptors (distinctive.cu); read under the store's lock, like every matcher's operands
void kfstore_resolve(ccm_kf_store* s, int32_t n, const uint64_t* uid, std::vector<const uint4*>& base, std::vector<int32_t>& n_feat,
                     int* device) {
  std::lock_guard<std::mutex> lock(s->mu);
  base.assign(n, nullptr); n_feat.assign(n, -1);
  for (int32_t k = 0; k < n; k++) {
    auto it = s->kf.find(uid[k]);
    if (it == s->kf.end()) continue;
    n_feat[k] = (int32_t)it->second.r.n;
    base[k] = it->second.r.n ? s->ptr(it->second.r) : nullptr;
  }
  *device = s->device;
}
}  // namespace ccm

namespace {
// ccmslam_msgs/CvKeyPoint as ROS serialises it: f32 x, f32 y, u8 size, f32 angle, u8 response, i8 octave (15 bytes, packed)
constexpr int WIRE_KP = 15;
void decode_wire_keypoint(const uint8_t* w, ccm_keypoint* k) {   // Converter::fromCvKeyPointMsg, S/Converter.cc:180-192
  memcpy(&k->x, w, 4); memcpy(&k->y, w + 4, 4);
  k->size = (float)w[8];
  memcpy(&k->angle, w + 9, 4);
  k->response = (float)w[13];
  k->octave = (int32_t)(int8_t)w[14];
}
void put(ccm_kf_store* s, uint64_t uid, int32_t n, std::vector<ccm_keypoint>&& kps, const uint8_t* desc) {
  ensure_device();
  std::lock_guard<std::mutex> lock(s->mu);
  CCM_CUDA(cudaSetDevice(s->device));
  auto it = s->kf.find(uid);
  if (it != s->kf.end()) {                         // the same keyframe again (an update message): same place if the size allows
    if (it->second.r.n != (size_t)n) { if (it->second.r.n) s->free_list.push_back(it->second.r); s->kf.erase(it); it = s->kf.end(); }
  }
  ccm_kf_store::Entry* e;
  if (it == s->kf.end()) {
    ccm_kf_store::Entry ne;
    ne.r = n > 0 ? s->take((size_t)n) : ccm_kf_store::Range{0, 0, 0};
    e = &(s->kf[uid] = std::move(ne));
  } else e = &it->second;
  e->kp = std::move(kps);
  e->angle.resize(n);
  for (int i = 0; i < n; i++) e->angle[i] = e->kp[i].angle;
  if (n > 0) {
    CCM_CUDA(cudaMemcpyAsync(const_cast<uint4*>(s->ptr(e->r)), desc, (size_t)n * 32, cudaMemcpyHostToDevice, s->stream));
    CCM_CUDA(cudaStreamSynchronize(s->stream));    // the message buffer may be released by the caller after the call
    s->h2d_bytes += (int64_t)n * 32;
  }
}
const ccm_kf_store::Entry& get(ccm_kf_store* s, uint64_t uid, const char* what) {
  auto it = s->kf.find(uid);
  CCM_REQUIRE(it != s->kf.end(), what);
  return it->second;
}
}  // namespace

extern "C" {

int ccm_kfstore_create(ccm_kf_store** out) {
  return guarded([&] {
    CCM_REQUIRE(out, "ccm_kfstore_create: null output");
    *out = nullptr;
    ensure_device();
    std::unique_ptr<ccm_kf_store> s(new ccm_kf_store);
    s->device = current_device();
    CCM_CUDA(cudaStreamCreateWithFlags(&s->stream, cudaStreamNonBlocking));
    *out = s.release();
  });
}
void ccm_kfstore_destroy(ccm_kf_store* s) { delete s; }

int ccm_kfstore_put_wire(ccm_kf_store* s, uint64_t uid, int32_t n, const uint8_t* keypoints_wire, const uint8_t* descriptors,
                         ccm_keypoint* kp_out) {
  return guarded([&] {
    CCM_REQUIRE(s && n >= 0 && (n == 0 || (keypoints_wire && descriptors)), "ccm_kfstore_put_wire: bad argument");
    std::vector<ccm_keypoint> kps(n);
    for (int i = 0; i < n; i++) decode_wire_keypoint(keypoints_wire + (size_t)i * WIRE_KP, &kps[i]);
    if (kp_out && n) memcpy(kp_out, kps.data(), sizeof(ccm_keypoint) * n);
    put(s, uid, n, std::move(kps), descriptors);
  });
}

int ccm_wire_keypoints_decode(const uint8_t* keypoints_wire, int32_t n, ccm_keypoint* out) {
  return guarded([&] {
    CCM_REQUIRE(n >= 0 && (n == 0 || (keypoints_wire && out)), "ccm_wire_keypoints_decode: bad argument");
    for (int i = 0; i < n; i++) decode_wire_keypoint(keypoints_wire + (size_t)i * WIRE_KP, out + i);
  });
}

int ccm_kfstore_put(ccm_kf_store* s, uint64_t uid, int32_t n, const ccm_keypoint* kps, const uint8_t* descriptors) {
  return guarded([&] {
    CCM_REQUIRE(s && n >= 0 && (n == 0 || (kps && descriptors)), "ccm_kfstore_put: bad argument");
    put(s, uid, n, std::vector<ccm_keypoint>(kps, kps + n), descriptors);
  });
}

int ccm_kfstore_erase(ccm_kf_store* s, uint64_t uid) {
  return guarded([&] {
    CCM_REQUIRE(s, "ccm_kfstore_erase: null store");
    std::lock_guard<std::mutex> lock(s->mu);
    auto it = s->kf.find(uid);
    if (it == s->kf.end()) return;                  // erasing what is not there is a no-op, as in the reference's containers
    if (it->second.r.n) s->free_list.push_back(it->second.r);
    s->kf.erase(it);
  });
}

int32_t ccm_kfstore_features(ccm_kf_store* s, uint64_t uid) {
  if (!s) return -1;
  std::lock_guard<std::mutex> lock(s->mu);
  auto it = s->kf.find(uid);
  return it == s->kf.end() ? -1 : (int32_t)it->second.r.n;
}
int64_t ccm_kfstore_keyframes(ccm_kf_store* s) { if (!s) return -1; std::lock_guard<std::mutex> lock(s->mu); return (int64_t)s->kf.size(); }
int64_t ccm_kfstore_h2d_bytes(ccm_kf_store* s) { if (!s) return -1; std::lock_guard<std::mutex> lock(s->mu); return s->h2d_bytes; }

int ccm_kfstore_get(ccm_kf_store* s, uint64_t uid, ccm_keypoint* kps, uint8_t* descriptors) {
  return guarded([&] {
    CCM_REQUIRE(s, "ccm_kfstore_get: null store");
    std::lock_guard<std::mutex> lock(s->mu);
    const auto& e = get(s, uid, "ccm_kfstore_get: unknown keyframe");
    if (kps && e.r.n) memcpy(kps, e.kp.data(), sizeof(ccm_keypoint) * e.r.n);
    if (descriptors && e.r.n) {
      CCM_CUDA(cudaSetDevice(s->device));
      CCM_CUDA(cudaMemcpyAsync(descriptors, s->ptr(e.r), e.r.n * 32, cudaMemcpyDeviceToHost, s->stream));
      CCM_CUDA(cudaStreamSynchronize(s->stream));
    }
  });
}

// D[i * n2 + j] = DescriptorDistance(kf1 feature i, kf2 feature j); both operands resident
int ccm_kfstore_hamming(ccm_kf_store* s, uint64_t uid1, uint64_t uid2, uint16_t* D) {
  return guarded([&] {
    CCM_REQUIRE(s && D, "ccm_kfstore_hamming: null argument");
    const uint4 *p1, *p2; int n1, n2;
    {
      std::lock_guard<std::mutex> lock(s->mu);
      const auto& a = get(s, uid1, "ccm_kfstore_hamming: unknown keyframe"); const auto& b = get(s, uid2, "ccm_kfstore_hamming: unknown keyframe");
      p1 = a.r.n ? s->ptr(a.r) : nullptr; p2 = b.r.n ? s->ptr(b.r) : nullptr; n1 = (int)a.r.n; n2 = (int)b.r.n;
    }
    if (!n1 || !n2) return;
    const uint16_t* h = hamming_matrix_mixed(nullptr, p1, n1, nullptr, p2, n2);
    memcpy(D, h, (size_t)n1 * n2 * sizeof(uint16_t));
  });
}

// host query descriptors (a frame, a set of map-point descriptors) against a resident keyframe: D[i * n + j], i over the queries
int ccm_kfstore_hamming_query(ccm_kf_store* s, const uint8_t* Q, int32_t nQ, uint64_t uid, uint16_t* D) {
  return guarded([&] {
    CCM_REQUIRE(s && D && nQ >= 0 && (nQ == 0 || Q), "ccm_kfstore_hamming_query: bad argument");
    const uint4* p; int n;
    {
      std::lock_guard<std::mutex> lock(s->mu);
      const auto& a = get(s, uid, "ccm_kfstore_hamming_query: unknown keyframe");
      p = a.r.n ? s->ptr(a.r) : nullptr; n = (int)a.r.n;
    }
    if (!n || !nQ) return;
    const uint16_t* h = hamming_matrix_mixed(Q, nullptr, nQ, nullptr, p, n);
    memcpy(D, h, (size_t)nQ * n * sizeof(uint16_t));
  });
}

// ORBmatcher::SearchByBoW(kfptr, kfptr, vpMatches12) (S/ORBmatcher.cpp:565-698) between two resident keyframes: distances on the device
// from the resident descriptors, angles from the stored keypoints; has_mp (which features carry a good map point) changes while the
// map lives and comes with the call, as do the FeatureVectors (ccm_kfstore_transform hands them out at ingest).
int ccm_kfstore_match_bow_kf_kf(ccm_kf_store* s, uint64_t uid1, const uint8_t* has_mp1, const ccm_feature_vector* fv1, uint64_t uid2,
                                const uint8_t* has_mp2, const ccm_feature_vector* fv2, float nnratio, int32_t check_orientation,
                                int32_t* match12, int32_t* nmatches) {
  const uint4 *p1 = nullptr, *p2 = nullptr; int n1 = 0, n2 = 0;
  std::vector<float> a1, a2;
  int rc = guarded([&] {
    CCM_REQUIRE(s, "ccm_kfstore_match_bow_kf_kf: null store");
    std::lock_guard<std::mutex> lock(s->mu);
    const auto& a = get(s, uid1, "ccm_kfstore_match_bow_kf_kf: unknown keyframe"); const auto& b = get(s, uid2, "ccm_kfstore_match_bow_kf_kf: unknown keyframe");
    p1 = a.r.n ? s->ptr(a.r) : nullptr; p2 = b.r.n ? s->ptr(b.r) : nullptr; n1 = (int)a.r.n; n2 = (int)b.r.n;
    a1 = a.angle; a2 = b.angle;
  });
  if (rc != CCM_OK) return rc;
  const uint16_t* D = nullptr;
  rc = guarded([&] { if (n1 && n2) D = hamming_matrix_mixed(nullptr, p1, n1, nullptr, p2, n2); });
  if (rc != CCM_OK) return rc;
  return ccm_select_bow_kf_kf(D, n1, has_mp1, a1.data(), fv1, n2, has_mp2, a2.data(), fv2, nnratio, check_orientation, match12, nmatches);
}

// the BoW transform of KeyFrame::WriteMembersFromMessage (S/KeyFrame.cpp:1723-1726) over the resident descriptors
int ccm_kfstore_transform(ccm_kf_store* s, uint64_t uid, ccm_voc_handle* voc, int32_t levelsup, uint32_t* word_of_feat, uint32_t* node_of_feat,
                          double* weight_of_feat, uint32_t* bow_id, double* bow_val, int32_t* bow_n, uint32_t* fv_node_id,
                          int32_t* fv_node_ptr, uint32_t* fv_feat, int32_t* fv_n_nodes) {
  const uint4* p = nullptr; int n = 0;
  int rc = guarded([&] {
    CCM_REQUIRE(s && voc, "ccm_kfstore_transform: null argument");
    std::lock_guard<std::mutex> lock(s->mu);
    const auto& a = get(s, uid, "ccm_kfstore_transform: unknown keyframe");
    p = a.r.n ? s->ptr(a.r) : nullptr; n = (int)a.r.n;
  });
  if (rc != CCM_OK) return rc;
  return voc_transform_resident(voc, p, n, levelsup, word_of_feat, node_of_feat, weight_of_feat, bow_id, bow_val, bow_n, fv_node_id, fv_node_ptr,
                                fv_feat, fv_n_nodes);
}

}  // extern "C"

// sim3_correction.cu — the Sim3 correction pass of the loop closure and the map merge, behind ccm_sim3_correction /
// ccm_sim3_correction_host (include/ccm_b200.h).
//
//   LoopFinder::CorrectLoop  cslam/src/LoopFinder.cpp:568-613      MapMerger::MergeMaps  cslam/src/MapMerger.cpp:349-395
//
// The reference walks CorrectedSim3 in map order; its only order dependences are the claim of each point by the first entry that
// lists it and the mix of corrected and pre-loop centres its normal reads (sim3_correction_math.cuh).  Both are functions of entry
// indices, so the walk becomes three launches on one stream whatever the size:
//   k_sc_entries  one thread per entry: pose, centre and Swi; the same grid also sets every point's claim to "none"
//   k_sc_claim    one thread per mvpMapPoints slot: atomicMin of the entry index into the point's claim (the minimum does not depend on
//                 the order the atomics land in, so the result is deterministic)
//   k_sc_points   one thread per point: move it with its claiming entry's pair, then UpdateNormalAndDepth with the centre rule
// One pinned upload of every input, one download of every output.  The host entry point runs the same three phases as loops.
#include <algorithm>
#include <climits>
#include <string>
#include <vector>

#include "common.cuh"
#include "sim3_correction_math.cuh"

using namespace ccm;

namespace {

constexpr int CTA = 256;
constexpr int32_t NO_CLAIM = INT_MAX;

struct In {                     // device addresses of the uploaded block
  const float* kf_centre;
  const uint8_t* kf_bad;
  const int32_t* kf_entry;
  const double* Siw_new;
  const double* Siw_old;
  const int64_t* slot_ptr;
  const int32_t* slot_mp;
  const float* mp_pos;
  const uint8_t* mp_skip;
  const int64_t* obs_ptr;
  const int32_t* obs_kf;
  const int32_t* mp_ref;
  const float* scale_ref;
  const float* scale_last;
};

struct Out {                    // device addresses of the output block (downloaded as one)
  float* Tcw;                   // [n_e][16]
  float* centre;                // [n_e][3]
  int32_t* mp_entry;            // [n_mp], the claim while the kernels run
  float* pos;                   // [n_mp][3]
  float* normal;                // [n_mp][3]
  float* max_dist;
  float* min_dist;
  uint8_t* status;
};

__global__ void __launch_bounds__(CTA) k_sc_entries(int32_t n_e, int32_t n_mp, In in, Out out, double* __restrict__ Swi) {
  const int32_t n = max(n_e, n_mp);
  for (int32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    if (i < n_mp) out.mp_entry[i] = NO_CLAIM;
    if (i < n_e) {
      S3 w;
      sc::entry_pose(s3_load(in.Siw_new + 8 * (size_t)i), out.Tcw + 16 * (size_t)i, out.centre + 3 * (size_t)i, &w);
      s3_store(w, Swi + 8 * (size_t)i);
    }
  }
}

__global__ void __launch_bounds__(CTA) k_sc_claim(int32_t n_e, int64_t n_slots, In in, Out out) {
  for (int64_t j = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; j < n_slots; j += (int64_t)gridDim.x * blockDim.x) {
    const int32_t p = __ldg(in.slot_mp + j);
    if (p < 0 || __ldg(in.mp_skip + p)) continue;
    int32_t lo = 0, hi = n_e;    // the entry e with slot_ptr[e] <= j < slot_ptr[e + 1]
    while (hi - lo > 1) {
      const int32_t mid = (lo + hi) >> 1;
      if (__ldg(in.slot_ptr + mid) <= j) lo = mid; else hi = mid;
    }
    atomicMin(out.mp_entry + p, lo);
  }
}

__global__ void __launch_bounds__(CTA) k_sc_points(int32_t n_mp, In in, Out out, const double* __restrict__ Swi) {
  for (int32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n_mp; i += gridDim.x * blockDim.x) {
    const int32_t c = out.mp_entry[i];
    float X[3] = {in.mp_pos[3 * (size_t)i], in.mp_pos[3 * (size_t)i + 1], in.mp_pos[3 * (size_t)i + 2]};
    float nv[3] = {0.f, 0.f, 0.f}, dmax = 0.f, dmin = 0.f;
    uint8_t st = 0;
    if (c != NO_CLAIM) {
      const float P[3] = {X[0], X[1], X[2]};
      sc::move_point(s3_load(in.Siw_old + 8 * (size_t)c), s3_load(Swi + 8 * (size_t)c), P, X);
      const sc::ClaimCentres at{in.kf_centre, out.centre, in.kf_entry, c};
      st = nd::update_point(X, in.obs_kf, in.obs_ptr[i], in.obs_ptr[i + 1], at, in.kf_bad, in.mp_ref[i], in.scale_ref[i], in.scale_last[i], nv,
                            &dmax, &dmin);
      if (!st) { nv[0] = nv[1] = nv[2] = 0.f; dmax = dmin = 0.f; }
    }
    out.mp_entry[i] = c == NO_CLAIM ? -1 : c;
    out.pos[3 * (size_t)i] = X[0]; out.pos[3 * (size_t)i + 1] = X[1]; out.pos[3 * (size_t)i + 2] = X[2];
    out.normal[3 * (size_t)i] = nv[0]; out.normal[3 * (size_t)i + 1] = nv[1]; out.normal[3 * (size_t)i + 2] = nv[2];
    out.max_dist[i] = dmax; out.min_dist[i] = dmin; out.status[i] = st;
  }
}

struct Args {
  int32_t n_kf;
  const float* kf_centre;
  const uint8_t* kf_bad;
  int32_t n_e;
  const int32_t* entry_kf;
  const double* Siw_new;
  const double* Siw_old;
  const int64_t* slot_ptr;
  const int32_t* slot_mp;
  int32_t n_mp;
  const float* mp_pos;
  const uint8_t* mp_skip;
  const int64_t* obs_ptr;
  const int32_t* obs_kf;
  const int32_t* mp_ref;
  const float* scale_ref;
  const float* scale_last;
  float* entry_Tcw;
  float* entry_centre;
  int32_t* mp_entry;
  float* mp_pos_out;
  float* normal;
  float* max_dist;
  float* min_dist;
  uint8_t* status;
  int64_t n_slots() const { return n_e ? slot_ptr[n_e] : 0; }
  int64_t n_obs() const { return n_mp ? obs_ptr[n_mp] : 0; }
};

// Everything the reference could not have been handed: rows out of range, a keyframe listed twice (map keys are unique), null arrays.
// Returns kf_entry, the entry of each keyframe row (-1: none).  Throws before any output is written.
std::vector<int32_t> validate(const std::string& f, const Args& a) {
  CCM_REQUIRE(a.n_kf >= 0 && a.n_e >= 0 && a.n_mp >= 0, f + ": negative size");
  CCM_REQUIRE(a.n_kf == 0 || (a.kf_centre && a.kf_bad), f + ": null keyframe array");
  CCM_REQUIRE(a.slot_ptr, f + ": null slot_ptr");
  CCM_REQUIRE(a.n_e == 0 || (a.entry_kf && a.Siw_new && a.Siw_old && a.entry_Tcw && a.entry_centre), f + ": null entry array");
  CCM_REQUIRE(a.n_mp == 0 || (a.mp_pos && a.mp_skip && a.obs_ptr && a.mp_ref && a.scale_ref && a.scale_last && a.mp_entry && a.mp_pos_out &&
                              a.normal && a.max_dist && a.min_dist && a.status),
              f + ": null point array");
  std::vector<int32_t> kf_entry((size_t)a.n_kf, -1);
  CCM_REQUIRE(a.slot_ptr[0] == 0, f + ": slot_ptr[0] must be 0");
  for (int32_t e = 0; e < a.n_e; e++) {
    const int32_t k = a.entry_kf[e];
    CCM_REQUIRE(k >= 0 && k < a.n_kf, f + ": entry " + std::to_string(e) + ": keyframe row " + std::to_string(k) + " out of range");
    CCM_REQUIRE(kf_entry[k] < 0, f + ": entry " + std::to_string(e) + ": keyframe row " + std::to_string(k) + " is already entry " +
                                     std::to_string(kf_entry[k]));
    kf_entry[k] = e;
    CCM_REQUIRE(a.slot_ptr[e + 1] >= a.slot_ptr[e], f + ": entry " + std::to_string(e) + ": slot_ptr is not monotone");
  }
  const int64_t S = a.n_slots();
  CCM_REQUIRE(S == 0 || a.slot_mp, f + ": null slot_mp");
  for (int32_t e = 0; e < a.n_e; e++)
    for (int64_t j = a.slot_ptr[e]; j < a.slot_ptr[e + 1]; j++)
      CCM_REQUIRE(a.slot_mp[j] >= -1 && a.slot_mp[j] < a.n_mp, f + ": entry " + std::to_string(e) + ", slot " + std::to_string(j - a.slot_ptr[e]) +
                                                                   ": point row " + std::to_string(a.slot_mp[j]) + " out of range");
  if (a.n_mp == 0) return kf_entry;
  CCM_REQUIRE(a.obs_ptr[0] == 0, f + ": obs_ptr[0] must be 0");
  for (int32_t i = 0; i < a.n_mp; i++) CCM_REQUIRE(a.obs_ptr[i + 1] >= a.obs_ptr[i], f + ": point " + std::to_string(i) + ": obs_ptr is not monotone");
  CCM_REQUIRE(a.n_obs() == 0 || a.obs_kf, f + ": null obs_kf");
  for (int32_t i = 0; i < a.n_mp; i++) {
    CCM_REQUIRE(a.mp_ref[i] >= -1 && a.mp_ref[i] < a.n_kf, f + ": point " + std::to_string(i) + ": reference row " + std::to_string(a.mp_ref[i]) +
                                                           " out of range");
    for (int64_t j = a.obs_ptr[i]; j < a.obs_ptr[i + 1]; j++)
      CCM_REQUIRE(a.obs_kf[j] >= 0 && a.obs_kf[j] < a.n_kf, f + ": point " + std::to_string(i) + ": observer row " + std::to_string(a.obs_kf[j]) +
                                                            " out of range");
  }
  return kf_entry;
}

// the block the kernels read, in one layout for measuring and for filling
void pack(Packer& pk, const Args& a, const std::vector<int32_t>& kf_entry, In* in) {
  const size_t K = (size_t)a.n_kf, E = (size_t)a.n_e, P = (size_t)a.n_mp;
  in->kf_centre = pk.put(a.kf_centre, 3 * K);
  in->kf_bad = pk.put(a.kf_bad, K);
  in->kf_entry = pk.put(kf_entry.data(), K);
  in->Siw_new = pk.put(a.Siw_new, 8 * E);
  in->Siw_old = pk.put(a.Siw_old, 8 * E);
  in->slot_ptr = pk.put(a.slot_ptr, E + 1);
  in->slot_mp = pk.put(a.slot_mp, (size_t)a.n_slots());
  in->mp_pos = pk.put(a.mp_pos, 3 * P);
  in->mp_skip = pk.put(a.mp_skip, P);
  in->obs_ptr = pk.put(a.obs_ptr, P ? P + 1 : 0);
  in->obs_kf = pk.put(a.obs_kf, (size_t)a.n_obs());
  in->mp_ref = pk.put(a.mp_ref, P);
  in->scale_ref = pk.put(a.scale_ref, P);
  in->scale_last = pk.put(a.scale_last, P);
}

// offsets of each output in the output block: the downloaded part, then Swi, which only the kernels use
struct OutLayout {
  size_t Tcw, centre, mp_entry, pos, normal, max_dist, min_dist, status, down, swi, bytes;
  explicit OutLayout(const Args& a) {
    Packer pk;
    const size_t E = (size_t)a.n_e, P = (size_t)a.n_mp;
    Tcw = pk.reserve(16 * E * sizeof(float)); centre = pk.reserve(3 * E * sizeof(float)); mp_entry = pk.reserve(P * sizeof(int32_t));
    pos = pk.reserve(3 * P * sizeof(float)); normal = pk.reserve(3 * P * sizeof(float)); max_dist = pk.reserve(P * sizeof(float));
    min_dist = pk.reserve(P * sizeof(float)); status = pk.reserve(P);
    down = pk.at;
    swi = pk.reserve(8 * E * sizeof(double));
    bytes = pk.at;
  }
  Out at(uint8_t* base) const {
    return Out{reinterpret_cast<float*>(base + Tcw), reinterpret_cast<float*>(base + centre), reinterpret_cast<int32_t*>(base + mp_entry),
               reinterpret_cast<float*>(base + pos), reinterpret_cast<float*>(base + normal), reinterpret_cast<float*>(base + max_dist),
               reinterpret_cast<float*>(base + min_dist), base + status};
  }
};

void scatter(const Args& a, const Out& o) {
  const size_t E = (size_t)a.n_e, P = (size_t)a.n_mp;
  if (E) { memcpy(a.entry_Tcw, o.Tcw, 16 * E * sizeof(float)); memcpy(a.entry_centre, o.centre, 3 * E * sizeof(float)); }
  if (P) {
    memcpy(a.mp_entry, o.mp_entry, P * sizeof(int32_t)); memcpy(a.mp_pos_out, o.pos, 3 * P * sizeof(float));
    memcpy(a.normal, o.normal, 3 * P * sizeof(float)); memcpy(a.max_dist, o.max_dist, P * sizeof(float));
    memcpy(a.min_dist, o.min_dist, P * sizeof(float)); memcpy(a.status, o.status, P);
  }
}

// per-thread staging (Staging): a merge corrects a whole map, a loop a few dozen keyframes
thread_local Staging t_stage;

}  // namespace

extern "C" int ccm_sim3_correction_host(int32_t n_kf, const float* kf_centre, const uint8_t* kf_bad, int32_t n_e, const int32_t* entry_kf,
                                        const double* entry_Siw_new, const double* entry_Siw_old, const int64_t* slot_ptr, const int32_t* slot_mp,
                                        int32_t n_mp, const float* mp_pos, const uint8_t* mp_skip, const int64_t* obs_ptr, const int32_t* obs_kf,
                                        const int32_t* mp_ref, const float* mp_scale_ref, const float* mp_scale_last, float* entry_Tcw,
                                        float* entry_centre, int32_t* mp_entry, float* mp_pos_out, float* normal, float* max_dist,
                                        float* min_dist, uint8_t* status) {
  return guarded([&] {
    const Args a{n_kf, kf_centre, kf_bad, n_e, entry_kf, entry_Siw_new, entry_Siw_old, slot_ptr, slot_mp, n_mp, mp_pos, mp_skip, obs_ptr,
                 obs_kf, mp_ref, mp_scale_ref, mp_scale_last, entry_Tcw, entry_centre, mp_entry, mp_pos_out, normal, max_dist, min_dist, status};
    const std::vector<int32_t> kf_entry = validate("ccm_sim3_correction_host", a);
    std::vector<S3> swi((size_t)n_e);
    for (int32_t e = 0; e < n_e; e++) sc::entry_pose(s3_load(entry_Siw_new + 8 * (size_t)e), entry_Tcw + 16 * (size_t)e, entry_centre + 3 * (size_t)e, &swi[e]);
    for (int32_t i = 0; i < n_mp; i++) mp_entry[i] = -1;
    for (int32_t e = 0; e < n_e; e++)
      for (int64_t j = slot_ptr[e]; j < slot_ptr[e + 1]; j++) {
        const int32_t p = slot_mp[j];
        if (p >= 0 && !mp_skip[p] && mp_entry[p] < 0) mp_entry[p] = e;
      }
    for (int32_t i = 0; i < n_mp; i++) {
      const int32_t c = mp_entry[i];
      float* X = mp_pos_out + 3 * (size_t)i;
      float* nv = normal + 3 * (size_t)i;
      X[0] = mp_pos[3 * (size_t)i]; X[1] = mp_pos[3 * (size_t)i + 1]; X[2] = mp_pos[3 * (size_t)i + 2];
      nv[0] = nv[1] = nv[2] = 0.f; max_dist[i] = min_dist[i] = 0.f; status[i] = 0;
      if (c < 0) continue;
      sc::move_point(s3_load(entry_Siw_old + 8 * (size_t)c), swi[c], mp_pos + 3 * (size_t)i, X);
      const sc::ClaimCentres at{kf_centre, entry_centre, kf_entry.data(), c};
      status[i] = nd::update_point(X, obs_kf, obs_ptr[i], obs_ptr[i + 1], at, kf_bad, mp_ref[i], mp_scale_ref[i], mp_scale_last[i], nv,
                                   max_dist + i, min_dist + i);
      if (!status[i]) { nv[0] = nv[1] = nv[2] = 0.f; max_dist[i] = min_dist[i] = 0.f; }
    }
  });
}

extern "C" int ccm_sim3_correction(int32_t n_kf, const float* kf_centre, const uint8_t* kf_bad, int32_t n_e, const int32_t* entry_kf,
                                   const double* entry_Siw_new, const double* entry_Siw_old, const int64_t* slot_ptr, const int32_t* slot_mp,
                                   int32_t n_mp, const float* mp_pos, const uint8_t* mp_skip, const int64_t* obs_ptr, const int32_t* obs_kf,
                                   const int32_t* mp_ref, const float* mp_scale_ref, const float* mp_scale_last, float* entry_Tcw,
                                   float* entry_centre, int32_t* mp_entry, float* mp_pos_out, float* normal, float* max_dist, float* min_dist,
                                   uint8_t* status) {
  return guarded([&] {
    const Args a{n_kf, kf_centre, kf_bad, n_e, entry_kf, entry_Siw_new, entry_Siw_old, slot_ptr, slot_mp, n_mp, mp_pos, mp_skip, obs_ptr,
                 obs_kf, mp_ref, mp_scale_ref, mp_scale_last, entry_Tcw, entry_centre, mp_entry, mp_pos_out, normal, max_dist, min_dist, status};
    const std::vector<int32_t> kf_entry = validate("ccm_sim3_correction", a);
    ensure_device();
    if (n_e == 0 && n_mp == 0) return;

    Staging& s = t_stage;
    In in{};
    const OutLayout ol(a);
    s.run([&] {
      s.upload([&](Packer& pk) { pack(pk, a, kf_entry, &in); }, ol.bytes, ol.down);
      const Out out = ol.at(s.out.p);
      double* swi = reinterpret_cast<double*>(s.out.p + ol.swi);
      k_sc_entries<<<grid_size(std::max(n_e, n_mp), CTA), CTA, 0, s.stream>>>(n_e, n_mp, in, out, swi);
      CCM_LAUNCHED();
      k_sc_claim<<<grid_size(a.n_slots(), CTA), CTA, 0, s.stream>>>(n_e, a.n_slots(), in, out);
      CCM_LAUNCHED();
      k_sc_points<<<grid_size(n_mp, CTA), CTA, 0, s.stream>>>(n_mp, in, out, swi);
      CCM_LAUNCHED();
      CCM_CUDA(cudaMemcpyAsync(s.h_out, s.out.p, ol.down, cudaMemcpyDeviceToHost, s.stream));
      CCM_CUDA(cudaStreamSynchronize(s.stream));
    });
    scatter(a, ol.at(s.h_out));
  });
}

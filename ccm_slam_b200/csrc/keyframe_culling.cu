// keyframe_culling.cu — the redundancy test of LocalMapping::KeyFrameCullingV3 (cslam/src/Mapping.cpp:771-863) for every candidate in
// one call, behind ccm_keyframe_culling / ccm_keyframe_culling_host (include/ccm_b200.h).
//
//   k_kc_count   one CTA per candidate: each thread takes slots, reads the slot's point and walks its observers through the CSR up to
//                th_obs (keyframe_culling_math.cuh); two integer block reductions give nMPs and nRedundant, so the bytes do not depend
//                on the schedule
//   settle       on the host, before the call returns: the candidates in order, each effective cull applied to the points it reaches
//                and every later candidate with a touched slot point counted again over the state as it then stands
// One pinned upload of every input the kernel reads, one launch, one download of the two counts.  The host entry point counts with a
// loop and runs the same settle.
#include <string>
#include <vector>

#include "common.cuh"
#include "keyframe_culling_math.cuh"

using namespace ccm;

namespace {

constexpr int CTA = 256;

struct In {                     // device addresses of the uploaded block
  const uint8_t* kf_bad;
  const int32_t* cand_kf;
  const int64_t* slot_ptr;
  const int32_t* slot_mp;
  const int32_t* slot_octave;
  const uint8_t* mp_bad;
  const int32_t* mp_nobs;
  const int64_t* obs_ptr;
  const int32_t* obs_kf;
  const int32_t* obs_octave;
};

__global__ void __launch_bounds__(CTA) k_kc_count(int32_t n_c, int32_t th, In in, int32_t* __restrict__ n_mps, int32_t* __restrict__ n_red) {
  __shared__ int32_t s_mps[CTA / 32], s_red[CTA / 32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int32_t c = blockIdx.x; c < n_c; c += gridDim.x) {
    const int32_t kf = __ldg(in.cand_kf + c);
    const int64_t b = __ldg(in.slot_ptr + c), e = __ldg(in.slot_ptr + c + 1);
    int32_t mps = 0, red = 0;
    for (int64_t j = b + threadIdx.x; j < e; j += CTA) {
      const int32_t p = __ldg(in.slot_mp + j);
      if (p < 0 || __ldg(in.mp_bad + p)) continue;
      mps++;
      red += kc::slot_redundant(kf, __ldg(in.slot_octave + j), __ldg(in.mp_nobs + p), in.obs_kf, in.obs_octave, __ldg(in.obs_ptr + p),
                                __ldg(in.obs_ptr + p + 1), in.kf_bad, th);
    }
    for (int o = 16; o; o >>= 1) {
      mps += __shfl_xor_sync(0xffffffffu, mps, o);
      red += __shfl_xor_sync(0xffffffffu, red, o);
    }
    if (lane == 0) { s_mps[warp] = mps; s_red[warp] = red; }
    __syncthreads();
    if (threadIdx.x == 0) {
      int32_t m = 0, r = 0;
      for (int w = 0; w < CTA / 32; w++) { m += s_mps[w]; r += s_red[w]; }
      n_mps[c] = m; n_red[c] = r;
    }
    __syncthreads();
  }
}

struct Args {
  int32_t n_kf;
  const uint8_t* kf_bad;
  int32_t n_c;
  const int32_t* cand_kf;
  const uint8_t* cand_not_erase;
  const int64_t* slot_ptr;
  const int32_t* slot_mp;
  const int32_t* slot_octave;
  int32_t n_mp;
  const uint8_t* mp_bad;
  const int32_t* mp_nobs;
  const int32_t* mp_ref;
  const int64_t* obs_ptr;
  const int32_t* obs_kf;
  const int32_t* obs_octave;
  int32_t th;
  double red_thres;
  uint8_t* cull;
  int32_t* n_mps;
  int32_t* n_red;
  int64_t n_slots() const { return slot_ptr[n_c]; }
  int64_t n_obs() const { return n_mp ? obs_ptr[n_mp] : 0; }
};

// Everything the reference could not have been handed: rows out of range, a candidate listed twice, null arrays.  Throws before any
// output is written.
void validate(const std::string& f, const Args& a) {
  CCM_REQUIRE(a.n_kf >= 0 && a.n_c >= 0 && a.n_mp >= 0, f + ": negative size");
  CCM_REQUIRE(a.n_kf == 0 || a.kf_bad, f + ": null kf_bad");
  CCM_REQUIRE(a.slot_ptr, f + ": null slot_ptr");
  CCM_REQUIRE(a.n_c == 0 || (a.cand_kf && a.cand_not_erase && a.cull && a.n_mps && a.n_red), f + ": null candidate array");
  CCM_REQUIRE(a.n_mp == 0 || (a.mp_bad && a.mp_nobs && a.mp_ref && a.obs_ptr), f + ": null point array");
  CCM_REQUIRE(a.slot_ptr[0] == 0, f + ": slot_ptr[0] must be 0");
  std::vector<int32_t> seen((size_t)a.n_kf, -1);
  for (int32_t c = 0; c < a.n_c; c++) {
    const int32_t k = a.cand_kf[c];
    CCM_REQUIRE(k >= 0 && k < a.n_kf, f + ": candidate " + std::to_string(c) + ": keyframe row " + std::to_string(k) + " out of range");
    CCM_REQUIRE(seen[k] < 0, f + ": candidate " + std::to_string(c) + ": keyframe row " + std::to_string(k) + " is already candidate " +
                                 std::to_string(seen[k]));
    seen[k] = c;
    CCM_REQUIRE(a.slot_ptr[c + 1] >= a.slot_ptr[c], f + ": candidate " + std::to_string(c) + ": slot_ptr is not monotone");
  }
  CCM_REQUIRE(a.n_slots() == 0 || (a.slot_mp && a.slot_octave), f + ": null slot array");
  for (int32_t c = 0; c < a.n_c; c++)
    for (int64_t j = a.slot_ptr[c]; j < a.slot_ptr[c + 1]; j++)
      CCM_REQUIRE(a.slot_mp[j] >= -1 && a.slot_mp[j] < a.n_mp, f + ": candidate " + std::to_string(c) + ", slot " + std::to_string(j - a.slot_ptr[c]) +
                                                                   ": point row " + std::to_string(a.slot_mp[j]) + " out of range");
  if (a.n_mp == 0) return;
  CCM_REQUIRE(a.obs_ptr[0] == 0, f + ": obs_ptr[0] must be 0");
  for (int32_t i = 0; i < a.n_mp; i++) CCM_REQUIRE(a.obs_ptr[i + 1] >= a.obs_ptr[i], f + ": point " + std::to_string(i) + ": obs_ptr is not monotone");
  CCM_REQUIRE(a.n_obs() == 0 || (a.obs_kf && a.obs_octave), f + ": null observer array");
  for (int32_t i = 0; i < a.n_mp; i++) {
    CCM_REQUIRE(a.mp_ref[i] >= -1 && a.mp_ref[i] < a.n_kf, f + ": point " + std::to_string(i) + ": reference row " + std::to_string(a.mp_ref[i]) +
                                                           " out of range");
    for (int64_t j = a.obs_ptr[i]; j < a.obs_ptr[i + 1]; j++)
      CCM_REQUIRE(a.obs_kf[j] >= 0 && a.obs_kf[j] < a.n_kf, f + ": point " + std::to_string(i) + ": observer row " + std::to_string(a.obs_kf[j]) +
                                                            " out of range");
  }
}

// nMPs / nRedundant of candidate c over the given keyframe and point state
void count(const Args& a, int32_t c, const uint8_t* kf_bad, const uint8_t* mp_bad, const int32_t* mp_nobs, int32_t* mps, int32_t* red) {
  int32_t m = 0, r = 0;
  for (int64_t j = a.slot_ptr[c]; j < a.slot_ptr[c + 1]; j++) {
    const int32_t p = a.slot_mp[j];
    if (p < 0 || mp_bad[p]) continue;
    m++;
    r += kc::slot_redundant(a.cand_kf[c], a.slot_octave[j], mp_nobs[p], a.obs_kf, a.obs_octave, a.obs_ptr[p], a.obs_ptr[p + 1], kf_bad, a.th);
  }
  *mps = m; *red = r;
}

// The serial walk over counts taken at the start of the member (mps / red, overwritten where a candidate is counted again): decides
// each candidate in order, applies each cull that takes effect and recounts a later candidate whose slots hold a touched point.
// Writes cull, n_mps and n_red; returns the number of candidates counted again.
int32_t settle(const Args& a, const int32_t* mps, const int32_t* red) {
  std::vector<uint8_t> kf_bad(a.kf_bad, a.kf_bad + a.n_kf), mp_bad, touched;
  std::vector<int32_t> nobs, ref, stamp;
  bool any = false;
  int32_t settled = 0;
  for (int32_t c = 0; c < a.n_c; c++) {
    int32_t m = mps[c], r = red[c];
    if (any) {
      bool hit = false;
      for (int64_t j = a.slot_ptr[c]; j < a.slot_ptr[c + 1] && !hit; j++) hit = a.slot_mp[j] >= 0 && touched[a.slot_mp[j]];
      if (hit) { count(a, c, kf_bad.data(), mp_bad.data(), nobs.data(), &m, &r); settled++; }
    }
    a.n_mps[c] = m; a.n_red[c] = r;
    a.cull[c] = kc::culled(r, m, a.red_thres);
    const int32_t kf = a.cand_kf[c];
    if (!a.cull[c] || kf_bad[kf] || a.cand_not_erase[c]) continue;   // KeyFrame::SetBadFlag returns at once (KeyFrame.cpp:936-990)
    if (!any) {
      mp_bad.assign(a.mp_bad, a.mp_bad + a.n_mp); nobs.assign(a.mp_nobs, a.mp_nobs + a.n_mp); ref.assign(a.mp_ref, a.mp_ref + a.n_mp);
      touched.assign((size_t)a.n_mp, 0); stamp.assign((size_t)a.n_mp, -1);
      any = true;
    }
    kf_bad[kf] = 1;
    for (int64_t j = a.slot_ptr[c]; j < a.slot_ptr[c + 1]; j++) {
      const int32_t p = a.slot_mp[j];
      if (p < 0 || stamp[p] == c) continue;
      stamp[p] = c; touched[p] = 1;
      kc::erase_observation(kf, p, a.obs_ptr, a.obs_kf, kf_bad.data(), mp_bad.data(), nobs.data(), ref.data());
    }
    for (int32_t p = 0; p < a.n_mp; p++)        // points that list the culled row but are not in its slots: it is now a bad observer
      if (!touched[p])
        for (int64_t j = a.obs_ptr[p]; j < a.obs_ptr[p + 1]; j++)
          if (a.obs_kf[j] == kf) { touched[p] = 1; break; }
  }
  return settled;
}

void pack(Packer& pk, const Args& a, In* in) {
  const size_t K = (size_t)a.n_kf, Cn = (size_t)a.n_c, P = (size_t)a.n_mp, S = (size_t)a.n_slots(), E = (size_t)a.n_obs();
  in->kf_bad = pk.put(a.kf_bad, K);
  in->cand_kf = pk.put(a.cand_kf, Cn);
  in->slot_ptr = pk.put(a.slot_ptr, Cn + 1);
  in->slot_mp = pk.put(a.slot_mp, S);
  in->slot_octave = pk.put(a.slot_octave, S);
  in->mp_bad = pk.put(a.mp_bad, P);
  in->mp_nobs = pk.put(a.mp_nobs, P);
  in->obs_ptr = pk.put(a.obs_ptr, P ? P + 1 : 0);
  in->obs_kf = pk.put(a.obs_kf, E);
  in->obs_octave = pk.put(a.obs_octave, E);
}

// per-thread staging (Staging): the member runs once per server keyframe
thread_local Staging t_stage;

}  // namespace

extern "C" int ccm_keyframe_culling_host(int32_t n_kf, const uint8_t* kf_bad, int32_t n_c, const int32_t* cand_kf, const uint8_t* cand_not_erase,
                                         const int64_t* slot_ptr, const int32_t* slot_mp, const int32_t* slot_octave, int32_t n_mp,
                                         const uint8_t* mp_bad, const int32_t* mp_nobs, const int32_t* mp_ref, const int64_t* obs_ptr,
                                         const int32_t* obs_kf, const int32_t* obs_octave, int32_t th_obs, double red_thres, uint8_t* cull,
                                         int32_t* n_mps, int32_t* n_red, int32_t* n_settled) {
  return guarded([&] {
    const Args a{n_kf, kf_bad, n_c, cand_kf, cand_not_erase, slot_ptr, slot_mp, slot_octave, n_mp, mp_bad, mp_nobs, mp_ref, obs_ptr, obs_kf,
                 obs_octave, th_obs, red_thres, cull, n_mps, n_red};
    validate("ccm_keyframe_culling_host", a);
    std::vector<int32_t> mps((size_t)n_c), red((size_t)n_c);
    for (int32_t c = 0; c < n_c; c++) count(a, c, kf_bad, mp_bad, mp_nobs, &mps[c], &red[c]);
    const int32_t s = settle(a, mps.data(), red.data());
    if (n_settled) *n_settled = s;
  });
}

extern "C" int ccm_keyframe_culling(int32_t n_kf, const uint8_t* kf_bad, int32_t n_c, const int32_t* cand_kf, const uint8_t* cand_not_erase,
                                    const int64_t* slot_ptr, const int32_t* slot_mp, const int32_t* slot_octave, int32_t n_mp,
                                    const uint8_t* mp_bad, const int32_t* mp_nobs, const int32_t* mp_ref, const int64_t* obs_ptr,
                                    const int32_t* obs_kf, const int32_t* obs_octave, int32_t th_obs, double red_thres, uint8_t* cull,
                                    int32_t* n_mps, int32_t* n_red, int32_t* n_settled) {
  return guarded([&] {
    const Args a{n_kf, kf_bad, n_c, cand_kf, cand_not_erase, slot_ptr, slot_mp, slot_octave, n_mp, mp_bad, mp_nobs, mp_ref, obs_ptr, obs_kf,
                 obs_octave, th_obs, red_thres, cull, n_mps, n_red};
    validate("ccm_keyframe_culling", a);
    ensure_device();
    if (n_c == 0) {
      if (n_settled) *n_settled = 0;
      return;
    }
    Staging& s = t_stage;
    In in{};
    const size_t down = 2 * (size_t)n_c * sizeof(int32_t);
    s.run([&] {
      s.upload([&](Packer& pk) { pack(pk, a, &in); }, down, down);
      int32_t* d = reinterpret_cast<int32_t*>(s.out.p);
      k_kc_count<<<grid_size(n_c, 1), CTA, 0, s.stream>>>(n_c, th_obs, in, d, d + n_c);
      CCM_LAUNCHED();
      CCM_CUDA(cudaMemcpyAsync(s.h_out, s.out.p, down, cudaMemcpyDeviceToHost, s.stream));
      CCM_CUDA(cudaStreamSynchronize(s.stream));
    });
    const int32_t* h = reinterpret_cast<const int32_t*>(s.h_out);
    const int32_t settled = settle(a, h, h + n_c);
    if (n_settled) *n_settled = settled;
  });
}

// normal_depth.cu — map-point normals and depth limits, behind ccm_normal_depth / ccm_normal_depth_host (include/ccm_b200.h).
//
//   MapPoint::UpdateNormalAndDepth   cslam/src/MapPoint.cpp:779-823
//
// After every write-back of a BA or of the essential graph the reference calls this member once per point: mean viewing direction
// over the observers that are not bad, and the scale-invariance distances from the reference keyframe.  Here: one thread per point,
// the observer loop sequential in mObservations order (the f32 sum depends on it: no tree reduction), keyframe centres gathered from a
// K x 12 B table that stays in L2.  Arithmetic in normal_depth_math.cuh; the host entry point runs the same body.
#include <vector>

#include "common.cuh"
#include "normal_depth_math.cuh"

using namespace ccm;

namespace {

// *bad_index is set when an observer or reference row lies outside [0, n_kf): the point is then left untouched and the call fails
__global__ void __launch_bounds__(256) k_normal_depth(int n, int n_kf, const float* __restrict__ centre, const uint8_t* __restrict__ kf_bad,
                                                      const float* __restrict__ pos, const int64_t* __restrict__ obs_ptr,
                                                      const int32_t* __restrict__ obs_kf, const int32_t* __restrict__ ref,
                                                      const float* __restrict__ scale_ref, const float* __restrict__ scale_last,
                                                      float* __restrict__ normal, float* __restrict__ max_dist, float* __restrict__ min_dist,
                                                      uint8_t* __restrict__ status, int* __restrict__ bad_index) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const int64_t b = obs_ptr[i], e = obs_ptr[i + 1];
    const int32_t r = ref[i];
    bool ok = r < n_kf;
    for (int64_t j = b; j < e && ok; j++) ok = (unsigned)obs_kf[j] < (unsigned)n_kf;
    float nv[3] = {0.f, 0.f, 0.f}, dmax = 0.f, dmin = 0.f;
    uint8_t st = 0;
    if (ok) {
      const float X[3] = {pos[3 * (size_t)i], pos[3 * (size_t)i + 1], pos[3 * (size_t)i + 2]};
      st = nd::update_point(X, obs_kf, b, e, nd::TableCentres{centre}, kf_bad, r, scale_ref[i], scale_last[i], nv, &dmax, &dmin);
    } else {
      atomicExch(bad_index, 1);
    }
    if (!st) { nv[0] = nv[1] = nv[2] = 0.f; dmax = dmin = 0.f; }
    normal[3 * (size_t)i] = nv[0]; normal[3 * (size_t)i + 1] = nv[1]; normal[3 * (size_t)i + 2] = nv[2];
    max_dist[i] = dmax; min_dist[i] = dmin; status[i] = st;
  }
}

void check_shape(const char* fn, int32_t n_kf, const float* kf_centre, const uint8_t* kf_bad, int32_t n_mp, const float* mp_pos,
                 const int64_t* obs_ptr, const int32_t* obs_kf, const int32_t* mp_ref, const float* mp_scale_ref, const float* mp_scale_last,
                 const float* normal, const float* max_dist, const float* min_dist, const uint8_t* status) {
  const std::string f(fn);
  CCM_REQUIRE(n_kf >= 0 && n_mp >= 0, f + ": negative size");
  CCM_REQUIRE(n_kf == 0 || (kf_centre && kf_bad), f + ": null keyframe array");
  CCM_REQUIRE(n_mp == 0 || (mp_pos && obs_ptr && mp_ref && mp_scale_ref && mp_scale_last && normal && max_dist && min_dist && status),
              f + ": null point array");
  if (n_mp == 0) return;
  CCM_REQUIRE(obs_ptr[0] == 0, f + ": obs_ptr[0] must be 0");
  for (int32_t i = 0; i < n_mp; i++) CCM_REQUIRE(obs_ptr[i + 1] >= obs_ptr[i], f + ": obs_ptr is not monotone");
  CCM_REQUIRE(obs_ptr[n_mp] == 0 || obs_kf, f + ": null obs_kf");
}

}  // namespace

extern "C" int ccm_normal_depth_host(int32_t n_kf, const float* kf_centre, const uint8_t* kf_bad, int32_t n_mp, const float* mp_pos,
                                     const int64_t* obs_ptr, const int32_t* obs_kf, const int32_t* mp_ref, const float* mp_scale_ref,
                                     const float* mp_scale_last, float* normal, float* max_dist, float* min_dist, uint8_t* status) {
  return guarded([&] {
    check_shape("ccm_normal_depth_host", n_kf, kf_centre, kf_bad, n_mp, mp_pos, obs_ptr, obs_kf, mp_ref, mp_scale_ref, mp_scale_last, normal,
                max_dist, min_dist, status);
    for (int32_t i = 0; i < n_mp; i++) {
      CCM_REQUIRE(mp_ref[i] < n_kf, "ccm_normal_depth_host: reference row out of range");
      for (int64_t j = obs_ptr[i]; j < obs_ptr[i + 1]; j++)
        CCM_REQUIRE(obs_kf[j] >= 0 && obs_kf[j] < n_kf, "ccm_normal_depth_host: observer row out of range");
    }
    for (int32_t i = 0; i < n_mp; i++) {
      float* nv = normal + 3 * (size_t)i;
      const uint8_t st = nd::update_point(mp_pos + 3 * (size_t)i, obs_kf, obs_ptr[i], obs_ptr[i + 1], nd::TableCentres{kf_centre}, kf_bad, mp_ref[i],
                                          mp_scale_ref[i], mp_scale_last[i], nv, max_dist + i, min_dist + i);
      if (!st) { nv[0] = nv[1] = nv[2] = 0.f; max_dist[i] = min_dist[i] = 0.f; }
      status[i] = st;
    }
  });
}

extern "C" int ccm_normal_depth(int32_t n_kf, const float* kf_centre, const uint8_t* kf_bad, int32_t n_mp, const float* mp_pos,
                                const int64_t* obs_ptr, const int32_t* obs_kf, const int32_t* mp_ref, const float* mp_scale_ref,
                                const float* mp_scale_last, float* normal, float* max_dist, float* min_dist, uint8_t* status) {
  return guarded([&] {
    check_shape("ccm_normal_depth", n_kf, kf_centre, kf_bad, n_mp, mp_pos, obs_ptr, obs_kf, mp_ref, mp_scale_ref, mp_scale_last, normal,
                max_dist, min_dist, status);
    ensure_device();
    if (n_mp == 0) return;
    const int64_t E = obs_ptr[n_mp];
    const CallStream cs;
    const cudaStream_t s = cs.s;
    DevBuf<float> d_centre, d_pos, d_sref, d_slast, d_normal, d_max, d_min;
    DevBuf<uint8_t> d_bad, d_status;
    DevBuf<int64_t> d_ptr;
    DevBuf<int32_t> d_obs, d_ref;
    DevBuf<int> d_flag;
    if (n_kf) { d_centre.upload(kf_centre, (size_t)n_kf * 3, s); d_bad.upload(kf_bad, n_kf, s); }
    else { d_centre.alloc(3); d_bad.alloc(1); }
    if (E) d_obs.upload(obs_kf, (size_t)E, s); else d_obs.alloc(1);
    d_pos.upload(mp_pos, (size_t)n_mp * 3, s); d_ptr.upload(obs_ptr, (size_t)n_mp + 1, s); d_ref.upload(mp_ref, n_mp, s);
    d_sref.upload(mp_scale_ref, n_mp, s); d_slast.upload(mp_scale_last, n_mp, s);
    d_normal.alloc((size_t)n_mp * 3); d_max.alloc(n_mp); d_min.alloc(n_mp); d_status.alloc(n_mp); d_flag.alloc_zero(1, s);
    k_normal_depth<<<grid_size(n_mp, 256), 256, 0, s>>>(n_mp, n_kf, d_centre.p, d_bad.p, d_pos.p, d_ptr.p, d_obs.p, d_ref.p, d_sref.p,
                                                         d_slast.p, d_normal.p, d_max.p, d_min.p, d_status.p, d_flag.p);
    CCM_LAUNCHED();
    int flag = 0;
    d_normal.download(normal, (size_t)n_mp * 3, s);
    d_max.download(max_dist, n_mp, s); d_min.download(min_dist, n_mp, s); d_status.download(status, n_mp, s);
    d_flag.download(&flag, 1, s);
    CCM_CUDA(cudaStreamSynchronize(s));
    CCM_REQUIRE(!flag, "ccm_normal_depth: observer or reference row out of range");
  });
}

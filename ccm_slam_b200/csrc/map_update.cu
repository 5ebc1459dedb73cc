// map_update.cu — the map update that follows a global BA, behind ccm_gba_map_update (include/ccm_b200.h); SURVEY.md §8(f) rank 1.
//
//   Map::RunGBA        S/Map.cpp:1441-1570        MapMerger::RunGBA   S/MapMerger.cpp:637-753
//
// Two passes in the reference, both serial over the pointer graph:
//   keyframes   breadth-first from the map origins through the spanning tree; a keyframe the BA did not hold inherits
//               mTcwGBA = (Tcw_child * Twc_parent) * mTcwGBA_parent; every visited keyframe keeps its old pose as mTcwBefGBA and takes
//               mTcwGBA as its pose;
//   map points  a point the BA held takes mPosGBA; any other point follows its reference keyframe: into that camera as it was
//               before, back out through the corrected pose.
// Here: the keyframe pass is a host walk over the flat parent array (K is thousands, the dependence is along the tree), the point
// pass — one independent f32 transform per point, millions of points on a merged map — is one kernel, a thread per point, 24 B of
// point traffic plus a gather of two 4x4 poses that stay in L2.  Arithmetic in map_update_math.cuh.
#include <vector>

#include "common.cuh"
#include "map_update_math.cuh"

using namespace ccm;

namespace {

// state: 0 skip, 1 take pos_gba, 2 follow reference keyframe `ref` (corrected when that keyframe was visited)
__global__ void __launch_bounds__(256) k_map_update_points(int n, const uint8_t* __restrict__ state, const int* __restrict__ ref,
                                                           const float* __restrict__ pos, const float* __restrict__ pos_gba,
                                                           const uint8_t* __restrict__ kf_visited, const float* __restrict__ kf_before,
                                                           const float* __restrict__ kf_twc, float* __restrict__ out,
                                                           uint8_t* __restrict__ corrected) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    float o[3] = {pos[3 * (size_t)i], pos[3 * (size_t)i + 1], pos[3 * (size_t)i + 2]};
    uint8_t done = 0;
    const uint8_t st = state[i];
    if (st == 1) {
      o[0] = pos_gba[3 * (size_t)i]; o[1] = pos_gba[3 * (size_t)i + 1]; o[2] = pos_gba[3 * (size_t)i + 2];
      done = 1;
    } else if (st == 2) {
      const int k = ref[i];
      if (k >= 0 && kf_visited[k]) {
        float Tb[16], Tw[16];
#pragma unroll
        for (int j = 0; j < 4; j++) {
          reinterpret_cast<float4*>(Tb)[j] = reinterpret_cast<const float4*>(kf_before + 16 * (size_t)k)[j];
          reinterpret_cast<float4*>(Tw)[j] = reinterpret_cast<const float4*>(kf_twc + 16 * (size_t)k)[j];
        }
        const float x[3] = {o[0], o[1], o[2]};
        mu::correct_point(Tb, Tw, x, o);
        done = 1;
      }
    }
    out[3 * (size_t)i] = o[0]; out[3 * (size_t)i + 1] = o[1]; out[3 * (size_t)i + 2] = o[2];
    corrected[i] = done;
  }
}

}  // namespace

extern "C" int ccm_gba_map_update(int32_t n_kf, const int32_t* kf_parent, const uint8_t* kf_optimized, const float* kf_Tcw, float* kf_TcwGBA,
                                  uint8_t* kf_visited, int32_t n_mp, const uint8_t* mp_state, const int32_t* mp_ref, const float* mp_pos,
                                  const float* mp_pos_gba, float* mp_pos_out, uint8_t* mp_corrected) {
  return guarded([&] {
    CCM_REQUIRE(n_kf >= 0 && n_mp >= 0, "ccm_gba_map_update: negative size");
    CCM_REQUIRE(n_kf == 0 || (kf_parent && kf_optimized && kf_Tcw && kf_TcwGBA && kf_visited), "ccm_gba_map_update: null keyframe array");
    CCM_REQUIRE(n_mp == 0 || (mp_state && mp_ref && mp_pos && mp_pos_gba && mp_pos_out && mp_corrected), "ccm_gba_map_update: null point array");
    for (int i = 0; i < n_mp; i++) CCM_REQUIRE(mp_state[i] <= 2 && mp_ref[i] < n_kf, "ccm_gba_map_update: bad point state or reference index");
    ensure_device();
    const char* bad = mu::update_keyframes(n_kf, kf_parent, kf_optimized, kf_Tcw, kf_TcwGBA, kf_visited);   // host: tree order
    CCM_REQUIRE(!bad, std::string("ccm_gba_map_update: ") + (bad ? bad : ""));
    if (n_mp == 0) return;
    std::vector<float> twc((size_t)n_kf * 16, 0.f);
    for (int k = 0; k < n_kf; k++)
      if (kf_visited[k]) mu::pose_inverse(kf_TcwGBA + 16 * (size_t)k, twc.data() + 16 * (size_t)k);   // SetPose(mTcwGBA)
    const CallStream cs;
    const cudaStream_t s = cs.s;
    DevBuf<uint8_t> d_state, d_vis, d_corr; DevBuf<int> d_ref; DevBuf<float> d_pos, d_gba, d_before, d_twc, d_out;
    d_state.upload(mp_state, n_mp, s); d_ref.upload(mp_ref, n_mp, s);
    d_pos.upload(mp_pos, (size_t)n_mp * 3, s); d_gba.upload(mp_pos_gba, (size_t)n_mp * 3, s);
    if (n_kf) { d_vis.upload(kf_visited, n_kf, s); d_before.upload(kf_Tcw, (size_t)n_kf * 16, s); d_twc.upload(twc.data(), twc.size(), s); }
    else { d_vis.alloc(1); d_before.alloc(16); d_twc.alloc(16); }
    d_out.alloc((size_t)n_mp * 3); d_corr.alloc(n_mp);
    k_map_update_points<<<grid_size(n_mp, 256), 256, 0, s>>>(n_mp, d_state.p, d_ref.p, d_pos.p, d_gba.p, d_vis.p, d_before.p, d_twc.p,
                                                              d_out.p, d_corr.p);
    CCM_LAUNCHED();
    d_out.download(mp_pos_out, (size_t)n_mp * 3, s);
    d_corr.download(mp_corrected, n_mp, s);
    CCM_CUDA(cudaStreamSynchronize(s));
  });
}

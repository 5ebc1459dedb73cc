// search_and_fuse.cu — the searches of LoopFinder::SearchAndFuse / MapMerger::SearchAndFuse for every corrected keyframe, behind
// ccm_search_and_fuse / ccm_search_and_fuse_host (include/ccm_b200.h).
//
//   LoopFinder::SearchAndFuse    cslam/src/LoopFinder.cpp:709-734
//   MapMerger::SearchAndFuse     cslam/src/MapMerger.cpp:574-598
//   ORBmatcher::Fuse(kfptr, Scw, vpPoints, th, vpReplacePoint)   cslam/src/ORBmatcher.cpp:995-1122
//
// A pair is (keyframe k, loop point i), ordered keyframe-major.  One launch, k_sf_pairs.  Each warp owns 32 consecutive points of one
// keyframe: every lane runs the prelude of its own pair (fuse_pairs.cuh, th = 4, no chi-square gate), most of which end there; then
// the warp walks the window of each lane that passed, one after another, 32 keypoints at a time (window_best.cuh), and a butterfly
// keeps the first minimum.  Each lane stores its own pair once.  A pair whose PredictScale level hangs on the last bit of logf comes
// back as -2 and is settled on the host before the call returns.
#include <cstring>
#include <string>
#include <vector>

#include "fuse_pairs.cuh"

using namespace ccm;
using namespace ccm::fusepair;

namespace {

constexpr int CTA = 256;
constexpr int FLAGGED_OUT = -2;
constexpr long long MAX_PAIRS = 1ll << 30;   // pairs with each keyframe's points padded to whole warps: the launch's thread count stays an int

__global__ void __launch_bounds__(CTA) k_sf_pairs(const Kf* __restrict__ kfs, Pts pts, int n_pts, int tiles_per_kf, int n_warps,
                                                  int32_t* __restrict__ out) {
  const int w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (w >= n_warps) return;   // warp-uniform
  const int lane = threadIdx.x & 31;
  const int kf = w / tiles_per_kf;
  const int row = (w - kf * tiles_per_kf) * 32 + lane;
  const Kf& k = kfs[kf];
  WinQuery q{};
  float ratio;
  const int r = row < n_pts ? pair_query(k, pts, row, q, &ratio) : fb::REJECT;
  int res = r == fb::FLAGGED ? FLAGGED_OUT : -1;
  unsigned pass = __ballot_sync(0xffffffffu, r == fb::PASS);
  while (pass) {
    const int src = __ffs(pass) - 1;
    pass &= pass - 1;
    WinQuery s;
    s.u = __shfl_sync(0xffffffffu, q.u, src);
    s.v = __shfl_sync(0xffffffffu, q.v, src);
    s.r = __shfl_sync(0xffffffffu, q.r, src);
    s.level = __shfl_sync(0xffffffffu, q.level, src);
    s.c0 = __shfl_sync(0xffffffffu, q.c0, src);
    s.c1 = __shfl_sync(0xffffffffu, q.c1, src);
    s.r0 = __shfl_sync(0xffffffffu, q.r0, src);
    s.r1 = __shfl_sync(0xffffffffu, q.r1, src);
    const size_t srow = (size_t)(row - lane + src);
    unsigned best = 0xffffffffu;
    int best_j = -1;
    window_lane_scan(s, lane, pts.desc[2 * srow], pts.desc[2 * srow + 1], k.cell_ptr, k.cell_feat, k.grid_rows, k.kp_xy, k.octave, k.desc,
                     nullptr, k.cam.nlevels, best, best_j);
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) {
      const unsigned ob = __shfl_xor_sync(0xffffffffu, best, off);
      const int oj = __shfl_xor_sync(0xffffffffu, best_j, off);
      if (ob < best) { best = ob; best_j = oj; }
    }
    if (lane == src) res = best_j >= 0 && window_key_distance(best, best_j) <= fb::TH_LOW ? best_j : -1;
  }
  if (row < n_pts) out[(size_t)kf * n_pts + row] = res;
}

// ---- host side ----------------------------------------------------------------------------------------------------------------

void check_args(const std::string& f, const ccm_fuse_kf* kfs, int32_t n_kf, const ccm_fuse_points* pts, int32_t* best) {
  CCM_REQUIRE(pts, f + ": null argument");
  CCM_REQUIRE(n_kf >= 0, f + ": negative size");
  CCM_REQUIRE(n_kf == 0 || kfs, f + ": null keyframe array");
  for (int k = 0; k < n_kf; k++) check_kf(f, &kfs[k], "keyframe " + std::to_string(k), false);
  check_points(f, pts);
  CCM_REQUIRE((long long)n_kf * pts->n == 0 || best, f + ": null output array");
  CCM_REQUIRE((long long)n_kf * (((long long)pts->n + 31) / 32 * 32) < MAX_PAIRS,
              f + ": more than " + std::to_string(MAX_PAIRS) + " pairs (each keyframe's points padded to a multiple of 32)");
}

std::vector<HostKf> host_kfs(const ccm_fuse_kf* kfs, int32_t n_kf) {
  std::vector<HostKf> v;
  v.reserve((size_t)n_kf);
  for (int k = 0; k < n_kf; k++) v.emplace_back(kfs[k], fb::TH_SCW, false);
  return v;
}

thread_local Staging t_stage;

// the Kf table followed by every array the kernel reads
void pack(Packer& pk, const std::vector<HostKf>& kfs, const ccm_fuse_kf* src, const ccm_fuse_points* pts, Pts* dp) {
  Kf* table = pk.host ? reinterpret_cast<Kf*>(pk.host + pk.at) : nullptr;
  pk.reserve(kfs.size() * sizeof(Kf));
  for (size_t r = 0; r < kfs.size(); r++) {
    const Kf k = put_kf(pk, kfs[r], src[r]);
    if (table) table[r] = k;
  }
  *dp = put_points(pk, pts);
}

}  // namespace

extern "C" int ccm_search_and_fuse_host(const ccm_fuse_kf* kfs, int32_t n_kf, const ccm_fuse_points* pts, int32_t* best, int32_t* n_settled) {
  return guarded([&] {
    check_args("ccm_search_and_fuse_host", kfs, n_kf, pts, best);
    const std::vector<HostKf> hk = host_kfs(kfs, n_kf);
    const HostPts hp(*pts);
    const int n = pts->n;
    std::vector<int32_t> out((size_t)n_kf * n);
    int settled = 0;
    for (int k = 0; k < n_kf; k++)
      for (int i = 0; i < n; i++) out[(size_t)k * n + i] = host_pair(hk[k].k, hp.p, i, &settled);
    if (!out.empty()) memcpy(best, out.data(), out.size() * sizeof(int32_t));
    if (n_settled) *n_settled = settled;
  });
}

extern "C" int ccm_search_and_fuse(const ccm_fuse_kf* kfs, int32_t n_kf, const ccm_fuse_points* pts, int32_t* best, int32_t* n_settled) {
  return guarded([&] {
    check_args("ccm_search_and_fuse", kfs, n_kf, pts, best);
    ensure_device();
    const int n = pts->n;
    const long long n_pairs = (long long)n_kf * n;
    if (n_pairs == 0) {
      if (n_settled) *n_settled = 0;
      return;
    }
    const std::vector<HostKf> hk = host_kfs(kfs, n_kf);
    Staging& s = t_stage;
    Pts dp{};
    const int tiles = (n + 31) / 32;
    const long long n_warps = (long long)n_kf * tiles;
    const size_t out_bytes = (size_t)n_pairs * sizeof(int32_t);
    s.run([&] {
      s.upload([&](Packer& pk) { pack(pk, hk, kfs, pts, &dp); }, out_bytes, out_bytes);
      int32_t* d_out = reinterpret_cast<int32_t*>(s.out.p);
      k_sf_pairs<<<div_up(n_warps * 32, CTA), CTA, 0, s.stream>>>(reinterpret_cast<const Kf*>(s.in.p), dp, n, tiles, (int)n_warps, d_out);
      CCM_LAUNCHED();
      CCM_CUDA(cudaMemcpyAsync(s.h_out, d_out, out_bytes, cudaMemcpyDeviceToHost, s.stream));
      CCM_CUDA(cudaStreamSynchronize(s.stream));
    });
    const int32_t* h_out = reinterpret_cast<const int32_t*>(s.h_out);
    std::vector<int32_t> out(h_out, h_out + n_pairs);
    int settled = 0;
    const HostPts hp(*pts);
    for (long long w = 0; w < n_pairs; w++) {
      if (out[w] != FLAGGED_OUT) continue;
      out[w] = settle(hk[w / n].k, hp.p, (int)(w % n));
      settled++;
    }
    memcpy(best, out.data(), (size_t)n_pairs * sizeof(int32_t));
    if (n_settled) *n_settled = settled;
  });
}

// fuse_neighbours.cu — the searches of LocalMapping::SearchInNeighbors for the current keyframe and all its fuse targets, behind
// ccm_fuse_neighbours / ccm_fuse_neighbours_host (include/ccm_b200.h).
//
//   LocalMapping::SearchInNeighbors   cslam/src/Mapping.cpp:471-547
//   ORBmatcher::Fuse(kfptr, vpMapPoints, th)   cslam/src/ORBmatcher.cpp:854-993
//
// A pair is (target t, slot i of the current keyframe) for the forward phase and (current keyframe, candidate c) for the backward one.
// One launch, k_fuse_pairs, one warp per pair: every lane runs the prelude (fuse_neighbours_math.cuh; the same values in every lane),
// then the lanes walk the window 32 keypoints at a time (window_best.cuh, the walk k_window_best uses) and a butterfly keeps the
// first minimum.  A pair whose PredictScale level hangs on the last bit of logf comes back as -2 and is settled on the host before
// the call returns.  The grids are the host's CSR over cells (CellIndex), uploaded with everything else in one pinned block.
#include <cstring>
#include <string>
#include <vector>

#include "fuse_pairs.cuh"

using namespace ccm;
using namespace ccm::fusepair;

namespace {

constexpr int CTA = 256;
constexpr int FLAGGED_OUT = -2;
constexpr long long MAX_PAIRS = 1ll << 26;   // warps of the launch: 32 * pairs must stay an int

__global__ void __launch_bounds__(CTA) k_fuse_pairs(const Kf* __restrict__ kfs, Pts pts, const int32_t* __restrict__ cur_point,
                                                    const int32_t* __restrict__ cand, int n_cur, int n_targets, int n_pairs,
                                                    int32_t* __restrict__ out) {
  const int w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (w >= n_pairs) return;   // warp-uniform
  const int lane = threadIdx.x & 31;
  const int n_fwd = n_cur * n_targets;
  const bool fwd = w < n_fwd;
  const Kf& k = kfs[fwd ? 1 + w / n_cur : 0];
  const int row = fwd ? cur_point[w % n_cur] : cand[w - n_fwd];
  WinQuery q;
  float ratio;
  const int r = pair_query(k, pts, row, q, &ratio);
  unsigned best = 0xffffffffu;
  int best_j = -1;
  if (r == fb::PASS)
    window_lane_scan(q, lane, pts.desc[2 * (size_t)row], pts.desc[2 * (size_t)row + 1], k.cell_ptr, k.cell_feat, k.grid_rows, k.kp_xy,
                     k.octave, k.desc, k.inv_sigma2, k.cam.nlevels, best, best_j);
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) {
    const unsigned ob = __shfl_xor_sync(0xffffffffu, best, off);
    const int oj = __shfl_xor_sync(0xffffffffu, best_j, off);
    if (ob < best) { best = ob; best_j = oj; }
  }
  if (lane == 0)
    out[w] = r == fb::FLAGGED ? FLAGGED_OUT : (best_j >= 0 && window_key_distance(best, best_j) <= fb::TH_LOW ? best_j : -1);
}

// ---- host side ----------------------------------------------------------------------------------------------------------------

// every pair on the host; returns the number settled with logf
int host_pairs(const std::vector<HostKf>& kfs, const Pts& p, const int32_t* cur_point, const int32_t* cand, int n_cur, int n_targets,
               int n_cand, int32_t* out) {
  int settled = 0;
  const long long n_fwd = (long long)n_cur * n_targets;
  for (long long w = 0; w < n_fwd + n_cand; w++) {
    const bool fwd = w < n_fwd;
    const Kf& k = kfs[fwd ? 1 + w / n_cur : 0].k;
    out[w] = host_pair(k, p, fwd ? cur_point[w % n_cur] : cand[w - n_fwd], &settled);
  }
  return settled;
}

// ---- validation -----------------------------------------------------------------------------------------------------------------

void check_args(const std::string& f, const ccm_fuse_kf* cur, const ccm_fuse_kf* targets, int32_t n_targets, const ccm_fuse_points* pts,
                const int32_t* cur_point, const int32_t* cand, int32_t n_cand, int32_t* fwd_best, int32_t* bwd_best) {
  CCM_REQUIRE(cur && pts, f + ": null argument");
  CCM_REQUIRE(n_targets >= 0 && n_cand >= 0 && pts->n >= 0, f + ": negative size");
  CCM_REQUIRE(n_targets == 0 || targets, f + ": null target array");
  check_kf(f, cur, "current keyframe", true);
  for (int t = 0; t < n_targets; t++) check_kf(f, &targets[t], "target " + std::to_string(t), true);
  const int n = cur->grid.n;
  CCM_REQUIRE(n == 0 || cur_point, f + ": null cur_point");
  CCM_REQUIRE(n_cand == 0 || cand, f + ": null cand");
  CCM_REQUIRE(((long long)n * n_targets == 0 || fwd_best) && (n_cand == 0 || bwd_best), f + ": null output array");
  CCM_REQUIRE((long long)n * n_targets + n_cand < MAX_PAIRS, f + ": more than " + std::to_string(MAX_PAIRS) + " pairs");
  check_points(f, pts);
  for (int i = 0; i < n; i++)
    CCM_REQUIRE(cur_point[i] >= -1 && cur_point[i] < pts->n,
                f + ": slot " + std::to_string(i) + " of the current keyframe: point row " + std::to_string(cur_point[i]) + " out of range");
  for (int c = 0; c < n_cand; c++)
    CCM_REQUIRE(cand[c] >= 0 && cand[c] < pts->n, f + ": candidate " + std::to_string(c) + ": point row " + std::to_string(cand[c]) + " out of range");
}

std::vector<HostKf> host_kfs(const ccm_fuse_kf* cur, const ccm_fuse_kf* targets, int32_t n_targets) {
  std::vector<HostKf> v;
  v.reserve(1 + (size_t)n_targets);
  v.emplace_back(*cur, fb::TH, true);
  for (int t = 0; t < n_targets; t++) v.emplace_back(targets[t], fb::TH, true);
  return v;
}

void scatter(const std::vector<int32_t>& out, long long n_fwd, int32_t* fwd_best, int32_t* bwd_best) {
  if (n_fwd) memcpy(fwd_best, out.data(), n_fwd * sizeof(int32_t));
  if ((long long)out.size() > n_fwd) memcpy(bwd_best, out.data() + n_fwd, (out.size() - n_fwd) * sizeof(int32_t));
}

thread_local Staging t_stage;

// the Kf table (row 0 the current keyframe) followed by every array the kernel reads
void pack(Packer& pk, const std::vector<HostKf>& kfs, const ccm_fuse_kf* cur, const ccm_fuse_kf* targets, const ccm_fuse_points* pts,
          const int32_t* cur_point, const int32_t* cand, int32_t n_cand, Pts* dp, const int32_t** d_cur_point, const int32_t** d_cand) {
  Kf* table = pk.host ? reinterpret_cast<Kf*>(pk.host + pk.at) : nullptr;
  pk.reserve(kfs.size() * sizeof(Kf));
  for (size_t r = 0; r < kfs.size(); r++) {
    const Kf k = put_kf(pk, kfs[r], r == 0 ? *cur : targets[r - 1]);
    if (table) table[r] = k;
  }
  *dp = put_points(pk, pts);
  *d_cur_point = pk.put(cur_point, (size_t)cur->grid.n);
  *d_cand = pk.put(cand, (size_t)n_cand);
}

}  // namespace

extern "C" int ccm_fuse_neighbours_host(const ccm_fuse_kf* cur, const ccm_fuse_kf* targets, int32_t n_targets, const ccm_fuse_points* pts,
                                        const int32_t* cur_point, const int32_t* cand, int32_t n_cand, int32_t* fwd_best, int32_t* bwd_best,
                                        int32_t* n_settled) {
  return guarded([&] {
    check_args("ccm_fuse_neighbours_host", cur, targets, n_targets, pts, cur_point, cand, n_cand, fwd_best, bwd_best);
    const std::vector<HostKf> kfs = host_kfs(cur, targets, n_targets);
    const HostPts hp(*pts);
    const long long n_fwd = (long long)cur->grid.n * n_targets;
    std::vector<int32_t> out(n_fwd + n_cand);
    const int settled = host_pairs(kfs, hp.p, cur_point, cand, cur->grid.n, n_targets, n_cand, out.data());
    scatter(out, n_fwd, fwd_best, bwd_best);
    if (n_settled) *n_settled = settled;
  });
}

extern "C" int ccm_fuse_neighbours(const ccm_fuse_kf* cur, const ccm_fuse_kf* targets, int32_t n_targets, const ccm_fuse_points* pts,
                                   const int32_t* cur_point, const int32_t* cand, int32_t n_cand, int32_t* fwd_best, int32_t* bwd_best,
                                   int32_t* n_settled) {
  return guarded([&] {
    const std::string f = "ccm_fuse_neighbours";
    check_args(f, cur, targets, n_targets, pts, cur_point, cand, n_cand, fwd_best, bwd_best);
    ensure_device();
    const int n = cur->grid.n;
    const long long n_fwd = (long long)n * n_targets, n_pairs = n_fwd + n_cand;
    if (n_settled) *n_settled = 0;
    if (n_pairs == 0) return;
    const std::vector<HostKf> kfs = host_kfs(cur, targets, n_targets);

    Staging& s = t_stage;
    Pts dp{};
    const int32_t *d_cur_point = nullptr, *d_cand = nullptr;
    const size_t out_bytes = (size_t)n_pairs * sizeof(int32_t);
    s.run([&] {
      s.upload([&](Packer& pk) { pack(pk, kfs, cur, targets, pts, cur_point, cand, n_cand, &dp, &d_cur_point, &d_cand); }, out_bytes, out_bytes);
      int32_t* d_out = reinterpret_cast<int32_t*>(s.out.p);
      k_fuse_pairs<<<div_up(n_pairs * 32, CTA), CTA, 0, s.stream>>>(reinterpret_cast<const Kf*>(s.in.p), dp, d_cur_point, d_cand, n,
                                                                     n_targets, (int)n_pairs, d_out);
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
      const bool fwd = w < n_fwd;
      out[w] = settle(kfs[fwd ? 1 + w / n : 0].k, hp.p, fwd ? cur_point[w % n] : cand[w - n_fwd]);
      settled++;
    }
    scatter(out, n_fwd, fwd_best, bwd_best);
    if (n_settled) *n_settled = settled;
  });
}

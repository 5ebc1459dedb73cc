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
#include <cmath>
#include <string>
#include <vector>

#include "common.cuh"
#include "fuse_neighbours_math.cuh"
#include "window_best.cuh"

using namespace ccm;

namespace {

namespace fb = ccm::fusenb;
namespace np = ccm::newpts;

constexpr int CTA = 256;
constexpr int FLAGGED_OUT = -2;
constexpr long long MAX_PAIRS = 1ll << 26;   // warps of the launch: 32 * pairs must stay an int

// one keyframe; the pointers are device addresses for the kernel and host arrays for the host entry point
struct Kf {
  fb::Cam cam;
  const float* scale;
  const float* inv_sigma2;
  const int* cell_ptr;
  const int* cell_feat;
  const float2* kp_xy;
  const int* octave;
  const uint4* desc;
  float grid_w_inv, grid_h_inv;
  int grid_cols, grid_rows;
};

struct Pts {
  const float* pos;
  const float* normal;
  const float* max_d;
  const float* min_d;
  const uint4* desc;
  const uint8_t* skip;
};

// GetFeaturesInArea's cell range of q in keyframe k (window_best.cuh, shared with CellIndex::range)
CCM_NP_HD bool cell_range(const Kf& k, WinQuery& q) {
  return ccm::cell_range(q.u, q.v, q.r, k.cam.min_x, k.cam.min_y, k.grid_w_inv, k.grid_h_inv, k.grid_cols, k.grid_rows, q.c0, q.c1, q.r0, q.r1);
}

// the query of point `row` in keyframe k: PASS with q filled, FLAGGED (q.u, q.v set; *ratio for the host), or REJECT
CCM_NP_HD int pair_query(const Kf& k, const Pts& p, int row, WinQuery& q, float* ratio) {
  q.c0 = 1; q.c1 = 0; q.r0 = 1; q.r1 = 0;
  if (row < 0 || p.skip[row]) return fb::REJECT;
  const float P[3] = {p.pos[3 * row], p.pos[3 * row + 1], p.pos[3 * row + 2]};
  const float N[3] = {p.normal[3 * row], p.normal[3 * row + 1], p.normal[3 * row + 2]};
  const int r = fb::prelude(k.cam, k.scale, P, N, p.max_d[row], p.min_d[row], q.u, q.v, q.r, q.level, *ratio);
  if (r == fb::PASS && !cell_range(k, q)) return fb::REJECT;   // no cell: GetFeaturesInArea returns nothing
  return r;
}

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

// a keyframe's host arrays: the CSR of its grid, and copies of the keypoints and descriptors at the alignment float2 / uint4 need
struct HostKf {
  CellIndex cells;
  std::vector<float2> xy;
  std::vector<uint4> desc;
  Kf k{};
  explicit HostKf(const ccm_fuse_kf& f) : cells(f.grid), xy(f.grid.n), desc(2 * (size_t)f.grid.n) {
    if (f.grid.n) {
      memcpy(xy.data(), f.grid.kp_xy, xy.size() * sizeof(float2));
      memcpy(desc.data(), f.grid.desc, desc.size() * sizeof(uint4));
    }
    fb::Cam& c = k.cam;
    memcpy(c.T, f.Tcw, sizeof c.T); memcpy(c.O, f.Ow, sizeof c.O);
    c.fx = f.fx; c.fy = f.fy; c.cx = f.cx; c.cy = f.cy;
    c.min_x = f.grid.min_x; c.min_y = f.grid.min_y; c.max_x = f.grid.max_x; c.max_y = f.grid.max_y;
    c.log_scale = f.log_scale_factor; c.nlevels = f.nlevels;
    k.scale = f.scale_factors; k.inv_sigma2 = f.inv_level_sigma2;
    k.cell_ptr = cells.ptr.data(); k.cell_feat = cells.feat.data(); k.kp_xy = xy.data(); k.octave = f.grid.octave; k.desc = desc.data();
    k.grid_w_inv = f.grid.grid_w_inv; k.grid_h_inv = f.grid.grid_h_inv; k.grid_cols = f.grid.grid_cols; k.grid_rows = f.grid.grid_rows;
  }
};

struct HostPts {
  std::vector<uint4> desc;
  Pts p{};
  explicit HostPts(const ccm_fuse_points& s) : desc(2 * (size_t)s.n) {
    if (s.n) memcpy(desc.data(), s.desc, desc.size() * sizeof(uint4));
    p.pos = s.pos; p.normal = s.normal; p.max_d = s.max_distance; p.min_d = s.min_distance; p.desc = desc.data(); p.skip = s.skip;
  }
};

// the kernel's 32 lanes one after another, then the minimum key
int host_scan(const Kf& k, const Pts& p, int row, const WinQuery& q) {
  unsigned best = 0xffffffffu;
  int best_j = -1;
  for (int lane = 0; lane < 32; lane++) {
    unsigned b = 0xffffffffu;
    int j = -1;
    window_lane_scan(q, lane, p.desc[2 * (size_t)row], p.desc[2 * (size_t)row + 1], k.cell_ptr, k.cell_feat, k.grid_rows, k.kp_xy, k.octave,
                     k.desc, k.inv_sigma2, k.cam.nlevels, b, j);
    if (b < best) { best = b; best_j = j; }
  }
  return best_j >= 0 && window_key_distance(best, best_j) <= fb::TH_LOW ? best_j : -1;
}

// a flagged pair: PredictScale with the host's logf, then the window search.  Every gate before the logarithm rounds as on the device;
// the host's f64 log may differ from the device's in its last bit, so the host may find no flag here, and the logf level holds anyway.
int settle(const Kf& k, const Pts& p, int row) {
  WinQuery q;
  float ratio;
  if (pair_query(k, p, row, q, &ratio) == fb::REJECT) return -1;
  q.level = fb::settle_level(ratio, k.cam.log_scale, k.cam.nlevels);
  q.r = np::fmul(fb::TH, k.scale[q.level]);
  return cell_range(k, q) ? host_scan(k, p, row, q) : -1;
}

// every pair on the host; returns the number settled with logf
int host_pairs(const std::vector<HostKf>& kfs, const Pts& p, const int32_t* cur_point, const int32_t* cand, int n_cur, int n_targets,
               int n_cand, int32_t* out) {
  int settled = 0;
  const long long n_fwd = (long long)n_cur * n_targets;
  for (long long w = 0; w < n_fwd + n_cand; w++) {
    const bool fwd = w < n_fwd;
    const Kf& k = kfs[fwd ? 1 + w / n_cur : 0].k;
    const int row = fwd ? cur_point[w % n_cur] : cand[w - n_fwd];
    WinQuery q;
    float ratio;
    const int r = pair_query(k, p, row, q, &ratio);
    if (r == fb::FLAGGED) { out[w] = settle(k, p, row); settled++; }
    else out[w] = r == fb::PASS ? host_scan(k, p, row, q) : -1;
  }
  return settled;
}

// ---- validation -----------------------------------------------------------------------------------------------------------------

void check_kf(const std::string& f, const ccm_fuse_kf* k, const std::string& who) {
  const std::string at = f + ": " + who + ": ";
  const ccm_feature_grid& g = k->grid;
  CCM_REQUIRE(g.n >= 0 && g.grid_cols > 0 && g.grid_rows > 0 && (long long)g.grid_cols * g.grid_rows <= (1 << 24), at + "bad grid");
  CCM_REQUIRE(g.n == 0 || (g.desc && g.kp_xy && g.octave), at + "null keypoint array");
  CCM_REQUIRE(window_key_fits(g), at + "too many keypoints for the 20-bit visiting position of the window key");
  CCM_REQUIRE(k->nlevels > 0 && k->scale_factors && k->inv_level_sigma2, at + "null or empty scale pyramid");
}

void check_args(const std::string& f, const ccm_fuse_kf* cur, const ccm_fuse_kf* targets, int32_t n_targets, const ccm_fuse_points* pts,
                const int32_t* cur_point, const int32_t* cand, int32_t n_cand, int32_t* fwd_best, int32_t* bwd_best) {
  CCM_REQUIRE(cur && pts, f + ": null argument");
  CCM_REQUIRE(n_targets >= 0 && n_cand >= 0 && pts->n >= 0, f + ": negative size");
  CCM_REQUIRE(n_targets == 0 || targets, f + ": null target array");
  check_kf(f, cur, "current keyframe");
  for (int t = 0; t < n_targets; t++) check_kf(f, &targets[t], "target " + std::to_string(t));
  const int n = cur->grid.n;
  CCM_REQUIRE(n == 0 || cur_point, f + ": null cur_point");
  CCM_REQUIRE(n_cand == 0 || cand, f + ": null cand");
  CCM_REQUIRE(((long long)n * n_targets == 0 || fwd_best) && (n_cand == 0 || bwd_best), f + ": null output array");
  CCM_REQUIRE((long long)n * n_targets + n_cand < MAX_PAIRS, f + ": more than " + std::to_string(MAX_PAIRS) + " pairs");
  CCM_REQUIRE(pts->n == 0 || (pts->pos && pts->normal && pts->max_distance && pts->min_distance && pts->desc && pts->skip),
              f + ": null point array");
  for (int i = 0; i < n; i++)
    CCM_REQUIRE(cur_point[i] >= -1 && cur_point[i] < pts->n,
                f + ": slot " + std::to_string(i) + " of the current keyframe: point row " + std::to_string(cur_point[i]) + " out of range");
  for (int c = 0; c < n_cand; c++)
    CCM_REQUIRE(cand[c] >= 0 && cand[c] < pts->n, f + ": candidate " + std::to_string(c) + ": point row " + std::to_string(cand[c]) + " out of range");
}

std::vector<HostKf> host_kfs(const ccm_fuse_kf* cur, const ccm_fuse_kf* targets, int32_t n_targets) {
  std::vector<HostKf> v;
  v.reserve(1 + (size_t)n_targets);
  v.emplace_back(*cur);
  for (int t = 0; t < n_targets; t++) v.emplace_back(targets[t]);
  return v;
}

void scatter(const std::vector<int32_t>& out, long long n_fwd, int32_t* fwd_best, int32_t* bwd_best) {
  if (n_fwd) memcpy(fwd_best, out.data(), n_fwd * sizeof(int32_t));
  if ((long long)out.size() > n_fwd) memcpy(bwd_best, out.data() + n_fwd, (out.size() - n_fwd) * sizeof(int32_t));
}

// per-thread staging: one pinned block for the upload and one for the download, device blocks grown on demand
struct Scratch {
  cudaStream_t stream = nullptr;
  int device = -1;
  uint8_t* h_blob = nullptr;
  size_t h_cap = 0;
  int32_t* h_out = nullptr;
  size_t h_out_cap = 0;
  DevBuf<uint8_t> blob;
  DevBuf<int32_t> out;
  ~Scratch() {
    if (h_blob) cudaFreeHost(h_blob);
    if (h_out) cudaFreeHost(h_out);
    if (stream) cudaStreamDestroy(stream);
  }
};
thread_local Scratch t_scr;

// the Kf table (row 0 the current keyframe) followed by every array the kernel reads
size_t pack(Packer& pk, const std::vector<HostKf>& kfs, const ccm_fuse_kf* cur, const ccm_fuse_kf* targets, const ccm_fuse_points* pts,
            const int32_t* cur_point, const int32_t* cand, int32_t n_cand, Pts* dp, const int32_t** d_cur_point, const int32_t** d_cand) {
  Kf* table = pk.host ? reinterpret_cast<Kf*>(pk.host + pk.at) : nullptr;
  pk.reserve(kfs.size() * sizeof(Kf));
  for (size_t r = 0; r < kfs.size(); r++) {
    const ccm_fuse_kf& f = r == 0 ? *cur : targets[r - 1];
    const HostKf& h = kfs[r];
    Kf k = h.k;
    const int n = f.grid.n, nl = f.nlevels;
    k.scale = pk.put(f.scale_factors, (size_t)nl);
    k.inv_sigma2 = pk.put(f.inv_level_sigma2, (size_t)nl);
    k.cell_ptr = pk.put(h.cells.ptr.data(), h.cells.ptr.size());
    k.cell_feat = pk.put(h.cells.feat.data(), h.cells.feat.size());
    k.kp_xy = pk.put(h.xy.data(), (size_t)n);
    k.octave = pk.put(f.grid.octave, (size_t)n);
    k.desc = pk.put(h.desc.data(), 2 * (size_t)n);
    if (table) table[r] = k;
  }
  const size_t P = (size_t)pts->n;
  dp->pos = pk.put(pts->pos, 3 * P);
  dp->normal = pk.put(pts->normal, 3 * P);
  dp->max_d = pk.put(pts->max_distance, P);
  dp->min_d = pk.put(pts->min_distance, P);
  dp->desc = reinterpret_cast<const uint4*>(pk.put(pts->desc, 32 * P));
  dp->skip = pk.put(pts->skip, P);
  *d_cur_point = pk.put(cur_point, (size_t)cur->grid.n);
  *d_cand = pk.put(cand, (size_t)n_cand);
  return pk.at;
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

    Scratch& s = t_scr;
    if (s.device != current_device()) {   // the blocks belong to the device they were allocated on
      if (s.stream) { cudaStreamDestroy(s.stream); s.stream = nullptr; }
      s.blob.release(); s.out.release();
      s.device = current_device();
    }
    if (!s.stream) CCM_CUDA(cudaStreamCreateWithFlags(&s.stream, cudaStreamNonBlocking));
    Pts dp{};
    const int32_t *d_cur_point = nullptr, *d_cand = nullptr;
    Packer measure;
    const size_t bytes = pack(measure, kfs, cur, targets, pts, cur_point, cand, n_cand, &dp, &d_cur_point, &d_cand);
    if (s.h_cap < bytes) {
      if (s.h_blob) cudaFreeHost(s.h_blob);
      s.h_blob = nullptr; s.h_cap = 0;
      CCM_CUDA(cudaMallocHost((void**)&s.h_blob, bytes + bytes / 4));
      s.h_cap = bytes + bytes / 4;
    }
    if (s.h_out_cap < (size_t)n_pairs) {
      if (s.h_out) cudaFreeHost(s.h_out);
      s.h_out = nullptr; s.h_out_cap = 0;
      CCM_CUDA(cudaMallocHost((void**)&s.h_out, (n_pairs + n_pairs / 4) * sizeof(int32_t)));
      s.h_out_cap = n_pairs + n_pairs / 4;
    }
    if (s.blob.n < bytes) s.blob.alloc(bytes + bytes / 4);
    if (s.out.n < (size_t)n_pairs) s.out.alloc(n_pairs + n_pairs / 4);
    Packer pk;
    pk.host = s.h_blob; pk.dev = s.blob.p;
    pack(pk, kfs, cur, targets, pts, cur_point, cand, n_cand, &dp, &d_cur_point, &d_cand);
    try {
      CCM_CUDA(cudaMemcpyAsync(s.blob.p, s.h_blob, bytes, cudaMemcpyHostToDevice, s.stream));
      k_fuse_pairs<<<div_up(n_pairs * 32, CTA), CTA, 0, s.stream>>>(reinterpret_cast<const Kf*>(s.blob.p), dp, d_cur_point, d_cand, n,
                                                                     n_targets, (int)n_pairs, s.out.p);
      CCM_LAUNCHED();
      s.out.download(s.h_out, (size_t)n_pairs, s.stream);
      CCM_CUDA(cudaStreamSynchronize(s.stream));
    } catch (...) {
      cudaStreamSynchronize(s.stream);   // nothing of this call may still read the pinned block
      throw;
    }
    std::vector<int32_t> out(s.h_out, s.h_out + n_pairs);
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

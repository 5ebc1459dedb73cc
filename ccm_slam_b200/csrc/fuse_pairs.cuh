// fuse_pairs.cuh — one (keyframe, map point) pair of ORBmatcher::Fuse, as the two batched fusion calls search it: neighbour fusion
// (fuse_neighbours.cu: Fuse(kf, points), th = 3, the chi-square gate on) and loop / merge fusion (search_and_fuse.cu: Fuse(kf, Scw, ...),
// th = 4, no chi-square gate).  The keyframe record carries the two differences, so the prelude, the lane walk, the host's 32-lane
// replay and the logf settlement are one copy for both.
#pragma once
#include <cmath>
#include <cstring>
#include <string>
#include <vector>

#include "common.cuh"
#include "fuse_neighbours_math.cuh"
#include "window_best.cuh"

namespace ccm {
namespace fusepair {

namespace fb = ccm::fusenb;
namespace np = ccm::newpts;

// one keyframe; the pointers are device addresses for the kernels and host arrays for the host entry points
struct Kf {
  fb::Cam cam;
  float th;                 // Fuse's radius factor
  const float* scale;
  const float* inv_sigma2;  // mvInvLevelSigma2 for Fuse(kf, points)'s chi-square gate; null for Fuse(Scw), which has none
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
  const int r = fb::prelude(k.cam, k.scale, k.th, P, N, p.max_d[row], p.min_d[row], q.u, q.v, q.r, q.level, *ratio);
  if (r == fb::PASS && !cell_range(k, q)) return fb::REJECT;   // no cell: GetFeaturesInArea returns nothing
  return r;
}

// a keyframe's host arrays: the CSR of its grid, and copies of the keypoints and descriptors at the alignment float2 / uint4 need
struct HostKf {
  CellIndex cells;
  std::vector<float2> xy;
  std::vector<uint4> desc;
  Kf k{};
  HostKf(const ccm_fuse_kf& f, float th, bool chi2) : cells(f.grid), xy(f.grid.n), desc(2 * (size_t)f.grid.n) {
    if (f.grid.n) {
      memcpy(xy.data(), f.grid.kp_xy, xy.size() * sizeof(float2));
      memcpy(desc.data(), f.grid.desc, desc.size() * sizeof(uint4));
    }
    fb::Cam& c = k.cam;
    memcpy(c.T, f.Tcw, sizeof c.T); memcpy(c.O, f.Ow, sizeof c.O);
    c.fx = f.fx; c.fy = f.fy; c.cx = f.cx; c.cy = f.cy;
    c.min_x = f.grid.min_x; c.min_y = f.grid.min_y; c.max_x = f.grid.max_x; c.max_y = f.grid.max_y;
    c.log_scale = f.log_scale_factor; c.nlevels = f.nlevels;
    k.th = th;
    k.scale = f.scale_factors; k.inv_sigma2 = chi2 ? f.inv_level_sigma2 : nullptr;
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

// the kernels' 32 lanes one after another, then the minimum key
inline int host_scan(const Kf& k, const Pts& p, int row, const WinQuery& q) {
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
inline int settle(const Kf& k, const Pts& p, int row) {
  WinQuery q;
  float ratio;
  if (pair_query(k, p, row, q, &ratio) == fb::REJECT) return -1;
  q.level = fb::settle_level(ratio, k.cam.log_scale, k.cam.nlevels);
  q.r = np::fmul(k.th, k.scale[q.level]);
  return cell_range(k, q) ? host_scan(k, p, row, q) : -1;
}

// one pair on the host; *settled is raised when its level was settled with logf
inline int host_pair(const Kf& k, const Pts& p, int row, int* settled) {
  WinQuery q;
  float ratio;
  const int r = pair_query(k, p, row, q, &ratio);
  if (r == fb::FLAGGED) { ++*settled; return settle(k, p, row); }
  return r == fb::PASS ? host_scan(k, p, row, q) : -1;
}

inline void check_kf(const std::string& f, const ccm_fuse_kf* k, const std::string& who, bool chi2) {
  const std::string at = f + ": " + who + ": ";
  const ccm_feature_grid& g = k->grid;
  CCM_REQUIRE(g.n >= 0 && g.grid_cols > 0 && g.grid_rows > 0 && (long long)g.grid_cols * g.grid_rows <= (1 << 24), at + "bad grid");
  CCM_REQUIRE(g.n == 0 || (g.desc && g.kp_xy && g.octave), at + "null keypoint array");
  CCM_REQUIRE(window_key_fits(g), at + "too many keypoints for the 20-bit visiting position of the window key");
  CCM_REQUIRE(k->nlevels > 0 && k->scale_factors && (!chi2 || k->inv_level_sigma2), at + "null or empty scale pyramid");
}

inline void check_points(const std::string& f, const ccm_fuse_points* pts) {
  CCM_REQUIRE(pts->n >= 0, f + ": negative size");
  CCM_REQUIRE(pts->n == 0 || (pts->pos && pts->normal && pts->max_distance && pts->min_distance && pts->desc && pts->skip),
              f + ": null point array");
}

// a keyframe's arrays into the upload block; returns its record with device addresses
inline Kf put_kf(Packer& pk, const HostKf& h, const ccm_fuse_kf& f) {
  Kf k = h.k;
  const int n = f.grid.n, nl = f.nlevels;
  k.scale = pk.put(f.scale_factors, (size_t)nl);
  k.inv_sigma2 = h.k.inv_sigma2 ? pk.put(f.inv_level_sigma2, (size_t)nl) : nullptr;
  k.cell_ptr = pk.put(h.cells.ptr.data(), h.cells.ptr.size());
  k.cell_feat = pk.put(h.cells.feat.data(), h.cells.feat.size());
  k.kp_xy = pk.put(h.xy.data(), (size_t)n);
  k.octave = pk.put(f.grid.octave, (size_t)n);
  k.desc = pk.put(h.desc.data(), 2 * (size_t)n);
  return k;
}

// the point table into the upload block
inline Pts put_points(Packer& pk, const ccm_fuse_points* pts) {
  const size_t P = (size_t)pts->n;
  Pts dp{};
  dp.pos = pk.put(pts->pos, 3 * P);
  dp.normal = pk.put(pts->normal, 3 * P);
  dp.max_d = pk.put(pts->max_distance, P);
  dp.min_d = pk.put(pts->min_distance, P);
  dp.desc = reinterpret_cast<const uint4*>(pk.put(pts->desc, 32 * P));
  dp.skip = pk.put(pts->skip, P);
  return dp;
}

}  // namespace fusepair
}  // namespace ccm

// window_best.cuh — the pieces of the on-device window search (CCM_MATCH_WINDOW=1, proj_match.cu: k_window_best) that are plain
// arithmetic: the lookup grid as a CSR over cells, the cell range of one query, one lane's walk over that range, and the host
// post-processing of the per-query winners.  Kept apart from the launch code so that a host build (tests/: the kernel's lanes
// run one after another by g++) can check the visiting-position key against the matrix-based host selection without a device.
//
//   Frame/KeyFrame::GetFeaturesInArea   S/Frame.cpp:200-253, S/KeyFrame.cpp:1162-1201 (grid: Frame.cpp:103-119, 255-265)
//   ORBmatcher::Fuse x2                 S/ORBmatcher.cpp:854-993, 995-1122   (first minimum over levels [L-1, L], TH_LOW)
//   ORBmatcher::SearchBySim3            S/ORBmatcher.cpp:1124-1348           (first minimum both ways, TH_HIGH, mutual agreement)
#pragma once
#include <stdint.h>
#include <math.h>

#include <algorithm>
#include <vector>

#include <vector_types.h>   // float2, uint4 (plain C structs; no CUDA runtime needed)

#include "../../include/ccm_b200.h"

#if defined(__CUDACC__)
#define CCM_WB_HD __host__ __device__ __forceinline__
#else
#define CCM_WB_HD inline
#endif

namespace ccm {

namespace wb {
CCM_WB_HD unsigned popc(unsigned x) {
#if defined(__CUDA_ARCH__)
  return __popc(x);
#else
  return (unsigned)__builtin_popcount(x);
#endif
}
// single-rounded f32 operations: no contraction into an FMA on the device, plain operators on the host
CCM_WB_HD float sub(float a, float b) {
#if defined(__CUDA_ARCH__)
  return __fsub_rn(a, b);
#else
  return a - b;
#endif
}
CCM_WB_HD float add(float a, float b) {
#if defined(__CUDA_ARCH__)
  return __fadd_rn(a, b);
#else
  return a + b;
#endif
}
CCM_WB_HD float mul(float a, float b) {
#if defined(__CUDA_ARCH__)
  return __fmul_rn(a, b);
#else
  return a * b;
#endif
}
}  // namespace wb

// GetFeaturesInArea's cell range (S/KeyFrame.cpp:1170-1184) with its early returns, each operation rounded once: the host grid
// (CellIndex::range) and the device (fuse_neighbours.cu) use this one copy.  false = no cell.
CCM_WB_HD bool cell_range(float x, float y, float r, float min_x, float min_y, float w_inv, float h_inv, int cols, int rows, int& c0, int& c1,
                          int& r0, int& r1) {
  const float dx = wb::sub(x, min_x), dy = wb::sub(y, min_y);
  const int a = (int)floorf(wb::mul(wb::sub(dx, r), w_inv));
  c0 = a > 0 ? a : 0;
  if (c0 >= cols) return false;
  const int b = (int)ceilf(wb::mul(wb::add(dx, r), w_inv));
  c1 = b < cols - 1 ? b : cols - 1;
  if (c1 < 0) return false;
  const int c = (int)floorf(wb::mul(wb::sub(dy, r), h_inv));
  r0 = c > 0 ? c : 0;
  if (r0 >= rows) return false;
  const int d = (int)ceilf(wb::mul(wb::add(dy, r), h_inv));
  r1 = d < rows - 1 ? d : rows - 1;
  if (r1 < 0) return false;
  return true;
}

// mGrid as cell_ptr / cell_feat; cell id = column * rows + row (mGrid[col][row])
struct CellIndex {
  const ccm_feature_grid& g;
  std::vector<int> ptr, feat;
  explicit CellIndex(const ccm_feature_grid& gg) : g(gg), ptr((size_t)gg.grid_cols * gg.grid_rows + 1, 0), feat() {
    std::vector<int> cell_of(g.n, -1);
    for (int i = 0; i < g.n; i++) {
      // PosInGrid: round() of a float expression, then the bounds test
      const int cx = (int)roundf((g.kp_xy[2 * i] - g.min_x) * g.grid_w_inv);
      const int cy = (int)roundf((g.kp_xy[2 * i + 1] - g.min_y) * g.grid_h_inv);
      if (cx < 0 || cx >= g.grid_cols || cy < 0 || cy >= g.grid_rows) continue;
      cell_of[i] = cx * g.grid_rows + cy;
      ptr[cell_of[i] + 1]++;
    }
    for (size_t c = 1; c < ptr.size(); c++) ptr[c] += ptr[c - 1];
    feat.resize(ptr.back());
    std::vector<int> fill(ptr.begin(), ptr.end() - 1);
    for (int i = 0; i < g.n; i++)
      if (cell_of[i] >= 0) feat[fill[cell_of[i]]++] = i;
  }

  // GetFeaturesInArea's cell range with its early returns; false = no cell
  bool range(float x, float y, float r, int& c0, int& c1, int& r0, int& r1) const {
    return cell_range(x, y, r, g.min_x, g.min_y, g.grid_w_inv, g.grid_h_inv, g.grid_cols, g.grid_rows, c0, c1, r0, r1);
  }

  // visits the keypoints GetFeaturesInArea(x, y, r[, lo, hi]) would return, in its order; levels: lo <= octave <= hi
  template <typename F>
  void visit(float x, float y, float r, int lo, int hi, F&& f) const {
    int c0, c1, r0, r1;
    if (!range(x, y, r, c0, c1, r0, r1)) return;
    for (int c = c0; c <= c1; c++) {
      const int* p = feat.data() + ptr[(size_t)c * g.grid_rows + r0];
      const int* e = feat.data() + ptr[(size_t)c * g.grid_rows + r1 + 1];   // rows r0..r1 of one column are contiguous
      for (; p < e; ++p) {
        const int j = *p;
        const int o = g.octave[j];
        if (o < lo || o > hi) continue;
        const float dx = g.kp_xy[2 * j] - x, dy = g.kp_xy[2 * j + 1] - y;
        if (fabsf(dx) < r && fabsf(dy) < r) f(j);
      }
    }
  }
};

struct WinQuery { float u, v, r; int level, c0, c1, r0, r1; };

// largest visiting position a walk can reach (every column's run padded to a multiple of 32) must fit the key's low 20 bits
inline bool window_key_fits(const ccm_feature_grid& g) { return (long long)g.n + 32ll * g.grid_cols * 2 < (1 << 20); }

// one WinQuery per query; invalid queries and queries whose range is empty get c0 > c1
inline void fill_window_queries(const CellIndex& cells, const ccm_proj_queries& q, std::vector<WinQuery>& out) {
  out.resize(q.m);
  for (int i = 0; i < q.m; i++) {
    WinQuery& Q = out[i];
    Q.u = q.uv[2 * i]; Q.v = q.uv[2 * i + 1]; Q.r = q.radius[i]; Q.level = q.level[i];
    Q.c0 = 1; Q.c1 = 0; Q.r0 = 1; Q.r1 = 0;
    if (!q.valid[i]) continue;
    int c0, c1, r0, r1;
    if (!cells.range(Q.u, Q.v, Q.r, c0, c1, r0, r1)) continue;
    Q.c0 = c0; Q.c1 = c1; Q.r0 = r0; Q.r1 = r1;
  }
}


// One lane's share of one query's window: the cell runs of columns c0..c1 (rows r0..r1) 32 keypoints at a time in visiting
// order; a keypoint that passes the window / level / chi-square tests forms key = distance << 20 | position-in-visit.  The
// minimum key over the 32 lanes is the reference's strict-'<' first minimum.  best / best_j are updated in place.
CCM_WB_HD void window_lane_scan(const WinQuery& q, int lane, const uint4 d0, const uint4 d1, const int* __restrict__ cell_ptr,
                                const int* __restrict__ cell_feat, int grid_rows, const float2* __restrict__ kp_xy,
                                const int* __restrict__ octave, const uint4* __restrict__ kdesc, const float* __restrict__ inv_sigma2,
                                int nlevels, unsigned& best, int& best_j) {
  unsigned ord = 0;
  for (int c = q.c0; c <= q.c1; c++) {
    const int beg = cell_ptr[c * grid_rows + q.r0], end = cell_ptr[c * grid_rows + q.r1 + 1];
    for (int p = beg; p < end; p += 32, ord += 32) {
      const int i = p + lane;
      if (i >= end) continue;
      const int j = cell_feat[i];
      const int o = octave[j];
      const float2 k = kp_xy[j];
      bool ok = o >= q.level - 1 && o <= q.level && fabsf(wb::sub(k.x, q.u)) < q.r && fabsf(wb::sub(k.y, q.v)) < q.r;
      if (ok && inv_sigma2) {  // Fuse(kf, points): e2 * invSigma2[level] > 5.99 rejects (f32 product, compared as double)
        const float ex = wb::sub(q.u, k.x), ey = wb::sub(q.v, k.y);
        const float e2 = wb::add(wb::mul(ex, ex), wb::mul(ey, ey));
        ok = o >= 0 && o < nlevels && !((double)wb::mul(e2, inv_sigma2[o]) > 5.99);
      }
      if (!ok) continue;
      const uint4 b0 = kdesc[(size_t)j * 2], b1 = kdesc[(size_t)j * 2 + 1];
      const unsigned d = wb::popc(d0.x ^ b0.x) + wb::popc(d0.y ^ b0.y) + wb::popc(d0.z ^ b0.z) + wb::popc(d0.w ^ b0.w) +
                         wb::popc(d1.x ^ b1.x) + wb::popc(d1.y ^ b1.y) + wb::popc(d1.z ^ b1.z) + wb::popc(d1.w ^ b1.w);
      const unsigned key = (d << 20) | (ord + (unsigned)lane);
      if (key < best) { best = key; best_j = j; }
    }
  }
}

// what lane 0 stores once the warp has its minimum key
CCM_WB_HD int window_key_distance(unsigned best, int best_j) { return best_j >= 0 ? (int)(best >> 20) : 0x7fffffff; }

// Fuse: a winner counts when its distance is within th (TH_LOW)
inline void fuse_from_windows(int m, const int* bi, const int* bd, int th, int32_t* best_idx, int32_t* nfound) {
  int found = 0;
  for (int i = 0; i < m; i++) {
    const bool hit = bi[i] >= 0 && bd[i] <= th;
    best_idx[i] = hit ? bi[i] : -1;
    found += hit;
  }
  *nfound = found;
}

// SearchBySim3: winners within th (TH_HIGH) in both directions that name each other
inline void by_sim3_from_windows(int m1, const int* i12, const int* d12, const int* i21, const int* d21, int th, int32_t* match12,
                                 int32_t* nfound) {
  int found = 0;
  for (int i1 = 0; i1 < m1; i1++) {
    const int j = (i12[i1] >= 0 && d12[i1] <= th) ? i12[i1] : -1;
    const bool agree = j >= 0 && i21[j] == i1 && d21[j] <= th;
    match12[i1] = agree ? j : -1;
    found += agree;
  }
  *nfound = found;
}

}  // namespace ccm

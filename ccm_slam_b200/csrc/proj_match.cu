// proj_match.cu — projection-guided matchers behind ccm_search_* / ccm_select_* (include/ccm_b200.h), SURVEY.md §8(f) rank 3.
//
//   ORBmatcher::SearchByProjection x4   S/ORBmatcher.cpp:71-148, 308-446, 1350-1476, 1478-1605
//   ORBmatcher::Fuse x2                 S/ORBmatcher.cpp:854-993, 995-1122
//   ORBmatcher::SearchBySim3            S/ORBmatcher.cpp:1124-1348
//   ORBmatcher::SearchForInitialization S/ORBmatcher.cpp:448-563
//   Frame/KeyFrame::GetFeaturesInArea   S/Frame.cpp:200-253, S/KeyFrame.cpp:1162-1201 (grid: Frame.cpp:103-119, 255-265)
//
// Device work: all (query, keypoint) descriptor distances in one k_hamming launch (match.cu) — the DescriptorDistance
// calls of every window at once; a query's row is m*n*2 bytes back over PCIe, small next to the per-window pointer chasing
// it replaces.  Host work: the lookup grid as a CSR over cells (counting sort in feature order == push_back order), the
// window walk in the reference's visiting order and the order-dependent choice.  ccm_select_* run the host half on a
// caller-supplied matrix and need no device.  The default (CCM_MATCH_WINDOW=0 switches it off) keeps the order-independent choices
// (Fuse x2, SearchBySim3) on the device: k_window_best, m indices back instead of an m x n matrix.
#include <climits>
#include <cmath>

#include "common.cuh"
#include "window_best.cuh"   // CellIndex, WinQuery, window_lane_scan and the host post-processing (shared with the host check in tests/)

using namespace ccm;

namespace {

constexpr int TH_HIGH = 100;      // ORBmatcher::TH_HIGH      (S/ORBmatcher.cpp:63)
constexpr int TH_LOW = 50;        // ORBmatcher::TH_LOW       (S/ORBmatcher.cpp:64)
constexpr int HISTO_LENGTH = 30;  // ORBmatcher::HISTO_LENGTH (S/ORBmatcher.cpp:65)

void check_grid(const ccm_feature_grid* g, const char* who) {
  CCM_REQUIRE(g && g->n >= 0 && g->grid_cols > 0 && g->grid_rows > 0 && (long long)g->grid_cols * g->grid_rows <= (1 << 24),
              std::string(who) + ": bad grid");
  CCM_REQUIRE(g->n == 0 || (g->desc && g->kp_xy && g->octave), std::string(who) + ": null grid array");
}

void check_queries(const ccm_proj_queries* q, const char* who) {
  CCM_REQUIRE(q && q->m >= 0, std::string(who) + ": bad queries");
  CCM_REQUIRE(q->m == 0 || (q->valid && q->uv && q->radius && q->level && q->desc), std::string(who) + ": null query array");
}

struct RotHist {
  std::vector<int> bins[HISTO_LENGTH];
  void add(float a_query, float a_feat, int what) {
    float rot = a_query - a_feat;
    if (rot < 0.0) rot += 360.0f;
    int bin = (int)round(rot * (1.0f / HISTO_LENGTH));
    if (bin == HISTO_LENGTH) bin = 0;
    bins[bin].push_back(what);
  }
  template <typename F>
  int prune(F&& drop) {   // ComputeThreeMaxima, S/ORBmatcher.cpp:1607-1648
    int max1 = 0, max2 = 0, max3 = 0, ind1 = -1, ind2 = -1, ind3 = -1;
    for (int i = 0; i < HISTO_LENGTH; i++) {
      const int s = (int)bins[i].size();
      if (s > max1) { max3 = max2; max2 = max1; max1 = s; ind3 = ind2; ind2 = ind1; ind1 = i; }
      else if (s > max2) { max3 = max2; max2 = s; ind3 = ind2; ind2 = i; }
      else if (s > max3) { max3 = s; ind3 = i; }
    }
    if (max2 < 0.1f * (float)max1) { ind2 = -1; ind3 = -1; }
    else if (max3 < 0.1f * (float)max1) { ind3 = -1; }
    int removed = 0;
    for (int i = 0; i < HISTO_LENGTH; i++) {
      if (i == ind1 || i == ind2 || i == ind3) continue;
      for (int v : bins[i]) { drop(v); removed++; }
    }
    return removed;
  }
};

// ---- the selections (host) ------------------------------------------------------------------------------------------

void select_track(const ccm_feature_grid* g, const ccm_proj_queries* q, const uint16_t* D, const uint8_t* query_has_obs,
                  const uint8_t* feat_blocked, float nnratio, int32_t* match_of_feat, int32_t* nmatches) {
  check_grid(g, "ccm_search_by_projection_track"); check_queries(q, "ccm_search_by_projection_track");
  CCM_REQUIRE(match_of_feat && nmatches && (q->m == 0 || query_has_obs) && (g->n == 0 || feat_blocked) && (D || !q->m || !g->n),
              "ccm_search_by_projection_track: null argument");
  const CellIndex cells(*g);
  std::vector<uint8_t> shut(feat_blocked, feat_blocked + g->n);
  std::fill(match_of_feat, match_of_feat + g->n, -1);
  int found = 0;
  for (int i = 0; i < q->m; i++) {
    if (!q->valid[i]) continue;
    const uint16_t* row = D + (size_t)i * g->n;
    const int L = q->level[i];
    int d1 = 256, d2 = 256, l1 = -1, l2 = -1, j1 = -1;
    cells.visit(q->uv[2 * i], q->uv[2 * i + 1], q->radius[i], L - 1, L, [&](int j) {
      if (shut[j]) return;
      const int d = row[j];
      if (d < d1) { d2 = d1; l2 = l1; d1 = d; l1 = g->octave[j]; j1 = j; }
      else if (d < d2) { d2 = d; l2 = g->octave[j]; }
    });
    if (d1 > TH_HIGH) continue;
    if (l1 == l2 && (float)d1 > nnratio * (float)d2) continue;
    match_of_feat[j1] = i;
    shut[j1] = query_has_obs[i] ? 1 : 0;
    found++;
  }
  *nmatches = found;
}

void select_frame(const ccm_feature_grid* g, const ccm_proj_queries* q, const uint16_t* D, const uint8_t* query_has_obs,
                  const uint8_t* feat_blocked, int reloc, int orb_dist, int check_orientation, int32_t* match_of_feat,
                  int32_t* nmatches) {
  check_grid(g, "ccm_search_by_projection_frame"); check_queries(q, "ccm_search_by_projection_frame");
  CCM_REQUIRE(match_of_feat && nmatches && (q->m == 0 || reloc || query_has_obs) && (g->n == 0 || feat_blocked) && (D || !q->m || !g->n),
              "ccm_search_by_projection_frame: null argument");
  CCM_REQUIRE(!check_orientation || ((q->m == 0 || q->angle) && (g->n == 0 || g->angle)), "ccm_search_by_projection_frame: angles missing");
  const CellIndex cells(*g);
  std::vector<uint8_t> shut(feat_blocked, feat_blocked + g->n);
  std::fill(match_of_feat, match_of_feat + g->n, -1);
  const int th = reloc ? orb_dist : TH_HIGH;
  RotHist hist;
  int found = 0;
  for (int i = 0; i < q->m; i++) {
    if (!q->valid[i]) continue;
    const uint16_t* row = D + (size_t)i * g->n;
    const int L = q->level[i];
    int best = 256, bj = -1;
    cells.visit(q->uv[2 * i], q->uv[2 * i + 1], q->radius[i], L - 1, L + 1, [&](int j) {
      if (shut[j]) return;
      if (row[j] < best) { best = row[j]; bj = j; }
    });
    if (bj < 0 || best > th) continue;
    match_of_feat[bj] = i;
    shut[bj] = reloc ? 1 : (query_has_obs[i] ? 1 : 0);
    found++;
    if (check_orientation) hist.add(q->angle[i], g->angle[bj], bj);
  }
  if (check_orientation) found -= hist.prune([&](int j) { match_of_feat[j] = -2; });
  *nmatches = found;
}

// best keypoint of one window at levels [L-1, L]; `shut` (may be null) hides keypoints; w (may be null) = invSigma2 table
// for Fuse's chi-square gate.  Returns the index or -1; *dist receives the distance.
int window_best(const CellIndex& cells, const ccm_proj_queries* q, int i, const uint16_t* row, const uint8_t* shut, const float* w,
                int nlevels, int* dist) {
  const float u = q->uv[2 * i], v = q->uv[2 * i + 1];
  const int L = q->level[i];
  int best = INT_MAX, bj = -1;
  cells.visit(u, v, q->radius[i], L - 1, L, [&](int j) {
    if (shut && shut[j]) return;
    if (w) {
      const int o = cells.g.octave[j];
      if (o < 0 || o >= nlevels) return;
      const float ex = u - cells.g.kp_xy[2 * j], ey = v - cells.g.kp_xy[2 * j + 1];
      const float e2 = ex * ex + ey * ey;
      if (e2 * w[o] > 5.99) return;
    }
    if (row[j] < best) { best = row[j]; bj = j; }
  });
  *dist = best;
  return bj;
}

void select_sim3proj(const ccm_feature_grid* g, const ccm_proj_queries* q, const uint16_t* D, const uint8_t* feat_matched,
                     const int32_t* existing_idx, int32_t* best_idx, int32_t* match_of_feat, int32_t* nmatches) {
  check_grid(g, "ccm_search_by_projection_sim3"); check_queries(q, "ccm_search_by_projection_sim3");
  CCM_REQUIRE(best_idx && match_of_feat && nmatches && (q->m == 0 || existing_idx) && (g->n == 0 || feat_matched) && (D || !q->m || !g->n),
              "ccm_search_by_projection_sim3: null argument");
  const CellIndex cells(*g);
  std::vector<uint8_t> shut(feat_matched, feat_matched + g->n);
  std::fill(match_of_feat, match_of_feat + g->n, -1);
  int found = 0;
  for (int i = 0; i < q->m; i++) {
    best_idx[i] = -1;
    if (!q->valid[i]) continue;
    int d;
    const int j = window_best(cells, q, i, D + (size_t)i * g->n, shut.data(), nullptr, 0, &d);
    if (j < 0 || d > TH_LOW) continue;
    best_idx[i] = j;
    if (existing_idx[i] == -1) {   // not yet observed by this keyframe: a new match; otherwise the caller remaps (:418-432)
      shut[j] = 1;
      match_of_feat[j] = i;
      found++;
    }
  }
  *nmatches = found;
}

void select_fuse(const ccm_feature_grid* g, const ccm_proj_queries* q, const uint16_t* D, const float* w, int nlevels,
                 int32_t* best_idx, int32_t* nfound) {
  check_grid(g, "ccm_fuse_search"); check_queries(q, "ccm_fuse_search");
  CCM_REQUIRE(best_idx && nfound && (D || !q->m || !g->n) && (!w || nlevels > 0), "ccm_fuse_search: null argument");
  const CellIndex cells(*g);
  int found = 0;
  for (int i = 0; i < q->m; i++) {
    best_idx[i] = -1;
    if (!q->valid[i]) continue;
    int d;
    const int j = window_best(cells, q, i, D + (size_t)i * g->n, nullptr, w, nlevels, &d);
    if (j >= 0 && d <= TH_LOW) { best_idx[i] = j; found++; }
  }
  *nfound = found;
}

void one_way(const ccm_feature_grid* g, const ccm_proj_queries* q, const uint16_t* D, std::vector<int>& out) {
  const CellIndex cells(*g);
  out.assign(q->m, -1);
  for (int i = 0; i < q->m; i++) {
    if (!q->valid[i]) continue;
    int d;
    const int j = window_best(cells, q, i, D + (size_t)i * g->n, nullptr, nullptr, 0, &d);
    if (j >= 0 && d <= TH_HIGH) out[i] = j;
  }
}

void select_by_sim3(const ccm_feature_grid* g1, const ccm_feature_grid* g2, const ccm_proj_queries* q12, const ccm_proj_queries* q21,
                    const uint16_t* D12, const uint16_t* D21, int32_t* match12, int32_t* nfound) {
  check_grid(g1, "ccm_search_by_sim3"); check_grid(g2, "ccm_search_by_sim3");
  check_queries(q12, "ccm_search_by_sim3"); check_queries(q21, "ccm_search_by_sim3");
  CCM_REQUIRE(match12 && nfound, "ccm_search_by_sim3: null output");
  CCM_REQUIRE(q12->m == g1->n && q21->m == g2->n, "ccm_search_by_sim3: one query per keypoint of the source keyframe");
  std::vector<int> m1, m2;
  one_way(g2, q12, D12, m1);
  one_way(g1, q21, D21, m2);
  int found = 0;
  for (int i1 = 0; i1 < q12->m; i1++) {
    const int j = m1[i1];
    const bool agree = j >= 0 && m2[j] == i1;
    match12[i1] = agree ? j : -1;
    found += agree;
  }
  *nfound = found;
}

// SearchForInitialization (S/ORBmatcher.cpp:448-563): F1's octave-0 keypoints looked up around their previous match in F2
void select_init(const ccm_feature_grid* g2, const ccm_proj_queries* q, const uint16_t* D, float nnratio, int check_orientation,
                 int32_t* match12, int32_t* nmatches) {
  check_grid(g2, "ccm_search_for_initialization"); check_queries(q, "ccm_search_for_initialization");
  CCM_REQUIRE(match12 && nmatches && (D || !q->m || !g2->n), "ccm_search_for_initialization: null argument");
  CCM_REQUIRE(!check_orientation || ((q->m == 0 || q->angle) && (g2->n == 0 || g2->angle)), "ccm_search_for_initialization: angles missing");
  const CellIndex cells(*g2);
  std::vector<int> holder(g2->n, -1), held_at(g2->n, INT_MAX);   // vnMatches21, vMatchedDistance
  std::fill(match12, match12 + q->m, -1);
  RotHist hist;
  int found = 0;
  for (int i = 0; i < q->m; i++) {
    if (q->level[i] > 0) continue;
    const uint16_t* row = D + (size_t)i * g2->n;
    int d1 = INT_MAX, d2 = INT_MAX, j1 = -1;
    cells.visit(q->uv[2 * i], q->uv[2 * i + 1], q->radius[i], q->level[i], q->level[i], [&](int j) {
      const int d = row[j];
      if (held_at[j] <= d) return;             // an earlier keypoint of F1 sits closer to this one
      if (d < d1) { d2 = d1; d1 = d; j1 = j; }
      else if (d < d2) d2 = d;
    });
    if (d1 > TH_LOW || !((float)d1 < (float)d2 * nnratio)) continue;
    if (holder[j1] >= 0) { match12[holder[j1]] = -1; found--; }
    match12[i] = j1; holder[j1] = i; held_at[j1] = d1;
    found++;
    if (check_orientation) hist.add(q->angle[i], g2->angle[j1], i);
  }
  if (check_orientation)
    hist.prune([&](int i) { if (match12[i] >= 0) { match12[i] = -1; found--; } });   // an entry may have lost its match already
  *nmatches = found;
}

// ---- device-side window search for the order-independent matchers (default; CCM_MATCH_WINDOW=0: full matrix + host selection) -------------
// Fuse x2 and both directions of SearchBySim3 choose, per query, the first minimum over the window at levels [L-1, L]: no query
// depends on another, so the whole choice can stay on the device and only m indices come back instead of an m x n matrix.
// One warp per query walks the cell runs (columns c0..c1, rows r0..r1 — computed on the host with the reference's float
// expressions), 32 keypoints at a time in visiting order; a lane that passes the window / level / chi-square tests forms
// key = distance << 20 | position-in-visit, the warp keeps the minimum key = the reference's strict-'<' first minimum.
__global__ void __launch_bounds__(256) k_window_best(const WinQuery* __restrict__ Q, const uint4* __restrict__ qdesc, int m,
                                                     const int* __restrict__ cell_ptr, const int* __restrict__ cell_feat, int grid_rows,
                                                     const float2* __restrict__ kp_xy, const int* __restrict__ octave,
                                                     const uint4* __restrict__ kdesc, const float* __restrict__ inv_sigma2, int nlevels,
                                                     int* __restrict__ best_idx, int* __restrict__ best_dist) {
  const int w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (w >= m) return;  // warp-uniform
  const int lane = threadIdx.x & 31;
  const WinQuery q = Q[w];
  unsigned best = 0xffffffffu;
  int best_j = -1;
  if (q.c0 <= q.c1 && q.r0 <= q.r1)
    window_lane_scan(q, lane, qdesc[(size_t)w * 2], qdesc[(size_t)w * 2 + 1], cell_ptr, cell_feat, grid_rows, kp_xy, octave, kdesc, inv_sigma2,
                     nlevels, best, best_j);   // window_best.cuh
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) {
    const unsigned ob = __shfl_xor_sync(0xffffffffu, best, off);
    const int oj = __shfl_xor_sync(0xffffffffu, best_j, off);
    if (ob < best) { best = ob; best_j = oj; }
  }
  if (lane == 0) {
    best_idx[w] = best_j;
    best_dist[w] = window_key_distance(best, best_j);
  }
}

bool window_on_device() {
  static const bool on = [] { const char* v = getenv("CCM_MATCH_WINDOW"); return !v || atoi(v) != 0; }();  // default on; CCM_MATCH_WINDOW=0: full matrix + host selection
  return on;
}

// best keypoint of every valid query's window on the device: out_idx[i] = index or -1, out_dist[i] = its distance
void device_window_best(const ccm_feature_grid* g, const ccm_proj_queries* q, const float* w, int nlevels, std::vector<int>& out_idx,
                        std::vector<int>& out_dist, const char* who) {
  check_grid(g, who); check_queries(q, who);
  out_idx.assign(q->m, -1); out_dist.assign(q->m, INT_MAX);
  if (q->m == 0 || g->n == 0) return;
  CCM_REQUIRE(window_key_fits(*g), std::string(who) + ": too many keypoints for the 20-bit visiting position");
  ensure_device();
  const CellIndex cells(*g);
  std::vector<WinQuery> hq;
  fill_window_queries(cells, *q, hq);
  const CallStream cs;
  const cudaStream_t s = cs.s;
  DevBuf<WinQuery> dQ; DevBuf<uint4> dqd, dkd; DevBuf<int> dptr, dfeat, doct, dbi, dbd; DevBuf<float2> dxy; DevBuf<float> dw;
  dQ.upload(hq.data(), hq.size(), s);
  dqd.upload(reinterpret_cast<const uint4*>(q->desc), (size_t)q->m * 2, s);
  dkd.upload(reinterpret_cast<const uint4*>(g->desc), (size_t)g->n * 2, s);
  dptr.upload(cells.ptr.data(), cells.ptr.size(), s);
  if (!cells.feat.empty()) dfeat.upload(cells.feat.data(), cells.feat.size(), s); else dfeat.alloc(1);
  doct.upload(g->octave, g->n, s);
  dxy.upload(reinterpret_cast<const float2*>(g->kp_xy), g->n, s);
  if (w) dw.upload(w, nlevels, s);
  dbi.alloc(q->m); dbd.alloc(q->m);
  k_window_best<<<div_up((long long)q->m * 32, 256), 256, 0, s>>>(dQ.p, dqd.p, q->m, dptr.p, dfeat.p, g->grid_rows, dxy.p, doct.p, dkd.p,
                                                                 w ? dw.p : nullptr, nlevels, dbi.p, dbd.p);
  CCM_LAUNCHED();
  dbi.download(out_idx.data(), q->m, s);
  dbd.download(out_dist.data(), q->m, s);
  CCM_CUDA(cudaStreamSynchronize(s));
}

const uint16_t* device_distances(const ccm_proj_queries* q, const ccm_feature_grid* g, const char* who) {
  check_grid(g, who); check_queries(q, who);
  return hamming_matrix_host(q->desc, q->m, g->desc, g->n);
}

}  // namespace

extern "C" {

int ccm_features_in_area(const ccm_feature_grid* g, float x, float y, float r, int32_t min_level, int32_t max_level, int32_t* out,
                         int32_t cap, int32_t* n) {
  return guarded([&] {
    check_grid(g, "ccm_features_in_area");
    CCM_REQUIRE(n && (cap == 0 || out), "ccm_features_in_area: null output");
    // Frame's overload checks levels when (minLevel>0)||(maxLevel>=0), and the upper bound only when maxLevel>=0
    const bool check = min_level > 0 || max_level >= 0;
    const int lo = check ? min_level : INT_MIN, hi = (check && max_level >= 0) ? max_level : INT_MAX;
    const CellIndex cells(*g);
    int k = 0;
    cells.visit(x, y, r, lo, hi, [&](int j) { if (k < cap) out[k] = j; k++; });
    *n = k;
  });
}

int ccm_select_by_projection_track(const ccm_feature_grid* g, const ccm_proj_queries* q, const uint16_t* D, const uint8_t* query_has_obs,
                                   const uint8_t* feat_blocked, float nnratio, int32_t* match_of_feat, int32_t* nmatches) {
  return guarded([&] { select_track(g, q, D, query_has_obs, feat_blocked, nnratio, match_of_feat, nmatches); });
}
int ccm_search_by_projection_track(const ccm_feature_grid* g, const ccm_proj_queries* q, const uint8_t* query_has_obs,
                                   const uint8_t* feat_blocked, float nnratio, int32_t* match_of_feat, int32_t* nmatches) {
  return guarded([&] {
    select_track(g, q, device_distances(q, g, "ccm_search_by_projection_track"), query_has_obs, feat_blocked, nnratio, match_of_feat, nmatches);
  });
}

int ccm_select_by_projection_frame(const ccm_feature_grid* g, const ccm_proj_queries* q, const uint16_t* D, const uint8_t* query_has_obs,
                                   const uint8_t* feat_blocked, int32_t reloc, int32_t orb_dist, int32_t check_orientation,
                                   int32_t* match_of_feat, int32_t* nmatches) {
  return guarded([&] { select_frame(g, q, D, query_has_obs, feat_blocked, reloc, orb_dist, check_orientation, match_of_feat, nmatches); });
}
int ccm_search_by_projection_frame(const ccm_feature_grid* g, const ccm_proj_queries* q, const uint8_t* query_has_obs,
                                   const uint8_t* feat_blocked, int32_t reloc, int32_t orb_dist, int32_t check_orientation,
                                   int32_t* match_of_feat, int32_t* nmatches) {
  return guarded([&] {
    select_frame(g, q, device_distances(q, g, "ccm_search_by_projection_frame"), query_has_obs, feat_blocked, reloc, orb_dist,
                 check_orientation, match_of_feat, nmatches);
  });
}

int ccm_select_by_projection_sim3(const ccm_feature_grid* g, const ccm_proj_queries* q, const uint16_t* D, const uint8_t* feat_matched,
                                  const int32_t* existing_idx, int32_t* best_idx, int32_t* match_of_feat, int32_t* nmatches) {
  return guarded([&] { select_sim3proj(g, q, D, feat_matched, existing_idx, best_idx, match_of_feat, nmatches); });
}
int ccm_search_by_projection_sim3(const ccm_feature_grid* g, const ccm_proj_queries* q, const uint8_t* feat_matched,
                                  const int32_t* existing_idx, int32_t* best_idx, int32_t* match_of_feat, int32_t* nmatches) {
  return guarded([&] {
    select_sim3proj(g, q, device_distances(q, g, "ccm_search_by_projection_sim3"), feat_matched, existing_idx, best_idx, match_of_feat, nmatches);
  });
}

int ccm_fuse_select(const ccm_feature_grid* g, const ccm_proj_queries* q, const uint16_t* D, const float* inv_level_sigma2, int32_t nlevels,
                    int32_t* best_idx, int32_t* nfound) {
  return guarded([&] { select_fuse(g, q, D, inv_level_sigma2, nlevels, best_idx, nfound); });
}
int ccm_fuse_search(const ccm_feature_grid* g, const ccm_proj_queries* q, const float* inv_level_sigma2, int32_t nlevels,
                    int32_t* best_idx, int32_t* nfound) {
  return guarded([&] {
    if (window_on_device()) {
      CCM_REQUIRE(best_idx && nfound && (!inv_level_sigma2 || nlevels > 0), "ccm_fuse_search: null argument");
      std::vector<int> bi, bd;
      device_window_best(g, q, inv_level_sigma2, nlevels, bi, bd, "ccm_fuse_search");
      fuse_from_windows(q->m, bi.data(), bd.data(), TH_LOW, best_idx, nfound);
      return;
    }
    select_fuse(g, q, device_distances(q, g, "ccm_fuse_search"), inv_level_sigma2, nlevels, best_idx, nfound);
  });
}

int ccm_select_for_initialization(const ccm_feature_grid* g2, const ccm_proj_queries* q, const uint16_t* D, float nnratio,
                                  int32_t check_orientation, int32_t* match12, int32_t* nmatches) {
  return guarded([&] { select_init(g2, q, D, nnratio, check_orientation, match12, nmatches); });
}
int ccm_search_for_initialization(const ccm_feature_grid* g2, const ccm_proj_queries* q, float nnratio, int32_t check_orientation,
                                  int32_t* match12, int32_t* nmatches) {
  return guarded([&] {
    select_init(g2, q, device_distances(q, g2, "ccm_search_for_initialization"), nnratio, check_orientation, match12, nmatches);
  });
}

int ccm_select_by_sim3(const ccm_feature_grid* g1, const ccm_feature_grid* g2, const ccm_proj_queries* q12, const ccm_proj_queries* q21,
                       const uint16_t* D12, const uint16_t* D21, int32_t* match12, int32_t* nfound) {
  return guarded([&] { select_by_sim3(g1, g2, q12, q21, D12, D21, match12, nfound); });
}
int ccm_search_by_sim3(const ccm_feature_grid* g1, const ccm_feature_grid* g2, const ccm_proj_queries* q12, const ccm_proj_queries* q21,
                       int32_t* match12, int32_t* nfound) {
  return guarded([&] {
    if (window_on_device()) {
      check_grid(g1, "ccm_search_by_sim3"); check_grid(g2, "ccm_search_by_sim3");
      check_queries(q12, "ccm_search_by_sim3"); check_queries(q21, "ccm_search_by_sim3");
      CCM_REQUIRE(match12 && nfound && q12->m == g1->n && q21->m == g2->n, "ccm_search_by_sim3: one query per keypoint of the source keyframe");
      std::vector<int> i12, d12, i21, d21;
      device_window_best(g2, q12, nullptr, 0, i12, d12, "ccm_search_by_sim3");
      device_window_best(g1, q21, nullptr, 0, i21, d21, "ccm_search_by_sim3");
      by_sim3_from_windows(q12->m, i12.data(), d12.data(), i21.data(), d21.data(), TH_HIGH, match12, nfound);
      return;
    }
    // the scratch matrix is per thread and reused by the next launch: keep a copy of the first direction
    const uint16_t* d = device_distances(q12, g2, "ccm_search_by_sim3");
    const std::vector<uint16_t> D12(d, d + (size_t)q12->m * g2->n);
    const uint16_t* D21 = device_distances(q21, g1, "ccm_search_by_sim3");
    select_by_sim3(g1, g2, q12, q21, D12.data(), D21, match12, nfound);
  });
}

}  // extern "C"

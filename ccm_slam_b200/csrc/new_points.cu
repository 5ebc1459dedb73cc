// new_points.cu — LocalMapping::CreateNewMapPoints for a keyframe and all its neighbours, behind ccm_new_map_points /
// ccm_new_map_points_host (include/ccm_b200.h).
//
//   LocalMapping::CreateNewMapPoints          cslam/src/Mapping.cpp:284-469
//   ORBmatcher::SearchForTriangulation        cslam/src/ORBmatcher.cpp:700-852, as ORBmatcher(0.6,false) runs it
//
// vbMatched2 is read but never written in SearchForTriangulation, and the member's matcher keeps no rotation histogram, so the idx2 chosen
// for one idx1 depends on that idx1 alone: the last minimum of the Hamming distance over the neighbour's features of the shared vocabulary
// node that pass the epipole and epipolar-line gates.  Across neighbours the one coupling is that a feature triangulated with neighbour i
// carries a map point when neighbour i+1 is searched: the lowest neighbour whose pair is accepted claims the feature.
//
// Three launches, whatever the number of neighbours:
//   k_np_candidates    one thread per (neighbour, FeatureVector entry of the current keyframe): walks the neighbour's features of the same
//                      node in FeatureVector order, distances from the 32-byte descriptors on the fly -> best2[nb][idx1]
//   k_np_triangulate   one thread per (neighbour, idx1) with a candidate: new_points_math.cuh -> verdict, point
//   k_np_claim         one CTA: per idx1 the first accepted neighbour, later ones read "claimed"; then count, scan and fill of the
//                      accepted pairs in (neighbour, idx1) order.  Positions come from the scan, so the output is the same every run.
// The work is small (about 2e5 descriptor comparisons and a few thousand 4x4 decompositions a keyframe); the call is bound by the
// latency of one upload, three launches and two small downloads, not by arithmetic.
#include <cmath>
#include <string>
#include <vector>

#include "common.cuh"
#include "new_points_math.cuh"

using namespace ccm;

namespace {

namespace np = ccm::newpts;

static_assert((int)np::NONE == CCM_NEWPTS_NONE && (int)np::ACCEPTED == CCM_NEWPTS_ACCEPTED && (int)np::PARALLAX == CCM_NEWPTS_PARALLAX &&
              (int)np::W_ZERO == CCM_NEWPTS_W_ZERO && (int)np::DEPTH1 == CCM_NEWPTS_DEPTH1 && (int)np::DEPTH2 == CCM_NEWPTS_DEPTH2 &&
              (int)np::REPROJ1 == CCM_NEWPTS_REPROJ1 && (int)np::REPROJ2 == CCM_NEWPTS_REPROJ2 && (int)np::DIST_ZERO == CCM_NEWPTS_DIST_ZERO &&
              (int)np::SCALE == CCM_NEWPTS_SCALE && (int)np::CLAIMED == CCM_NEWPTS_CLAIMED, "verdict codes");

constexpr int CTA = 128;
constexpr int CLAIM_CTA = 1024;
constexpr int MAX_NEIGHBOURS = 65535;   // the neighbour is the y index of the launch grids; the member passes at most 20

// one keyframe; the pointers are device addresses for the kernels and the caller's arrays for the host entry point
struct View {
  const uint8_t* desc;
  const uint8_t* has_mp;
  const float* xy;
  const int32_t* octave;
  const float* sigma2;
  const float* scale;
  const int32_t* node_ptr;
  const uint32_t* feat;
  const int32_t* aux;   // current keyframe: the node of each FeatureVector entry; neighbour: its node for each node of the current keyframe, or -1
  int32_t n, n_entries;
  np::Camera cam;
  float F12[9], ex, ey;   // neighbours only
  float ratio_factor;     // current keyframe only: 1.5f * mfScaleFactor
};

__host__ __device__ __forceinline__ void load_desc(const uint8_t* p, uint32_t d[8]) {
#if defined(__CUDA_ARCH__)
  const uint4 a = reinterpret_cast<const uint4*>(p)[0], b = reinterpret_cast<const uint4*>(p)[1];
  d[0] = a.x; d[1] = a.y; d[2] = a.z; d[3] = a.w; d[4] = b.x; d[5] = b.y; d[6] = b.z; d[7] = b.w;
#else
  memcpy(d, p, 32);
#endif
}

__host__ __device__ __forceinline__ int popc(uint32_t v) {
#if defined(__CUDA_ARCH__)
  return __popc(v);
#else
  return __builtin_popcount(v);
#endif
}

// the inner loop of SearchForTriangulation for feature i of the current keyframe over entries [kb, ke) of the neighbour's FeatureVector
__host__ __device__ __forceinline__ int best_candidate(const View& c, const View& v, int i, int kb, int ke) {
  float l[4];
  np::epipolar_line(c.xy[2 * i], c.xy[2 * i + 1], v.F12, l);
  uint32_t d1[8], d2[8];
  load_desc(c.desc + 32 * (size_t)i, d1);
  int best = np::TH_LOW, best_j = -1;
  for (int k = kb; k < ke; k++) {
    const int j = (int)v.feat[k];
    if (v.has_mp[j]) continue;
    load_desc(v.desc + 32 * (size_t)j, d2);
    int d = 0;
#pragma unroll
    for (int w = 0; w < 8; w++) d += popc(d1[w] ^ d2[w]);
    if (d > np::TH_LOW || d > best) continue;   // ties replace the incumbent
    const int o = v.octave[j];
    if (!np::passes_epipolar(l, v.ex, v.ey, v.xy[2 * j], v.xy[2 * j + 1], v.scale[o], v.sigma2[o])) continue;
    best_j = j; best = d;
  }
  return best_j;
}

__host__ __device__ __forceinline__ uint8_t pair_verdict(const View& c, const View& v, int i, int j, float X[3]) {
  const int o1 = c.octave[i], o2 = v.octave[j];
  return np::triangulate_pair(c.cam, v.cam, c.xy[2 * i], c.xy[2 * i + 1], c.sigma2[o1], c.scale[o1], v.xy[2 * j], v.xy[2 * j + 1],
                              v.sigma2[o2], v.scale[o2], c.ratio_factor, X);
}

// views[0] the current keyframe, views[1 + b] neighbour b; best2 arrives filled with -1
__global__ void __launch_bounds__(CTA) k_np_candidates(const View* __restrict__ views, int32_t* __restrict__ best2) {
  const View& c = views[0];
  const View& v = views[1 + blockIdx.y];
  const int k1 = blockIdx.x * CTA + threadIdx.x;
  if (k1 >= c.n_entries) return;
  const int b = v.aux[c.aux[k1]];
  if (b < 0) return;
  const int i = (int)c.feat[k1];
  if (c.has_mp[i]) return;
  best2[(size_t)blockIdx.y * c.n + i] = best_candidate(c, v, i, v.node_ptr[b], v.node_ptr[b + 1]);
}

__global__ void __launch_bounds__(CTA) k_np_triangulate(const View* __restrict__ views, const int32_t* __restrict__ best2,
                                                        uint8_t* __restrict__ verdict, float* __restrict__ X3) {
  const View& c = views[0];
  const int i = blockIdx.x * CTA + threadIdx.x;
  if (i >= c.n) return;
  const size_t at = (size_t)blockIdx.y * c.n + i;
  const int j = best2[at];
  if (j < 0) return;
  float X[3] = {0.f, 0.f, 0.f};
  verdict[at] = pair_verdict(c, views[1 + blockIdx.y], i, j, X);
  X3[3 * at] = X[0]; X3[3 * at + 1] = X[1]; X3[3 * at + 2] = X[2];
}

__global__ void __launch_bounds__(CLAIM_CTA) k_np_claim(int n, int n_nb, int32_t* __restrict__ best2, uint8_t* __restrict__ verdict,
                                                        const float* __restrict__ X3, ccm_new_point* __restrict__ out,
                                                        int32_t* __restrict__ n_out) {
  __shared__ int wsum[CLAIM_CTA / 32];
  for (int i = threadIdx.x; i < n; i += CLAIM_CTA) {
    bool claimed = false;
    for (int b = 0; b < n_nb; b++) {
      const size_t at = (size_t)b * n + i;
      if (claimed) { verdict[at] = np::CLAIMED; best2[at] = -1; }
      else claimed = verdict[at] == np::ACCEPTED;
    }
  }
  __syncthreads();
  const int total = n * n_nb;   // below 2^30: checked on entry
  const int chunk = (total + CLAIM_CTA - 1) / CLAIM_CTA;
  const int lo = min(total, chunk * (int)threadIdx.x), hi = min(total, lo + chunk);
  int cnt = 0;
  for (int t = lo; t < hi; t++) cnt += verdict[t] == np::ACCEPTED;
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  int inc = cnt;
  for (int d = 1; d < 32; d <<= 1) {
    const int up = __shfl_up_sync(0xffffffffu, inc, d);
    if (lane >= d) inc += up;
  }
  if (lane == 31) wsum[w] = inc;
  __syncthreads();
  int base = 0, all = 0;
  for (int q = 0; q < CLAIM_CTA / 32; q++) { base += q < w ? wsum[q] : 0; all += wsum[q]; }
  int pos = base + inc - cnt;
  for (int t = lo; t < hi; t++)
    if (verdict[t] == np::ACCEPTED) {
      ccm_new_point* p = out + pos++;
      p->nb = t / n; p->idx1 = t % n; p->idx2 = best2[t];
      p->x3D[0] = X3[3 * (size_t)t]; p->x3D[1] = X3[3 * (size_t)t + 1]; p->x3D[2] = X3[3 * (size_t)t + 2];
    }
  if (threadIdx.x == 0) *n_out = all;
}

// ---- validation -----------------------------------------------------------------------------------------------------------------

std::string who(int b) { return b < 0 ? std::string("current keyframe") : "neighbour " + std::to_string(b); }

void check_view(const std::string& f, const ccm_newpts_view* p, int b) {
  const std::string at = f + ": " + who(b) + ": ";
  const ccm_tri_view& v = p->v;
  CCM_REQUIRE(v.n >= 0, at + "negative feature count");
  CCM_REQUIRE(v.n == 0 || (v.desc && v.has_mp && v.kp_xy && v.octave), at + "null feature array");
  CCM_REQUIRE(p->nlevels > 0 && p->level_sigma2 && p->scale_factors, at + "null or empty scale pyramid");
  const ccm_feature_vector* fv = v.fv;
  CCM_REQUIRE(fv && fv->n_nodes >= 0 && (fv->n_nodes == 0 || (fv->node_id && fv->node_ptr && fv->feat)), at + "bad FeatureVector");
  CCM_REQUIRE(fv->n_nodes == 0 || fv->node_ptr[0] == 0, at + "bad FeatureVector: node_ptr[0] must be 0");
  for (int i = 0; i < fv->n_nodes; i++) {
    CCM_REQUIRE(fv->node_ptr[i] <= fv->node_ptr[i + 1], at + "bad FeatureVector: node_ptr is not monotone");
    if (i) CCM_REQUIRE(fv->node_id[i - 1] < fv->node_id[i], at + "bad FeatureVector: node ids are not ascending");
  }
  const int ne = fv->n_nodes ? fv->node_ptr[fv->n_nodes] : 0;
  std::vector<uint8_t> seen(b < 0 ? v.n : 0, 0);
  for (int k = 0; k < ne; k++) {
    CCM_REQUIRE(fv->feat[k] < (uint32_t)v.n, at + "bad FeatureVector: feature " + std::to_string(fv->feat[k]) + " out of range");
    if (b < 0) {
      CCM_REQUIRE(!seen[fv->feat[k]], at + "bad FeatureVector: feature " + std::to_string(fv->feat[k]) + " listed twice");
      seen[fv->feat[k]] = 1;
    }
  }
  for (int i = 0; i < v.n; i++)
    CCM_REQUIRE(v.octave[i] >= 0 && v.octave[i] < p->nlevels, at + "octave of feature " + std::to_string(i) + " out of range");
  for (int k = 0; k < 12; k++) CCM_REQUIRE(std::isfinite(p->Tcw[k]), at + "non-finite Tcw");
  for (int k = 0; k < 3; k++) CCM_REQUIRE(std::isfinite(p->Ow[k]), at + "non-finite Ow");
}

void check_args(const std::string& f, const ccm_newpts_view* cur, const ccm_newpts_neighbour* nb, int32_t n_nb, ccm_new_point* out,
                int32_t capacity, int32_t* n_out) {
  CCM_REQUIRE(cur && n_out, f + ": null argument");
  CCM_REQUIRE(n_nb >= 0 && capacity >= 0, f + ": negative size");
  CCM_REQUIRE(n_nb <= MAX_NEIGHBOURS, f + ": more than " + std::to_string(MAX_NEIGHBOURS) + " neighbours");
  CCM_REQUIRE(n_nb == 0 || nb, f + ": null neighbour array");
  CCM_REQUIRE(capacity == 0 || out, f + ": null output array");
  check_view(f, cur, -1);
  for (int b = 0; b < n_nb; b++) check_view(f, &nb[b].view, b);
  CCM_REQUIRE((long long)cur->v.n * n_nb < (1ll << 30), f + ": too many (neighbour, feature) pairs");
}

int entries_of(const ccm_feature_vector* fv) { return fv->n_nodes ? fv->node_ptr[fv->n_nodes] : 0; }

// the node of the neighbour that carries each node id of the current keyframe, or -1 (the reference's merge-join); returns how many are shared
int shared_nodes(const ccm_feature_vector* f1, const ccm_feature_vector* f2, int32_t* peer) {
  int a = 0, b = 0, n = 0;
  for (int k = 0; k < f1->n_nodes; k++) peer[k] = -1;
  while (a < f1->n_nodes && b < f2->n_nodes) {
    const uint32_t na = f1->node_id[a], nb = f2->node_id[b];
    if (na == nb) { peer[a] = b; n++; a++; b++; }
    else if (na < nb) a++;
    else b++;
  }
  return n;
}

View view_of(const ccm_newpts_view* p) {
  View v{};
  v.desc = p->v.desc; v.has_mp = p->v.has_mp; v.xy = p->v.kp_xy; v.octave = p->v.octave;
  v.sigma2 = p->level_sigma2; v.scale = p->scale_factors;
  v.node_ptr = p->v.fv->node_ptr; v.feat = p->v.fv->feat;
  v.n = p->v.n; v.n_entries = entries_of(p->v.fv);
  v.cam.fx = p->v.fx; v.cam.fy = p->v.fy; v.cam.cx = p->v.cx; v.cam.cy = p->v.cy;
  memcpy(v.cam.T, p->Tcw, sizeof v.cam.T); memcpy(v.cam.O, p->Ow, sizeof v.cam.O);
  v.ratio_factor = 1.5f * p->scale_factor;
  return v;
}

View view_of(const ccm_newpts_neighbour* p) {
  View v = view_of(&p->view);
  memcpy(v.F12, p->F12, sizeof v.F12); v.ex = p->ex; v.ey = p->ey;
  return v;
}

bool any_free(const ccm_newpts_view* cur) {
  for (int i = 0; i < cur->v.n; i++)
    if (!cur->v.has_mp[i]) return true;
  return false;
}

void fill_empty(int64_t cells, int32_t* n_out, int32_t* best2, uint8_t* verdict) {
  *n_out = 0;
  for (int64_t t = 0; t < cells; t++) {
    if (best2) best2[t] = -1;
    if (verdict) verdict[t] = np::NONE;
  }
}

[[noreturn]] void too_small(const std::string& f, int capacity, int needed) {
  throw Error(CCM_ERR_INVALID, f + ": capacity " + std::to_string(capacity) + " below the " + std::to_string(needed) + " points needed");
}

// per-thread staging (Staging): LocalMapping calls once per keyframe
thread_local Staging t_stage;

// the View table (views[0] the current keyframe, then the neighbours) followed by every array the views point to
void pack_views(Packer& pk, const ccm_newpts_view* cur, const ccm_newpts_neighbour* nb, int32_t n_nb, const std::vector<int32_t>& ent_node,
                  const std::vector<int32_t>& peer) {
  const int n_nodes1 = cur->v.fv->n_nodes;
  View* table = pk.host ? reinterpret_cast<View*>(pk.host + pk.at) : nullptr;
  pk.reserve((size_t)(1 + n_nb) * sizeof(View));
  for (int b = -1; b < n_nb; b++) {
    const ccm_newpts_view* p = b < 0 ? cur : &nb[b].view;
    View v = b < 0 ? view_of(cur) : view_of(&nb[b]);
    const ccm_feature_vector* fv = p->v.fv;
    v.desc = pk.put(p->v.desc, (size_t)p->v.n * 32);
    v.has_mp = pk.put(p->v.has_mp, (size_t)p->v.n);
    v.xy = pk.put(p->v.kp_xy, (size_t)p->v.n * 2);
    v.octave = pk.put(p->v.octave, (size_t)p->v.n);
    v.sigma2 = pk.put(p->level_sigma2, (size_t)p->nlevels);
    v.scale = pk.put(p->scale_factors, (size_t)p->nlevels);
    v.node_ptr = pk.put(fv->node_ptr, fv->n_nodes ? (size_t)fv->n_nodes + 1 : 0);
    v.feat = pk.put(fv->feat, (size_t)v.n_entries);
    v.aux = b < 0 ? pk.put(ent_node.data(), ent_node.size()) : pk.put(peer.data() + (size_t)b * n_nodes1, (size_t)n_nodes1);
    if (table) table[b + 1] = v;
  }
}

}  // namespace

extern "C" int ccm_new_map_points_host(const ccm_newpts_view* cur, const ccm_newpts_neighbour* nb, int32_t n_nb, ccm_new_point* out,
                                       int32_t capacity, int32_t* n_out, int32_t* best2, uint8_t* verdict) {
  return guarded([&] {
    const std::string f = "ccm_new_map_points_host";
    check_args(f, cur, nb, n_nb, out, capacity, n_out);
    const int n = cur->v.n;
    const size_t cells = (size_t)n * n_nb;
    std::vector<int32_t> b2(cells, -1);
    std::vector<uint8_t> vd(cells, np::NONE);
    std::vector<float> X3(3 * cells, 0.f);
    const View c = view_of(cur);
    std::vector<int32_t> peer(cur->v.fv->n_nodes);
    for (int b = 0; b < n_nb; b++) {
      const View v = view_of(&nb[b]);
      shared_nodes(cur->v.fv, nb[b].view.v.fv, peer.data());
      for (int a = 0; a < cur->v.fv->n_nodes; a++) {
        if (peer[a] < 0) continue;
        for (int k1 = c.node_ptr[a]; k1 < c.node_ptr[a + 1]; k1++) {
          const int i = (int)c.feat[k1];
          if (c.has_mp[i]) continue;
          b2[(size_t)b * n + i] = best_candidate(c, v, i, v.node_ptr[peer[a]], v.node_ptr[peer[a] + 1]);
        }
      }
      for (int i = 0; i < n; i++) {
        const size_t at = (size_t)b * n + i;
        if (b2[at] >= 0) vd[at] = pair_verdict(c, v, i, b2[at], &X3[3 * at]);
      }
    }
    int count = 0;
    for (int i = 0; i < n; i++) {
      bool claimed = false;
      for (int b = 0; b < n_nb; b++) {
        const size_t at = (size_t)b * n + i;
        if (claimed) { vd[at] = np::CLAIMED; b2[at] = -1; }
        else if (vd[at] == np::ACCEPTED) { claimed = true; count++; }
      }
    }
    *n_out = count;
    if (capacity < count) too_small(f, capacity, count);
    int pos = 0;
    for (size_t t = 0; t < cells; t++)
      if (vd[t] == np::ACCEPTED) {
        ccm_new_point& p = out[pos++];
        p.nb = (int32_t)(t / n); p.idx1 = (int32_t)(t % n); p.idx2 = b2[t];
        memcpy(p.x3D, &X3[3 * t], sizeof p.x3D);
      }
    if (best2 && cells) memcpy(best2, b2.data(), cells * sizeof(int32_t));
    if (verdict && cells) memcpy(verdict, vd.data(), cells);
  });
}

extern "C" int ccm_new_map_points(const ccm_newpts_view* cur, const ccm_newpts_neighbour* nb, int32_t n_nb, ccm_new_point* out,
                                  int32_t capacity, int32_t* n_out, int32_t* best2, uint8_t* verdict) {
  return guarded([&] {
    const std::string f = "ccm_new_map_points";
    check_args(f, cur, nb, n_nb, out, capacity, n_out);
    ensure_device();
    const int n = cur->v.n, n_nodes1 = cur->v.fv->n_nodes, ne1 = entries_of(cur->v.fv);
    const size_t cells = (size_t)n * n_nb;
    std::vector<int32_t> peer((size_t)n_nodes1 * n_nb);
    int shared = 0;
    for (int b = 0; b < n_nb; b++) shared += shared_nodes(cur->v.fv, nb[b].view.v.fv, peer.data() + (size_t)b * n_nodes1);
    if (cells == 0 || ne1 == 0 || shared == 0 || !any_free(cur)) { fill_empty((int64_t)cells, n_out, best2, verdict); return; }

    std::vector<int32_t> ent_node(ne1);
    for (int a = 0; a < n_nodes1; a++)
      for (int k = cur->v.fv->node_ptr[a]; k < cur->v.fv->node_ptr[a + 1]; k++) ent_node[k] = a;
    // the output block holds only what the kernels write; the copies go from it to the caller's arrays
    Packer lay;
    const size_t at_best2 = lay.reserve(cells * sizeof(int32_t)), at_verdict = lay.reserve(cells), at_X3 = lay.reserve(3 * cells * sizeof(float)),
                 at_out = lay.reserve(cells * sizeof(ccm_new_point)), at_count = lay.reserve(sizeof(int32_t));
    Staging& s = t_stage;
    s.run([&] {
      s.upload([&](Packer& pk) { pack_views(pk, cur, nb, n_nb, ent_node, peer); }, lay.at, 0);
      int32_t* d_best2 = reinterpret_cast<int32_t*>(s.out.p + at_best2);
      uint8_t* d_verdict = s.out.p + at_verdict;
      float* d_X3 = reinterpret_cast<float*>(s.out.p + at_X3);
      ccm_new_point* d_out = reinterpret_cast<ccm_new_point*>(s.out.p + at_out);
      int32_t* d_count = reinterpret_cast<int32_t*>(s.out.p + at_count);
      CCM_CUDA(cudaMemsetAsync(d_best2, 0xff, cells * sizeof(int32_t), s.stream));
      CCM_CUDA(cudaMemsetAsync(d_verdict, 0, cells, s.stream));
      const View* d_views = reinterpret_cast<const View*>(s.in.p);
      k_np_candidates<<<dim3(div_up(ne1, CTA), n_nb), CTA, 0, s.stream>>>(d_views, d_best2);
      CCM_LAUNCHED();
      k_np_triangulate<<<dim3(div_up(n, CTA), n_nb), CTA, 0, s.stream>>>(d_views, d_best2, d_verdict, d_X3);
      CCM_LAUNCHED();
      k_np_claim<<<1, CLAIM_CTA, 0, s.stream>>>(n, n_nb, d_best2, d_verdict, d_X3, d_out, d_count);
      CCM_LAUNCHED();
      int32_t count = 0;
      CCM_CUDA(cudaMemcpyAsync(&count, d_count, sizeof(int32_t), cudaMemcpyDeviceToHost, s.stream));
      CCM_CUDA(cudaStreamSynchronize(s.stream));
      *n_out = count;
      if (capacity < count) too_small(f, capacity, count);
      if (count) CCM_CUDA(cudaMemcpyAsync(out, d_out, (size_t)count * sizeof(ccm_new_point), cudaMemcpyDeviceToHost, s.stream));
      if (best2) CCM_CUDA(cudaMemcpyAsync(best2, d_best2, cells * sizeof(int32_t), cudaMemcpyDeviceToHost, s.stream));
      if (verdict) CCM_CUDA(cudaMemcpyAsync(verdict, d_verdict, cells, cudaMemcpyDeviceToHost, s.stream));
      CCM_CUDA(cudaStreamSynchronize(s.stream));
    });
  });
}

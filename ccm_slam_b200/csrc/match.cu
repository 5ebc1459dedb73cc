// match.cu — 256-bit Hamming matching behind ccm_hamming_matrix / ccm_match_* (include/ccm_b200.h).
//
// The data-parallel part of ORBmatcher::SearchByBoW (S/ORBmatcher.cpp:178-306, 565-698) and SearchForTriangulation
// (:700-852) is DescriptorDistance (:1653-1669) over every candidate pair; k_hamming computes the whole nA x nB distance
// matrix in one launch (uint4 loads, shared-memory tiles, __popc).  The selection that follows is order dependent in the
// reference (a frame feature taken by an earlier keyframe feature is skipped by later ones; vbMatched2; ties), so it runs
// on the host over the distance matrix, in the reference's iteration order: vocabulary nodes ascending, features in
// FeatureVector order.  Rotation-histogram consistency keeps the reference's bin = round(rot / 30) arithmetic.
#include <cmath>

#include "common.cuh"

using namespace ccm;

namespace {

constexpr int TH_LOW = 50;        // ORBmatcher::TH_LOW      (S/ORBmatcher.cpp:64)
constexpr int HISTO_LENGTH = 30;  // ORBmatcher::HISTO_LENGTH (S/ORBmatcher.cpp:65)

// 32 x 32 output tile per CTA of 256 threads; each thread produces 4 distances
__global__ void __launch_bounds__(256) k_hamming(const uint4* __restrict__ A, int nA, const uint4* __restrict__ B, int nB,
                                                 uint16_t* __restrict__ D) {
  __shared__ uint4 sa[32][2], sb[32][2];
  const int i0 = blockIdx.y * 32, j0 = blockIdx.x * 32;
  const int t = threadIdx.x;
  if (t < 64) {
    const int r = t >> 1, h = t & 1;
    sa[r][h] = (i0 + r < nA) ? A[(size_t)(i0 + r) * 2 + h] : make_uint4(0, 0, 0, 0);
  } else if (t < 128) {
    const int r = (t - 64) >> 1, h = t & 1;
    sb[r][h] = (j0 + r < nB) ? B[(size_t)(j0 + r) * 2 + h] : make_uint4(0, 0, 0, 0);
  }
  __syncthreads();
  const int j = t & 31, ib = (t >> 5) * 4;
  const uint4 b0 = sb[j][0], b1 = sb[j][1];
#pragma unroll
  for (int k = 0; k < 4; k++) {
    const uint4 a0 = sa[ib + k][0], a1 = sa[ib + k][1];
    const int d = __popc(a0.x ^ b0.x) + __popc(a0.y ^ b0.y) + __popc(a0.z ^ b0.z) + __popc(a0.w ^ b0.w) +
                  __popc(a1.x ^ b1.x) + __popc(a1.y ^ b1.y) + __popc(a1.z ^ b1.z) + __popc(a1.w ^ b1.w);
    if (i0 + ib + k < nA && j0 + j < nB) D[(size_t)(i0 + ib + k) * nB + j0 + j] = (uint16_t)d;
  }
}

// per-thread staging (Staging; the matchers are called from several threads): the host operands go straight from the caller's memory
// into the device input block, the distances come back through the pinned output block
thread_local Staging t_stage;

// Either operand may already live on the device (dA / dB != nullptr: the keyframe store of kf_store.cu); host operands are uploaded.
const uint16_t* distance_matrix_any(const uint8_t* A, const uint4* dA, int nA, const uint8_t* B, const uint4* dB, int nB) {
  ensure_device();
  Staging& s = t_stage;
  const size_t n = (size_t)nA * nB;
  if (n == 0) return reinterpret_cast<const uint16_t*>(s.h_out);
  Packer lay;
  const size_t at_a = lay.reserve(dA ? 0 : (size_t)nA * 32), at_b = lay.reserve(dB ? 0 : (size_t)nB * 32);
  s.run([&] {
    s.reserve(lay.at, n * sizeof(uint16_t), 0, n * sizeof(uint16_t));
    if (!dA) {
      CCM_CUDA(cudaMemcpyAsync(s.in.p + at_a, A, (size_t)nA * 32, cudaMemcpyHostToDevice, s.stream));
      dA = reinterpret_cast<const uint4*>(s.in.p + at_a);
    }
    if (!dB) {
      CCM_CUDA(cudaMemcpyAsync(s.in.p + at_b, B, (size_t)nB * 32, cudaMemcpyHostToDevice, s.stream));
      dB = reinterpret_cast<const uint4*>(s.in.p + at_b);
    }
    uint16_t* D = reinterpret_cast<uint16_t*>(s.out.p);
    dim3 g(div_up(nB, 32), div_up(nA, 32));
    k_hamming<<<g, 256, 0, s.stream>>>(dA, nA, dB, nB, D);
    CCM_LAUNCHED();
    CCM_CUDA(cudaMemcpyAsync(s.h_out, D, n * sizeof(uint16_t), cudaMemcpyDeviceToHost, s.stream));
    CCM_CUDA(cudaStreamSynchronize(s.stream));
  });
  return reinterpret_cast<const uint16_t*>(s.h_out);
}
const uint16_t* distance_matrix(const uint8_t* A, int nA, const uint8_t* B, int nB) { return distance_matrix_any(A, nullptr, nA, B, nullptr, nB); }

struct RotHist {
  std::vector<int> bins[HISTO_LENGTH];
  void add(float a1, float a2, int what) {
    float rot = a1 - a2;
    if (rot < 0.0) rot += 360.0f;
    int bin = (int)round(rot * (1.0f / HISTO_LENGTH));
    if (bin == HISTO_LENGTH) bin = 0;
    bins[bin].push_back(what);
  }
  // ComputeThreeMaxima (S/ORBmatcher.cpp:1607-1648): calls `drop` for every entry outside the three dominant bins
  template <typename F>
  int prune(F&& drop) {
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

// walk the nodes two FeatureVectors share, ascending (the reference's merge-join with lower_bound)
template <typename F>
void for_shared_nodes(const ccm_feature_vector* f1, const ccm_feature_vector* f2, F&& body) {
  int a = 0, b = 0;
  while (a < f1->n_nodes && b < f2->n_nodes) {
    const uint32_t na = f1->node_id[a], nb = f2->node_id[b];
    if (na == nb) { body(a, b); a++; b++; }
    else if (na < nb) a++;
    else b++;
  }
}

void check_fv(const ccm_feature_vector* f, int n, const char* what) {
  CCM_REQUIRE(f && f->n_nodes >= 0 && (f->n_nodes == 0 || (f->node_id && f->node_ptr && f->feat)), what);
  for (int i = 0; i < f->n_nodes; i++) {
    CCM_REQUIRE(f->node_ptr[i] <= f->node_ptr[i + 1], what);
    if (i) CCM_REQUIRE(f->node_id[i - 1] < f->node_id[i], what);
  }
  for (int k = 0; k < (f->n_nodes ? f->node_ptr[f->n_nodes] : 0); k++) CCM_REQUIRE((int)f->feat[k] < n, what);
}

}  // namespace

// shared with proj_match.cu / kf_store.cu: the (thread-local, pinned) distance matrix of one call; valid until the next call on this thread
namespace ccm {
const uint16_t* hamming_matrix_host(const uint8_t* A, int nA, const uint8_t* B, int nB) { return distance_matrix(A, nA, B, nB); }
const uint16_t* hamming_matrix_mixed(const uint8_t* A, const void* dA, int nA, const uint8_t* B, const void* dB, int nB) {
  return distance_matrix_any(A, static_cast<const uint4*>(dA), nA, B, static_cast<const uint4*>(dB), nB);
}
}  // namespace ccm

extern "C" int ccm_hamming_matrix(const uint8_t* A, int32_t nA, const uint8_t* B, int32_t nB, uint16_t* D) {
  return guarded([&] {
    CCM_REQUIRE(nA >= 0 && nB >= 0 && (nA == 0 || A) && (nB == 0 || B) && D, "ccm_hamming_matrix: bad argument");
    const uint16_t* h = distance_matrix(A, nA, B, nB);
    if ((size_t)nA * nB) memcpy(D, h, (size_t)nA * nB * sizeof(uint16_t));
  });
}

// ---- the selection halves: everything after the distance matrix, on the host, in the reference's visiting order -------------------
namespace {
void select_bow_kf_frame(const uint16_t* D, int32_t n_kf, const uint8_t* kf_has_mp, const float* angle_kf, const ccm_feature_vector* fv_kf,
                       int32_t n_f, const float* angle_f, const ccm_feature_vector* fv_f, float nnratio, int32_t check_orientation,
                       int32_t* match_kf_of_f, int32_t* nmatches) {
  CCM_REQUIRE(match_kf_of_f && nmatches && kf_has_mp && (D || (size_t)n_kf * n_f == 0), "ccm_match_bow_kf_frame: null argument");
  check_fv(fv_kf, n_kf, "ccm_match_bow_kf_frame: bad keyframe FeatureVector");
  check_fv(fv_f, n_f, "ccm_match_bow_kf_frame: bad frame FeatureVector");
  for (int i = 0; i < n_f; i++) match_kf_of_f[i] = -1;
  int found = 0;
  RotHist hist;
  for_shared_nodes(fv_kf, fv_f, [&](int a, int b) {
    for (int ik = fv_kf->node_ptr[a]; ik < fv_kf->node_ptr[a + 1]; ik++) {
      const int i = (int)fv_kf->feat[ik];
      if (!kf_has_mp[i]) continue;
      const uint16_t* row = D + (size_t)i * n_f;
      int best = 256, second = 256, bestJ = -1;
      for (int jf = fv_f->node_ptr[b]; jf < fv_f->node_ptr[b + 1]; jf++) {
        const int j = (int)fv_f->feat[jf];
        if (match_kf_of_f[j] >= 0) continue;  // already holds a MapPoint
        const int d = row[j];
        if (d < best) { second = best; best = d; bestJ = j; }
        else if (d < second) second = d;
      }
      if (best <= TH_LOW && static_cast<float>(best) < nnratio * static_cast<float>(second)) {
        match_kf_of_f[bestJ] = i;
        if (check_orientation) hist.add(angle_kf[i], angle_f[bestJ], bestJ);
        found++;
      }
    }
  });
  if (check_orientation) found -= hist.prune([&](int j) { match_kf_of_f[j] = -1; });
  *nmatches = found;
}

void select_bow_kf_kf(const uint16_t* D, int32_t n1, const uint8_t* has_mp1, const float* angle1, const ccm_feature_vector* fv1, int32_t n2,
                    const uint8_t* has_mp2, const float* angle2, const ccm_feature_vector* fv2, float nnratio, int32_t check_orientation,
                    int32_t* match12, int32_t* nmatches) {
  CCM_REQUIRE(match12 && nmatches && has_mp1 && has_mp2 && (D || (size_t)n1 * n2 == 0), "ccm_match_bow_kf_kf: null argument");
  check_fv(fv1, n1, "ccm_match_bow_kf_kf: bad FeatureVector 1");
  check_fv(fv2, n2, "ccm_match_bow_kf_kf: bad FeatureVector 2");
  for (int i = 0; i < n1; i++) match12[i] = -1;
  std::vector<char> taken(n2, 0);
  int found = 0;
  RotHist hist;
  for_shared_nodes(fv1, fv2, [&](int a, int b) {
    for (int k1 = fv1->node_ptr[a]; k1 < fv1->node_ptr[a + 1]; k1++) {
      const int i = (int)fv1->feat[k1];
      if (!has_mp1[i]) continue;
      const uint16_t* row = D + (size_t)i * n2;
      int best = 256, second = 256, bestJ = -1;
      for (int k2 = fv2->node_ptr[b]; k2 < fv2->node_ptr[b + 1]; k2++) {
        const int j = (int)fv2->feat[k2];
        if (taken[j] || !has_mp2[j]) continue;
        const int d = row[j];
        if (d < best) { second = best; best = d; bestJ = j; }
        else if (d < second) second = d;
      }
      if (best < TH_LOW && static_cast<float>(best) < nnratio * static_cast<float>(second)) {  // strict '<' in this overload
        match12[i] = bestJ;
        taken[bestJ] = 1;
        if (check_orientation) hist.add(angle1[i], angle2[bestJ], i);
        found++;
      }
    }
  });
  if (check_orientation) found -= hist.prune([&](int i) { match12[i] = -1; });
  *nmatches = found;
}

void check_tri(const ccm_tri_view* v1, const ccm_tri_view* v2, const float F12[9], const float* level_sigma2, const float* scale_factors,
             int32_t nlevels, const int32_t* pairs, const int32_t* npairs) {
  CCM_REQUIRE(v1 && v2 && F12 && level_sigma2 && scale_factors && pairs && npairs, "ccm_match_triangulation: null argument");
  check_fv(v1->fv, v1->n, "ccm_match_triangulation: bad FeatureVector 1");
  check_fv(v2->fv, v2->n, "ccm_match_triangulation: bad FeatureVector 2");
  for (int j = 0; j < v2->n; j++) CCM_REQUIRE(v2->octave[j] >= 0 && v2->octave[j] < nlevels, "ccm_match_triangulation: octave out of range");
}

void select_triangulation(const uint16_t* D, const ccm_tri_view* v1, const ccm_tri_view* v2, const float F12[9], float ex, float ey,
                        const float* level_sigma2, const float* scale_factors, int32_t check_orientation, int32_t* pairs, int32_t* npairs) {
  CCM_REQUIRE(D || (size_t)v1->n * v2->n == 0, "ccm_select_triangulation: null distance matrix");
  std::vector<char> taken(v2->n, 0);
  std::vector<int> m12(v1->n, -1);
  int found = 0;
  RotHist hist;
  for_shared_nodes(v1->fv, v2->fv, [&](int a, int b) {
    for (int k1 = v1->fv->node_ptr[a]; k1 < v1->fv->node_ptr[a + 1]; k1++) {
      const int i = (int)v1->fv->feat[k1];
      if (v1->has_mp[i]) continue;  // only untracked keypoints are triangulated
      const float x1 = v1->kp_xy[2 * i], y1 = v1->kp_xy[2 * i + 1];
      // epipolar line of kp1 in image 2: l = x1' F12 (CheckDistEpipolarLine, S/ORBmatcher.cpp:159-176), f32 arithmetic
      const float la = x1 * F12[0] + y1 * F12[3] + F12[6];
      const float lb = x1 * F12[1] + y1 * F12[4] + F12[7];
      const float lc = x1 * F12[2] + y1 * F12[5] + F12[8];
      const float den = la * la + lb * lb;
      const uint16_t* row = D + (size_t)i * v2->n;
      int bestDist = TH_LOW, bestJ = -1;
      for (int k2 = v2->fv->node_ptr[b]; k2 < v2->fv->node_ptr[b + 1]; k2++) {
        const int j = (int)v2->fv->feat[k2];
        if (taken[j] || v2->has_mp[j]) continue;  // vbMatched2 is never set in the reference; kept for fidelity
        const int d = row[j];
        if (d > TH_LOW || d > bestDist) continue;   // ties replace the incumbent
        const float x2 = v2->kp_xy[2 * j], y2 = v2->kp_xy[2 * j + 1];
        const float dex = ex - x2, dey = ey - y2;
        if (dex * dex + dey * dey < 100 * scale_factors[v2->octave[j]]) continue;  // too close to the epipole
        const float num = la * x2 + lb * y2 + lc;
        if (den == 0) continue;
        const float dsqr = num * num / den;
        if (dsqr < 3.84 * level_sigma2[v2->octave[j]]) { bestJ = j; bestDist = d; }
      }
      if (bestJ >= 0) {
        m12[i] = bestJ;
        found++;
        if (check_orientation) hist.add(v1->angle[i], v2->angle[bestJ], i);
      }
    }
  });
  if (check_orientation) found -= hist.prune([&](int i) { m12[i] = -1; });
  int np = 0;
  for (int i = 0; i < v1->n; i++)
    if (m12[i] >= 0) { pairs[2 * np] = i; pairs[2 * np + 1] = m12[i]; np++; }
  *npairs = np;
}
}  // namespace

extern "C" int ccm_match_bow_kf_frame(const uint8_t* desc_kf, int32_t n_kf, const uint8_t* kf_has_mp, const float* angle_kf,
                                      const ccm_feature_vector* fv_kf, const uint8_t* desc_f, int32_t n_f, const float* angle_f,
                                      const ccm_feature_vector* fv_f, float nnratio, int32_t check_orientation,
                                      int32_t* match_kf_of_f, int32_t* nmatches) {
  return guarded([&] {
    CCM_REQUIRE(n_kf >= 0 && n_f >= 0 && (n_kf == 0 || desc_kf) && (n_f == 0 || desc_f), "ccm_match_bow_kf_frame: bad descriptors");
    select_bow_kf_frame(distance_matrix(desc_kf, n_kf, desc_f, n_f), n_kf, kf_has_mp, angle_kf, fv_kf, n_f, angle_f, fv_f, nnratio,
                        check_orientation, match_kf_of_f, nmatches);
  });
}
extern "C" int ccm_select_bow_kf_frame(const uint16_t* D, int32_t n_kf, const uint8_t* kf_has_mp, const float* angle_kf,
                                       const ccm_feature_vector* fv_kf, int32_t n_f, const float* angle_f, const ccm_feature_vector* fv_f,
                                       float nnratio, int32_t check_orientation, int32_t* match_kf_of_f, int32_t* nmatches) {
  return guarded([&] {
    CCM_REQUIRE(n_kf >= 0 && n_f >= 0, "ccm_select_bow_kf_frame: bad sizes");
    select_bow_kf_frame(D, n_kf, kf_has_mp, angle_kf, fv_kf, n_f, angle_f, fv_f, nnratio, check_orientation, match_kf_of_f, nmatches);
  });
}

extern "C" int ccm_match_bow_kf_kf(const uint8_t* desc1, int32_t n1, const uint8_t* has_mp1, const float* angle1,
                                   const ccm_feature_vector* fv1, const uint8_t* desc2, int32_t n2, const uint8_t* has_mp2,
                                   const float* angle2, const ccm_feature_vector* fv2, float nnratio,
                                   int32_t check_orientation, int32_t* match12, int32_t* nmatches) {
  return guarded([&] {
    CCM_REQUIRE(n1 >= 0 && n2 >= 0 && (n1 == 0 || desc1) && (n2 == 0 || desc2), "ccm_match_bow_kf_kf: bad descriptors");
    select_bow_kf_kf(distance_matrix(desc1, n1, desc2, n2), n1, has_mp1, angle1, fv1, n2, has_mp2, angle2, fv2, nnratio, check_orientation,
                     match12, nmatches);
  });
}
extern "C" int ccm_select_bow_kf_kf(const uint16_t* D, int32_t n1, const uint8_t* has_mp1, const float* angle1, const ccm_feature_vector* fv1,
                                    int32_t n2, const uint8_t* has_mp2, const float* angle2, const ccm_feature_vector* fv2, float nnratio,
                                    int32_t check_orientation, int32_t* match12, int32_t* nmatches) {
  return guarded([&] {
    CCM_REQUIRE(n1 >= 0 && n2 >= 0, "ccm_select_bow_kf_kf: bad sizes");
    select_bow_kf_kf(D, n1, has_mp1, angle1, fv1, n2, has_mp2, angle2, fv2, nnratio, check_orientation, match12, nmatches);
  });
}

extern "C" int ccm_match_triangulation(const ccm_tri_view* v1, const ccm_tri_view* v2, const float F12[9], float ex, float ey,
                                       const float* level_sigma2, const float* scale_factors, int32_t nlevels,
                                       int32_t check_orientation, int32_t* pairs, int32_t* npairs) {
  return guarded([&] {
    check_tri(v1, v2, F12, level_sigma2, scale_factors, nlevels, pairs, npairs);
    select_triangulation(distance_matrix(v1->desc, v1->n, v2->desc, v2->n), v1, v2, F12, ex, ey, level_sigma2, scale_factors,
                         check_orientation, pairs, npairs);
  });
}
extern "C" int ccm_select_triangulation(const uint16_t* D, const ccm_tri_view* v1, const ccm_tri_view* v2, const float F12[9], float ex, float ey,
                                        const float* level_sigma2, const float* scale_factors, int32_t nlevels,
                                        int32_t check_orientation, int32_t* pairs, int32_t* npairs) {
  return guarded([&] {
    check_tri(v1, v2, F12, level_sigma2, scale_factors, nlevels, pairs, npairs);
    select_triangulation(D, v1, v2, F12, ex, ey, level_sigma2, scale_factors, check_orientation, pairs, npairs);
  });
}

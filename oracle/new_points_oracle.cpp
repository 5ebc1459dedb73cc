// new_points_oracle.cpp — CPU oracle for LocalMapping::CreateNewMapPoints (TEST INFRASTRUCTURE, NOT PRODUCT).
//
// The sequential loop as the reference writes it (S/Mapping.cpp:312-468): neighbour by neighbour, SearchForTriangulation through the
// oracle's reference-pinned orc_match_triangulation (match_oracle.cpp) with check_ori = false, each match triangulated and gated in
// the order of :362-448, and has_mp1[idx1] set after each accepted point (:456) so that the next neighbour's search skips it.
// The expressions below are the reference's, written out in C++ float / double arithmetic (this file is compiled with
// -ffp-contract=off); only the 4x4 decomposition comes from the product's new_points_math.cuh, because cv::SVD::compute has no
// single bit pattern of its own (OpenCV's Jacobi iteration or LAPACK's sgesdd, by build) and the product states one.
//
// mutate (tests only): 1 = a pair that fails a gate still sets has_mp1, i.e. a rejected pair claims its feature.
#include <cmath>
#include <cstdint>
#include <cstring>
#include <vector>

#include "../ccm_slam_b200/csrc/new_points_math.cuh"
#include "ccm_b200.h"

extern "C" int orc_match_triangulation(const ccm_tri_view* v1, const ccm_tri_view* v2, const float F12[9], float ex, float ey,
                                       const float* level_sigma2, const float* scale_factors, int check_ori, int* pairs);

namespace {

double norm3(float x, float y, float z) { return std::sqrt((double)x * x + (double)y * y + (double)z * z); }

// Rcw.row(r).dot(x3Dt) + tcw(r): Mat::dot in double, the float translation added in double, stored to float
float cam_row(const float* T, int r, const float* X) {
  const double d = (double)T[4 * r] * X[0] + (double)T[4 * r + 1] * X[1] + (double)T[4 * r + 2] * X[2];
  return (float)(d + T[4 * r + 3]);
}

uint8_t triangulate(const ccm_newpts_view* k1, const ccm_newpts_view* k2, int idx1, int idx2, float ratioFactor, float* X) {
  const float *Tcw1 = k1->Tcw, *Tcw2 = k2->Tcw;
  const float fx1 = k1->v.fx, fy1 = k1->v.fy, cx1 = k1->v.cx, cy1 = k1->v.cy, invfx1 = 1.0f / fx1, invfy1 = 1.0f / fy1;
  const float fx2 = k2->v.fx, fy2 = k2->v.fy, cx2 = k2->v.cx, cy2 = k2->v.cy, invfx2 = 1.0f / fx2, invfy2 = 1.0f / fy2;
  const float kp1x = k1->v.kp_xy[2 * idx1], kp1y = k1->v.kp_xy[2 * idx1 + 1];
  const float kp2x = k2->v.kp_xy[2 * idx2], kp2y = k2->v.kp_xy[2 * idx2 + 1];
  const int oct1 = k1->v.octave[idx1], oct2 = k2->v.octave[idx2];

  const float xn1[3] = {(kp1x - cx1) * invfx1, (kp1y - cy1) * invfy1, 1.0f};
  const float xn2[3] = {(kp2x - cx2) * invfx2, (kp2y - cy2) * invfy2, 1.0f};
  float ray1[3], ray2[3];
  for (int i = 0; i < 3; i++) {   // Rwc = Rcw.t()
    ray1[i] = Tcw1[i] * xn1[0] + Tcw1[4 + i] * xn1[1] + Tcw1[8 + i] * xn1[2];
    ray2[i] = Tcw2[i] * xn2[0] + Tcw2[4 + i] * xn2[1] + Tcw2[8 + i] * xn2[2];
  }
  const double dot = (double)ray1[0] * ray2[0] + (double)ray1[1] * ray2[1] + (double)ray1[2] * ray2[2];
  const float cosParallaxRays = (float)(dot / (norm3(ray1[0], ray1[1], ray1[2]) * norm3(ray2[0], ray2[1], ray2[2])));
  const float cosParallaxStereo = cosParallaxRays + 1;
  if (!(cosParallaxRays < cosParallaxStereo && cosParallaxRays > 0 && (cosParallaxRays < 0.9998))) return CCM_NEWPTS_PARALLAX;

  float A[16];
  for (int j = 0; j < 4; j++) {
    A[j] = xn1[0] * Tcw1[8 + j] - Tcw1[j];
    A[4 + j] = xn1[1] * Tcw1[8 + j] - Tcw1[4 + j];
    A[8 + j] = xn2[0] * Tcw2[8 + j] - Tcw2[j];
    A[12 + j] = xn2[1] * Tcw2[8 + j] - Tcw2[4 + j];
  }
  float x3D[4];
  ccm::newpts::svd4_null(A, x3D);
  if (x3D[3] == 0) return CCM_NEWPTS_W_ZERO;
  const float inv_w = (float)(1.0 / x3D[3]);           // Mat / double: convertTo with the scale taken as float
  for (int i = 0; i < 3; i++) X[i] = x3D[i] * inv_w + 0.f;

  const float z1 = cam_row(Tcw1, 2, X);
  if (z1 <= 0) return CCM_NEWPTS_DEPTH1;
  const float z2 = cam_row(Tcw2, 2, X);
  if (z2 <= 0) return CCM_NEWPTS_DEPTH2;

  const float sigmaSquare1 = k1->level_sigma2[oct1];
  const float x1 = cam_row(Tcw1, 0, X), y1 = cam_row(Tcw1, 1, X);
  const float invz1 = 1.0 / z1;
  const float u1 = fx1 * x1 * invz1 + cx1, v1 = fy1 * y1 * invz1 + cy1;
  const float errX1 = u1 - kp1x, errY1 = v1 - kp1y;
  if ((errX1 * errX1 + errY1 * errY1) > 5.991 * sigmaSquare1) return CCM_NEWPTS_REPROJ1;

  const float sigmaSquare2 = k2->level_sigma2[oct2];
  const float x2 = cam_row(Tcw2, 0, X), y2 = cam_row(Tcw2, 1, X);
  const float invz2 = 1.0 / z2;
  const float u2 = fx2 * x2 * invz2 + cx2, v2 = fy2 * y2 * invz2 + cy2;
  const float errX2 = u2 - kp2x, errY2 = v2 - kp2y;
  if ((errX2 * errX2 + errY2 * errY2) > 5.991 * sigmaSquare2) return CCM_NEWPTS_REPROJ2;

  const float dist1 = norm3(X[0] - k1->Ow[0], X[1] - k1->Ow[1], X[2] - k1->Ow[2]);
  const float dist2 = norm3(X[0] - k2->Ow[0], X[1] - k2->Ow[1], X[2] - k2->Ow[2]);
  if (dist1 == 0 || dist2 == 0) return CCM_NEWPTS_DIST_ZERO;
  const float ratioDist = dist2 / dist1;
  const float ratioOctave = k1->scale_factors[oct1] / k2->scale_factors[oct2];
  if (ratioDist * ratioFactor < ratioOctave || ratioDist > ratioOctave * ratioFactor) return CCM_NEWPTS_SCALE;
  return CCM_NEWPTS_ACCEPTED;
}

}  // namespace

// the contract of ccm_new_map_points on valid input; returns 0, or 1 when capacity is too small (*n_out then holds the count needed)
extern "C" int orc_new_map_points(const ccm_newpts_view* cur, const ccm_newpts_neighbour* nb, int32_t n_nb, ccm_new_point* out,
                                  int32_t capacity, int32_t* n_out, int32_t* best2, uint8_t* verdict, int32_t mutate) {
  const int n = cur->v.n;
  std::vector<uint8_t> has_mp1(cur->v.has_mp, cur->v.has_mp + n), by_call(n, 0);
  std::vector<int> pairs(2 * (size_t)n + 2);
  std::vector<ccm_new_point> pts;
  std::vector<int32_t> b2((size_t)n * n_nb, -1);
  std::vector<uint8_t> vd((size_t)n * n_nb, CCM_NEWPTS_NONE);
  const float ratioFactor = 1.5f * cur->scale_factor;
  for (int i = 0; i < n_nb; i++) {
    const ccm_newpts_view* k2 = &nb[i].view;
    for (int f = 0; f < n; f++)
      if (by_call[f]) vd[(size_t)i * n + f] = CCM_NEWPTS_CLAIMED;
    ccm_tri_view v1 = cur->v;
    v1.has_mp = has_mp1.data();
    const int nmatches = orc_match_triangulation(&v1, &k2->v, nb[i].F12, nb[i].ex, nb[i].ey, k2->level_sigma2, k2->scale_factors, 0, pairs.data());
    for (int ikp = 0; ikp < nmatches; ikp++) {
      const int idx1 = pairs[2 * ikp], idx2 = pairs[2 * ikp + 1];
      float X[3] = {0.f, 0.f, 0.f};
      const uint8_t verd = triangulate(cur, k2, idx1, idx2, ratioFactor, X);
      b2[(size_t)i * n + idx1] = idx2;
      vd[(size_t)i * n + idx1] = verd;
      if (verd == CCM_NEWPTS_ACCEPTED) {
        ccm_new_point p;
        p.nb = i; p.idx1 = idx1; p.idx2 = idx2;
        memcpy(p.x3D, X, sizeof X);
        pts.push_back(p);
      }
      if (verd == CCM_NEWPTS_ACCEPTED || mutate == 1) { has_mp1[idx1] = 1; by_call[idx1] = 1; }   // AddMapPoint(pMP, idx1)
    }
  }
  *n_out = (int32_t)pts.size();
  if (capacity < (int32_t)pts.size()) return 1;
  if (!pts.empty()) memcpy(out, pts.data(), pts.size() * sizeof(ccm_new_point));
  if (best2 && !b2.empty()) memcpy(best2, b2.data(), b2.size() * sizeof(int32_t));
  if (verdict && !vd.empty()) memcpy(verdict, vd.data(), vd.size());
  return 0;
}

// the decomposition alone, for the witness comparison: A row-major 4x4 -> vt.row(3)
extern "C" void orc_svd4_null(const float* A, float* x) { ccm::newpts::svd4_null(A, x); }

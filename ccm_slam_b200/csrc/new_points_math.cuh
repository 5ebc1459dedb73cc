// new_points_math.cuh — arithmetic of LocalMapping::CreateNewMapPoints (cslam/src/Mapping.cpp:362-448) and of the gates of
// ORBmatcher::SearchForTriangulation (cslam/src/ORBmatcher.cpp:159-176, 770-778), shared by the kernels (new_points.cu, nvcc), the host
// entry point ccm_new_map_points_host and the oracle (g++ -ffp-contract=off).  Every product and sum is one explicit rounding, so the
// device contracts nothing the host does not.
//
// The reference evaluates cv::Mat expressions on CV_32F data.  What each one does, and how it is written here:
//   xn = ((x-cx)*invfx, (y-cy)*invfy, 1)    f32, invfx = 1.0f/fx (Frame's member)
//   ray = Rwc*xn                            a 3x3 by 3x1 CV_32F product: f32 products summed left to right
//   cosParallaxRays                         Mat::dot and cv::norm accumulate in double; the quotient is formed in double and rounded once
//   A.row(k) = xn_k*Tcw.row(2)-Tcw.row(k')  f32: one product, one difference per entry
//   cv::SVD::compute(A), vt.row(3)          svd4_null below.  OpenCV runs its own Jacobi iteration or LAPACK's sgesdd depending on how it
//                                           was built, so the reference has no single bit pattern here; this file states one.
//   x3D.rowRange(0,3)/x3D(3)                Mat / double is convertTo with scale 1.0/w taken as float: x * (float)(1.0/w) + 0.f
//   z = Rcw.row(2).dot(x3Dt)+tcw(2)         Mat::dot returns double, the float tcw entry is added in double, the sum rounded to float
//   invz = 1.0/z                            double quotient rounded to float
//   u = fx*x*invz+cx                        f32, left to right
//   err2 > 5.991*sigma2                     f32 sum of squares against a double product (5.991 is a double constant)
//   dist = cv::norm(x3D-Ow)                 f32 difference, double norm, rounded to float
//   ratioDist, ratioOctave and their gate   f32
#pragma once
#include <stdint.h>

#include <cmath>

#if defined(__CUDACC__)
#define CCM_NP_HD __host__ __device__ __forceinline__
#else
#define CCM_NP_HD inline
#endif

namespace ccm {
namespace newpts {

// verdict of one (neighbour, feature) pair; the values of ccm_newpts_verdict (include/ccm_b200.h)
enum : uint8_t { NONE = 0, ACCEPTED = 1, PARALLAX = 2, W_ZERO = 3, DEPTH1 = 4, DEPTH2 = 5, REPROJ1 = 6, REPROJ2 = 7, DIST_ZERO = 8,
                 SCALE = 9, CLAIMED = 10 };

constexpr int TH_LOW = 50;            // ORBmatcher::TH_LOW (cslam/src/ORBmatcher.cpp:64)
constexpr int SVD_MAX_SWEEPS = 30;
constexpr float SVD_EPS = 2.384185791015625e-07f;   // 2^-22

CCM_NP_HD float fsub(float a, float b) {
#if defined(__CUDA_ARCH__)
  return __fsub_rn(a, b);
#else
  return a - b;
#endif
}
CCM_NP_HD float fmul(float a, float b) {
#if defined(__CUDA_ARCH__)
  return __fmul_rn(a, b);
#else
  return a * b;
#endif
}
CCM_NP_HD float fadd(float a, float b) {
#if defined(__CUDA_ARCH__)
  return __fadd_rn(a, b);
#else
  return a + b;
#endif
}
CCM_NP_HD float fdiv(float a, float b) {
#if defined(__CUDA_ARCH__)
  return __fdiv_rn(a, b);
#else
  return a / b;
#endif
}
CCM_NP_HD float fsqrt(float a) {
#if defined(__CUDA_ARCH__)
  return __fsqrt_rn(a);
#else
  return std::sqrt(a);
#endif
}
CCM_NP_HD double dmul(double a, double b) {
#if defined(__CUDA_ARCH__)
  return __dmul_rn(a, b);
#else
  return a * b;
#endif
}
CCM_NP_HD double dadd(double a, double b) {
#if defined(__CUDA_ARCH__)
  return __dadd_rn(a, b);
#else
  return a + b;
#endif
}
CCM_NP_HD double ddiv(double a, double b) {
#if defined(__CUDA_ARCH__)
  return __ddiv_rn(a, b);
#else
  return a / b;
#endif
}
CCM_NP_HD double dsqrt(double a) {
#if defined(__CUDA_ARCH__)
  return __dsqrt_rn(a);
#else
  return std::sqrt(a);
#endif
}
CCM_NP_HD float to_f32(double a) {
#if defined(__CUDA_ARCH__)
  return __double2float_rn(a);
#else
  return (float)a;
#endif
}

// ---- the gates of SearchForTriangulation's inner loop ----------------------------------------------------------------------------

// l = x1' F12 (CheckDistEpipolarLine); l[3] = a*a + b*b
CCM_NP_HD void epipolar_line(float x1, float y1, const float* F, float l[4]) {
  l[0] = fadd(fadd(fmul(x1, F[0]), fmul(y1, F[3])), F[6]);
  l[1] = fadd(fadd(fmul(x1, F[1]), fmul(y1, F[4])), F[7]);
  l[2] = fadd(fadd(fmul(x1, F[2]), fmul(y1, F[5])), F[8]);
  l[3] = fadd(fmul(l[0], l[0]), fmul(l[1], l[1]));
}

// the epipole gate (:775-778), then CheckDistEpipolarLine (:166-175) for a feature of the neighbour at (x2, y2)
CCM_NP_HD bool passes_epipolar(const float l[4], float ex, float ey, float x2, float y2, float scale2, float sigma2_2) {
  const float dx = fsub(ex, x2), dy = fsub(ey, y2);
  if (fadd(fmul(dx, dx), fmul(dy, dy)) < fmul(100.f, scale2)) return false;
  const float num = fadd(fadd(fmul(l[0], x2), fmul(l[1], y2)), l[2]);
  if (l[3] == 0) return false;
  const float dsqr = fdiv(fmul(num, num), l[3]);
  return (double)dsqr < dmul(3.84, (double)sigma2_2);
}

// ---- the 4x4 singular value decomposition ---------------------------------------------------------------------------------------
//
// One-sided Jacobi (Hestenes) in f32 on the columns of W = A, V = I.  A sweep visits the column pairs (p, q) in the order
// (0,1) (0,2) (0,3) (1,2) (1,3) (2,3).  For a pair: a = sum_k W[k][p]^2, b = sum_k W[k][q]^2, c = sum_k W[k][p] W[k][q], each summed
// over k = 0..3 in order.  The pair is left alone when |c| <= 2^-22 * sqrt(a*b).  Otherwise, with p2 = 2c, beta = a - b,
// gamma = sqrt(p2*p2 + beta*beta):
//   beta <  0:  s  = sqrt(((gamma - beta) * 0.5) / gamma),  cs = p2 / ((gamma * s) * 2)
//   beta >= 0:  cs = sqrt((gamma + beta) / (gamma * 2)),    s  = p2 / ((gamma * cs) * 2)
// and columns p, q of W and of V become (cs*x + s*y, cs*y - s*x).  The iteration ends after the first sweep that rotates nothing, or
// after SVD_MAX_SWEEPS sweeps.  The squared singular values are the column sums a_j recomputed at the end; sorted descending, equal
// values keeping ascending column order, the last one is the highest column among the smallest.  vt.row(3) is that column of V.
// Its sign is whatever the rotations left: it cancels in x / w.
template <int P, int Q>
CCM_NP_HD bool jacobi_pair(float* W, float* V) {
  float a = 0.f, b = 0.f, c = 0.f;
#pragma unroll
  for (int k = 0; k < 4; k++) {
    const float x = W[4 * k + P], y = W[4 * k + Q];
    a = fadd(a, fmul(x, x)); b = fadd(b, fmul(y, y)); c = fadd(c, fmul(x, y));
  }
  if (!(std::fabs(c) > fmul(SVD_EPS, fsqrt(fmul(a, b))))) return false;
  const float p2 = fmul(c, 2.f), beta = fsub(a, b);
  const float gamma = fsqrt(fadd(fmul(p2, p2), fmul(beta, beta)));
  float cs, s;
  if (beta < 0) {
    s = fsqrt(fdiv(fmul(fsub(gamma, beta), 0.5f), gamma));
    cs = fdiv(p2, fmul(fmul(gamma, s), 2.f));
  } else {
    cs = fsqrt(fdiv(fadd(gamma, beta), fmul(gamma, 2.f)));
    s = fdiv(p2, fmul(fmul(gamma, cs), 2.f));
  }
#pragma unroll
  for (int k = 0; k < 4; k++) {
    const float x = W[4 * k + P], y = W[4 * k + Q];
    W[4 * k + P] = fadd(fmul(cs, x), fmul(s, y));
    W[4 * k + Q] = fsub(fmul(cs, y), fmul(s, x));
    const float vx = V[4 * k + P], vy = V[4 * k + Q];
    V[4 * k + P] = fadd(fmul(cs, vx), fmul(s, vy));
    V[4 * k + Q] = fsub(fmul(cs, vy), fmul(s, vx));
  }
  return true;
}

// A row-major 4x4; x = the right singular vector of the smallest singular value (vt.row(3))
CCM_NP_HD void svd4_null(const float A[16], float x[4]) {
  float W[16], V[16];
#pragma unroll
  for (int k = 0; k < 16; k++) { W[k] = A[k]; V[k] = (k % 5 == 0) ? 1.f : 0.f; }
  for (int sweep = 0; sweep < SVD_MAX_SWEEPS; sweep++) {
    bool r = jacobi_pair<0, 1>(W, V);
    r |= jacobi_pair<0, 2>(W, V);
    r |= jacobi_pair<0, 3>(W, V);
    r |= jacobi_pair<1, 2>(W, V);
    r |= jacobi_pair<1, 3>(W, V);
    r |= jacobi_pair<2, 3>(W, V);
    if (!r) break;
  }
  float best = 0.f;
#pragma unroll
  for (int j = 0; j < 4; j++) {
    float a = 0.f;
#pragma unroll
    for (int k = 0; k < 4; k++) a = fadd(a, fmul(W[4 * k + j], W[4 * k + j]));
    if (j == 0 || a <= best) {
      best = a;
#pragma unroll
      for (int k = 0; k < 4; k++) x[k] = V[4 * k + j];
    }
  }
}

// ---- triangulation and its gates ------------------------------------------------------------------------------------------------

struct Camera {       // one keyframe as the triangulation reads it
  float fx, fy, cx, cy;
  float T[12];        // [Rcw | tcw], 3x4 row-major
  float O[3];         // camera centre
};

// Rcw.row(r).dot(X) + tcw(r)
CCM_NP_HD float cam_coord(const float* T, int r, const float X[3]) {
  double d = dmul((double)T[4 * r], (double)X[0]);
  d = dadd(d, dmul((double)T[4 * r + 1], (double)X[1]));
  d = dadd(d, dmul((double)T[4 * r + 2], (double)X[2]));
  return to_f32(dadd(d, (double)T[4 * r + 3]));
}

CCM_NP_HD double norm3(const float d[3]) {
  double s = dmul((double)d[0], (double)d[0]);
  s = dadd(s, dmul((double)d[1], (double)d[1]));
  s = dadd(s, dmul((double)d[2], (double)d[2]));
  return dsqrt(s);
}

// (x, y) the undistorted keypoint, z the depth already gated; true when the reprojection error passes
CCM_NP_HD bool reprojection_ok(const Camera& c, const float X[3], float z, float x, float y, float sigma2) {
  const float xc = cam_coord(c.T, 0, X), yc = cam_coord(c.T, 1, X);
  const float invz = to_f32(ddiv(1.0, (double)z));
  const float u = fadd(fmul(fmul(c.fx, xc), invz), c.cx);
  const float v = fadd(fmul(fmul(c.fy, yc), invz), c.cy);
  const float ex = fsub(u, x), ey = fsub(v, y);
  return !((double)fadd(fmul(ex, ex), fmul(ey, ey)) > dmul(5.991, (double)sigma2));
}

// One matched pair: keypoint (x1, y1) of the current keyframe c1 at an octave with mvLevelSigma2 sigma2_1 and mvScaleFactors scale1,
// likewise for the neighbour c2; ratio_factor = 1.5f * mfScaleFactor of the current keyframe.  Returns the verdict; X is written
// whenever the gates reached it (every verdict from DEPTH1 on).
CCM_NP_HD uint8_t triangulate_pair(const Camera& c1, const Camera& c2, float x1, float y1, float sigma2_1, float scale1, float x2, float y2,
                                   float sigma2_2, float scale2, float ratio_factor, float X[3]) {
  const float xn1[3] = {fmul(fsub(x1, c1.cx), fdiv(1.f, c1.fx)), fmul(fsub(y1, c1.cy), fdiv(1.f, c1.fy)), 1.f};
  const float xn2[3] = {fmul(fsub(x2, c2.cx), fdiv(1.f, c2.fx)), fmul(fsub(y2, c2.cy), fdiv(1.f, c2.fy)), 1.f};
  float r1[3], r2[3];
#pragma unroll
  for (int i = 0; i < 3; i++) {   // Rwc = Rcw.t()
    r1[i] = fadd(fadd(fmul(c1.T[i], xn1[0]), fmul(c1.T[4 + i], xn1[1])), fmul(c1.T[8 + i], xn1[2]));
    r2[i] = fadd(fadd(fmul(c2.T[i], xn2[0]), fmul(c2.T[4 + i], xn2[1])), fmul(c2.T[8 + i], xn2[2]));
  }
  double dot = dmul((double)r1[0], (double)r2[0]);
  dot = dadd(dot, dmul((double)r1[1], (double)r2[1]));
  dot = dadd(dot, dmul((double)r1[2], (double)r2[2]));
  const float cosp = to_f32(ddiv(dot, dmul(norm3(r1), norm3(r2))));
  if (!(cosp < fadd(cosp, 1.f) && cosp > 0 && (double)cosp < 0.9998)) return PARALLAX;

  float A[16];
#pragma unroll
  for (int j = 0; j < 4; j++) {
    A[j] = fsub(fmul(xn1[0], c1.T[8 + j]), c1.T[j]);
    A[4 + j] = fsub(fmul(xn1[1], c1.T[8 + j]), c1.T[4 + j]);
    A[8 + j] = fsub(fmul(xn2[0], c2.T[8 + j]), c2.T[j]);
    A[12 + j] = fsub(fmul(xn2[1], c2.T[8 + j]), c2.T[4 + j]);
  }
  float h[4];
  svd4_null(A, h);
  if (h[3] == 0) return W_ZERO;
  const float s = to_f32(ddiv(1.0, (double)h[3]));
#pragma unroll
  for (int i = 0; i < 3; i++) X[i] = fadd(fmul(h[i], s), 0.f);

  const float z1 = cam_coord(c1.T, 2, X);
  if (z1 <= 0) return DEPTH1;
  const float z2 = cam_coord(c2.T, 2, X);
  if (z2 <= 0) return DEPTH2;
  if (!reprojection_ok(c1, X, z1, x1, y1, sigma2_1)) return REPROJ1;
  if (!reprojection_ok(c2, X, z2, x2, y2, sigma2_2)) return REPROJ2;

  const float n1[3] = {fsub(X[0], c1.O[0]), fsub(X[1], c1.O[1]), fsub(X[2], c1.O[2])};
  const float n2[3] = {fsub(X[0], c2.O[0]), fsub(X[1], c2.O[1]), fsub(X[2], c2.O[2])};
  const float dist1 = to_f32(norm3(n1)), dist2 = to_f32(norm3(n2));
  if (dist1 == 0 || dist2 == 0) return DIST_ZERO;
  const float ratio_dist = fdiv(dist2, dist1), ratio_octave = fdiv(scale1, scale2);
  if (fmul(ratio_dist, ratio_factor) < ratio_octave || ratio_dist > fmul(ratio_octave, ratio_factor)) return SCALE;
  return ACCEPTED;
}

}  // namespace newpts
}  // namespace ccm

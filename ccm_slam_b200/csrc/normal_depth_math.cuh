// normal_depth_math.cuh — arithmetic of MapPoint::UpdateNormalAndDepth (cslam/src/MapPoint.cpp:779-823), shared by the kernel
// (normal_depth.cu), the host entry point ccm_normal_depth_host and a host build in tests/ (g++ -ffp-contract=off).
//
// The reference evaluates cv::Mat expressions on CV_32F 3-vectors.  What each one does in OpenCV, and how it is pinned:
//   d = X - O_k                 cv::subtract, f32: one rounding
//   r = cv::norm(d)             norm.cpp, the contiguous CV_32F / NORM_L2 path (normL2Sqr_<float,double>): each component widened to
//                               double, squares summed in index order in double, std::sqrt.  Checked against cv2.norm 4.13.
//   normal = normal + d/r       MatOp_AddEx folds `d/r` (alpha = 1.0/r in double) and `+ normal` into cv::scaleAdd(d, 1.0/r, normal),
//                               which for f32 is fmaf(d_i, (float)(1.0/r), normal_i): one rounding.  Checked against cv2.scaleAdd 4.13
//                               (a separate multiply and add differs in most cases).
//   mNormalVector = normal/n    MatOp_AddEx::assign turns `Mat / double` into convertTo(dst, CV_32F, 1.0/n, 0); convert_scale.simd.hpp's
//                               cvt_32f takes the scale as float and, for a 3-vector (shorter than one SIMD pair), runs its scalar tail
//                               dst[j] = src[j]*a + b with a = (float)(1.0/n), b = 0.f: x * (float)(1.0/n), not x / n.  Pinned to that
//                               source line (python's cv2 has no convertTo); the + 0.f is kept because it turns -0 into +0.
//   dist = cv::norm(Pos - O_ref) as r, then rounded to float
//   mfMaxDistance = dist * scale_ref, mfMinDistance = mfMaxDistance / scale_last: f32, one rounding each.
// n = 0 (every observer bad) gives 1.0/0 = inf and 0 * inf = NaN per component; a point on an observer's centre gives r = 0 and the
// same NaN.  Both are the reference's values and are reproduced, not filtered.
#pragma once
#include <stdint.h>

#include <cmath>

#if defined(__CUDACC__)
#define CCM_ND_HD __host__ __device__ __forceinline__
#else
#define CCM_ND_HD inline
#endif

namespace ccm {
namespace nd {

CCM_ND_HD float fsub(float a, float b) {
#if defined(__CUDA_ARCH__)
  return __fsub_rn(a, b);
#else
  return a - b;
#endif
}
CCM_ND_HD float fmul(float a, float b) {
#if defined(__CUDA_ARCH__)
  return __fmul_rn(a, b);
#else
  return a * b;
#endif
}
CCM_ND_HD float fadd(float a, float b) {
#if defined(__CUDA_ARCH__)
  return __fadd_rn(a, b);
#else
  return a + b;
#endif
}
CCM_ND_HD float fdiv(float a, float b) {
#if defined(__CUDA_ARCH__)
  return __fdiv_rn(a, b);
#else
  return a / b;
#endif
}
CCM_ND_HD float ffma(float a, float b, float c) {   // the one fused step: cv::scaleAdd
#if defined(__CUDA_ARCH__)
  return __fmaf_rn(a, b, c);
#else
  return std::fma(a, b, c);
#endif
}
CCM_ND_HD double drcp(double a) {   // 1.0 / a, correctly rounded
#if defined(__CUDA_ARCH__)
  return __drcp_rn(a);
#else
  return 1.0 / a;
#endif
}
CCM_ND_HD float to_f32(double a) {
#if defined(__CUDA_ARCH__)
  return __double2float_rn(a);
#else
  return (float)a;
#endif
}

CCM_ND_HD void centre_of(const float* centre, int32_t k, float O[3]) {
#if defined(__CUDA_ARCH__)
  O[0] = __ldg(centre + 3 * (size_t)k); O[1] = __ldg(centre + 3 * (size_t)k + 1); O[2] = __ldg(centre + 3 * (size_t)k + 2);
#else
  O[0] = centre[3 * (size_t)k]; O[1] = centre[3 * (size_t)k + 1]; O[2] = centre[3 * (size_t)k + 2];
#endif
}

// cv::norm of a CV_32F 3-vector
CCM_ND_HD double norm3(const float d[3]) {
#if defined(__CUDA_ARCH__)
  double s = __dmul_rn((double)d[0], (double)d[0]);
  s = __dadd_rn(s, __dmul_rn((double)d[1], (double)d[1]));
  s = __dadd_rn(s, __dmul_rn((double)d[2], (double)d[2]));
  return __dsqrt_rn(s);
#else
  double s = (double)d[0] * (double)d[0];
  s = s + (double)d[1] * (double)d[1];
  s = s + (double)d[2] * (double)d[2];
  return std::sqrt(s);
#endif
}

// The centre lookup of update_point when every keyframe reads its row of one [K][3] table (ccm_normal_depth).  The Sim3 correction
// (sim3_correction_math.cuh) passes its own lookup instead: there a keyframe's centre depends on the point being corrected.
struct TableCentres {
  const float* centre;
  CCM_ND_HD void operator()(int32_t k, float O[3]) const { centre_of(centre, k, O); }
};

// One point.  X its position; obs_kf[b..e) its observers' keyframe rows in mObservations order; centre_at(k, O) writes GetCameraCenter()
// of keyframe row k as this point sees it; bad [K] the keyframe flags; ref the row of mpRefKF; scale_ref = mvScaleFactors[octave of the
// reference observation], scale_last = mvScaleFactors[nLevels-1].
// Returns 1 and writes the three members, or 0 (no observers or no reference keyframe: the reference returns before writing).
template <typename Centres>
CCM_ND_HD uint8_t update_point(const float X[3], const int32_t* obs_kf, int64_t b, int64_t e, const Centres& centre_at, const uint8_t* bad,
                               int32_t ref, float scale_ref, float scale_last, float normal[3], float* max_dist, float* min_dist) {
  if (b >= e || ref < 0) return 0;
  float nv[3] = {0.f, 0.f, 0.f};
  int n = 0;
  for (int64_t j = b; j < e; j++) {
    const int32_t k = obs_kf[j];
    if (bad[k]) continue;
    float O[3];
    centre_at(k, O);
    const float d[3] = {fsub(X[0], O[0]), fsub(X[1], O[1]), fsub(X[2], O[2])};
    const float a = to_f32(drcp(norm3(d)));
    nv[0] = ffma(d[0], a, nv[0]);
    nv[1] = ffma(d[1], a, nv[1]);
    nv[2] = ffma(d[2], a, nv[2]);
    n++;
  }
  float O[3];
  centre_at(ref, O);
  const float pc[3] = {fsub(X[0], O[0]), fsub(X[1], O[1]), fsub(X[2], O[2])};
  const float dist = to_f32(norm3(pc));
  *max_dist = fmul(dist, scale_ref);
  *min_dist = fdiv(*max_dist, scale_last);
  const float s = to_f32(drcp((double)n));
  normal[0] = fadd(fmul(nv[0], s), 0.f);
  normal[1] = fadd(fmul(nv[1], s), 0.f);
  normal[2] = fadd(fmul(nv[2], s), 0.f);
  return 1;
}

}  // namespace nd
}  // namespace ccm

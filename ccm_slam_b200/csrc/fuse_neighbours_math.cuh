// fuse_neighbours_math.cuh — the per-pair prelude of ORBmatcher::Fuse(kfptr, const vector<mpptr>&, th) (cslam/src/ORBmatcher.cpp:877-922)
// as LocalMapping::SearchInNeighbors runs it (th = 3), and of Fuse(kfptr, Scw, vpPoints, th, vpReplacePoint) (:1010-1069) as
// SearchAndFuse runs it (th = 4, the camera from the caller's split of Scw).  Shared by the kernels (fuse_neighbours.cu,
// search_and_fuse.cu, nvcc) and the host entry points (g++ -ffp-contract=off).  Every product and sum is one explicit rounding, so the device contracts nothing the
// host does not.
//
// The reference evaluates cv::Mat expressions on CV_32F data.  What each one does, and how it is written here:
//   p3Dc = Rcw*p3Dw + tcw          cv::gemm's small-matrix path: f32 products summed left to right, then + t (map_update_math.cuh)
//   invz = 1/z, u = fx*x + cx      f32, left to right.  Fuse(Scw) writes 1.0/z: an f64 quotient rounded to f32, which equals the f32
//                                  quotient (double rounding of a division is innocuous when 53 >= 2*24 + 2)
//   IsInImage                      mnMinX <= u < mnMaxX, mnMinY <= v < mnMaxY
//   1.2f*mfMaxDistance, 0.8f*mfMinDistance   GetMaxDistanceInvariance / GetMinDistanceInvariance, f32
//   dist3D = cv::norm(p3Dw - Ow)   f32 difference, squares summed in double, sqrt, rounded to float (normal_depth_math.cuh)
//   PO.dot(Pn) < 0.5*dist3D        Mat::dot accumulates in double; 0.5*dist3D is a double
//   PredictScale                   ratio = mfMaxDistance/dist3D in f32, then ceil(log(ratio)/mfLogScaleFactor).  MapPoint.h has
//                                  `using namespace std`, so log(float) is std::log(float): glibc's logf, which the device cannot
//                                  reproduce bit for bit.  See level_bracket below.
//   radius = th*mvScaleFactors[l]  f32
#pragma once
#include <stdint.h>

#include <cmath>

#include "new_points_math.cuh"   // the single-rounded f32 / f64 operations and cv::norm of a 3-vector

namespace ccm {
namespace fusenb {

namespace np = ccm::newpts;

constexpr float TH = 3.0f;      // Fuse's default radius factor (cslam/include/cslam/ORBmatcher.h), as SearchInNeighbors calls it
constexpr float TH_SCW = 4.0f;  // the radius factor LoopFinder / MapMerger::SearchAndFuse pass to Fuse(Scw)
constexpr int TH_LOW = 50;   // ORBmatcher::TH_LOW

// one keyframe as the prelude reads it
struct Cam {
  float T[12];                          // [Rcw | tcw], 3x4 row-major
  float O[3];                           // GetCameraCenter(), or Fuse(Scw)'s Ow = -Rcw^T tcw
  float fx, fy, cx, cy;
  float min_x, min_y, max_x, max_y;     // mnMinX, mnMinY, mnMaxX, mnMaxY
  float log_scale;                      // mfLogScaleFactor
  int nlevels;                          // mnScaleLevels
};

// what the prelude decided for one (keyframe, point) pair
enum : int { REJECT = 0, PASS = 1, FLAGGED = 2 };

// nScale from the quotient log(ratio)/mfLogScaleFactor as the reference converts it: ceil, then the implicit float -> int conversion
// (x86's cvttss2si answers INT_MIN for NaN and anything out of int range), then the clamp to [0, mnScaleLevels-1]
CCM_NP_HD int level_of_quotient(float q, int nlevels) {
  const float c = std::ceil(q);
  const int n = (c > -2147483648.f && c < 2147483648.f) ? (int)c : INT32_MIN;
  return n < 0 ? 0 : (n >= nlevels ? nlevels - 1 : n);
}

// The PredictScale rule.  logf(ratio) is within one ulp of the exact logarithm, so it is one of the two floats lo <= hi on either side
// of the f64 log.  When both give the same level, that is the reference's level whatever logf answers; otherwise the pair is FLAGGED
// and the caller settles it with the host's logf (settle_level).  lo == hi when the f64 log is a float.
CCM_NP_HD bool level_bracket(float ratio, float log_scale, int nlevels, int* level) {
  const double L = std::log((double)ratio);
  float lo, hi;
#if defined(__CUDA_ARCH__)
  lo = __double2float_rd(L);
  hi = __double2float_ru(L);
#else
  lo = hi = (float)L;
  if ((double)lo > L) lo = std::nextafter(lo, -INFINITY);
  else if ((double)hi < L) hi = std::nextafter(hi, INFINITY);
#endif
  const int a = level_of_quotient(np::fdiv(lo, log_scale), nlevels), b = level_of_quotient(np::fdiv(hi, log_scale), nlevels);
  *level = a;
  return a == b;
}

// the reference's own arithmetic for a flagged pair; host only
inline int settle_level(float ratio, float log_scale, int nlevels) { return level_of_quotient(logf(ratio) / log_scale, nlevels); }

// The gates of Fuse for point P (world position, normal, mfMaxDistance, mfMinDistance) against keyframe c, radius factor th.  PASS: u, v, radius and
// level are the query of GetFeaturesInArea.  FLAGGED: u, v and ratio are set, the level is the caller's to settle (radius then follows
// from it).  REJECT: a gate failed.
CCM_NP_HD int prelude(const Cam& c, const float* scale_factors, float th, const float P[3], const float N[3], float max_d, float min_d, float& u, float& v,
                      float& radius, int& level, float& ratio) {
  float pc[3];
#pragma unroll
  for (int r = 0; r < 3; r++) {
    float s = np::fmul(c.T[4 * r], P[0]);
    s = np::fadd(s, np::fmul(c.T[4 * r + 1], P[1]));
    s = np::fadd(s, np::fmul(c.T[4 * r + 2], P[2]));
    pc[r] = np::fadd(s, c.T[4 * r + 3]);
  }
  if (pc[2] < 0.0f) return REJECT;                                   // depth must be positive
  const float invz = np::fdiv(1.f, pc[2]);
  u = np::fadd(np::fmul(c.fx, np::fmul(pc[0], invz)), c.cx);
  v = np::fadd(np::fmul(c.fy, np::fmul(pc[1], invz)), c.cy);
  if (!(u >= c.min_x && u < c.max_x && v >= c.min_y && v < c.max_y)) return REJECT;   // IsInImage
  const float maxDistance = np::fmul(1.2f, max_d), minDistance = np::fmul(0.8f, min_d);
  const float PO[3] = {np::fsub(P[0], c.O[0]), np::fsub(P[1], c.O[1]), np::fsub(P[2], c.O[2])};
  const float dist3D = np::to_f32(np::norm3(PO));
  if (dist3D < minDistance || dist3D > maxDistance) return REJECT;   // scale-invariance range
  double dot = np::dmul((double)PO[0], (double)N[0]);
  dot = np::dadd(dot, np::dmul((double)PO[1], (double)N[1]));
  dot = np::dadd(dot, np::dmul((double)PO[2], (double)N[2]));
  if (dot < np::dmul(0.5, (double)dist3D)) return REJECT;            // viewing angle within 60 degrees
  ratio = np::fdiv(max_d, dist3D);
  if (!level_bracket(ratio, c.log_scale, c.nlevels, &level)) return FLAGGED;
  radius = np::fmul(th, scale_factors[level]);
  return PASS;
}

}  // namespace fusenb
}  // namespace ccm

// sim3_correction_math.cuh — arithmetic of the Sim3 correction pass of the loop closure and the map merge, shared by the kernels
// (sim3_correction.cu), the host entry point ccm_sim3_correction_host and a host build in tests/host/ (g++ -ffp-contract=off).
//
//   LoopFinder::CorrectLoop  cslam/src/LoopFinder.cpp:568-613      MapMerger::MergeMaps  cslam/src/MapMerger.cpp:349-395   (one body twice)
//
// Per entry (keyframe pKFi, corrected Sim3 CorrectedSiw, uncorrected Siw), in CorrectedSim3's map order:
//   Swi = CorrectedSiw.inverse()                         G/types/sim3.h:233-236, no normalisation
//   R = rotation().toRotationMatrix(); t *= (1./s)       Eigen's quaternion-to-matrix; one division 1./s, then three products
//   correctedTiw = Converter::toCvSE3(R, t)              each element rounded to f32
//   pKFi->SetPose(correctedTiw)                          Ow = -Rwc*tcw, cv::gemm's f32 left-to-right sum (map_update_math.cuh)
// Per point: Swi.map(Siw.map(P)) in f64 (G/types/sim3.h:144-146: s*(r*x) + t, r*x Eigen's _transformVector), each component to f32
// (Converter::toCvMat).  The f64 operations are those of sim3_math.cuh in the same order, but each one is written as an explicitly
// rounded operation: the library is built with nvcc's default FMA contraction, which would otherwise fuse the products into the sums
// on the device and part the device from the host.  tests/test_sim3_correction.py checks these against sim3_math.cuh on the host.
//
// The reference walks the entries in order and, for each point of an entry, moves it, tags it and calls UpdateNormalAndDepth() at once.
// Two rules follow (DESIGN.md §5):
//   claim    the first entry in map order that lists a point not bad and not yet tagged moves it; later entries skip it;
//   centres  the normal of a point claimed by entry c reads the corrected centre of every keyframe that is an entry before c (its
//            SetPose has run) and the pre-loop centre of every other keyframe, c itself included (its SetPose comes after its points).
#pragma once
#include <stdint.h>

#include "ba_math.cuh"
#include "map_update_math.cuh"
#include "new_points_math.cuh"
#include "normal_depth_math.cuh"
#include "sim3_math.cuh"

#if defined(__CUDACC__)
#define CCM_SC_HD __host__ __device__ __forceinline__
#else
#define CCM_SC_HD inline
#endif

namespace ccm {
namespace sc {

// the explicitly rounded f64 operations of new_points_math.cuh, and the one it lacks
using newpts::dadd;
using newpts::ddiv;
using newpts::dmul;
CCM_SC_HD double dsub(double a, double b) {
#if defined(__CUDA_ARCH__)
  return __dsub_rn(a, b);
#else
  return a - b;
#endif
}

// q * v for a unit-or-not quaternion: v + w*(2 q x v) + q x (2 q x v), as quat_rotate (ba_math.cuh)
CCM_SC_HD void rotate(const S3& q, const double v[3], double o[3]) {
  double ux = dsub(dmul(q.qy, v[2]), dmul(q.qz, v[1]));
  double uy = dsub(dmul(q.qz, v[0]), dmul(q.qx, v[2]));
  double uz = dsub(dmul(q.qx, v[1]), dmul(q.qy, v[0]));
  ux = dadd(ux, ux); uy = dadd(uy, uy); uz = dadd(uz, uz);
  o[0] = dadd(dadd(v[0], dmul(q.qw, ux)), dsub(dmul(q.qy, uz), dmul(q.qz, uy)));
  o[1] = dadd(dadd(v[1], dmul(q.qw, uy)), dsub(dmul(q.qz, ux), dmul(q.qx, uz)));
  o[2] = dadd(dadd(v[2], dmul(q.qw, uz)), dsub(dmul(q.qx, uy), dmul(q.qy, ux)));
}

// Sim3::map: s*(r*x) + t, as s3_map
CCM_SC_HD void map(const S3& S, const double x[3], double o[3]) {
  double r[3];
  rotate(S, x, r);
  o[0] = dadd(dmul(S.s, r[0]), S.tx);
  o[1] = dadd(dmul(S.s, r[1]), S.ty);
  o[2] = dadd(dmul(S.s, r[2]), S.tz);
}

// Sim3::inverse: (conj r, conj r * ((-1./s) t), 1./s), as s3_inv
CCM_SC_HD S3 inverse(const S3& a) {
  S3 r;
  r.qx = -a.qx; r.qy = -a.qy; r.qz = -a.qz; r.qw = a.qw;
  const double k = ddiv(-1., a.s);
  const double kt[3] = {dmul(k, a.tx), dmul(k, a.ty), dmul(k, a.tz)};
  double o[3];
  rotate(r, kt, o);
  r.tx = o[0]; r.ty = o[1]; r.tz = o[2];
  r.s = ddiv(1., a.s);
  return r;
}

// Quaternion::toRotationMatrix, as quat_to_R (row-major)
CCM_SC_HD void rotation_matrix(const S3& q, double R[9]) {
  const double tx = dmul(2., q.qx), ty = dmul(2., q.qy), tz = dmul(2., q.qz);
  const double twx = dmul(tx, q.qw), twy = dmul(ty, q.qw), twz = dmul(tz, q.qw);
  const double txx = dmul(tx, q.qx), txy = dmul(ty, q.qx), txz = dmul(tz, q.qx);
  const double tyy = dmul(ty, q.qy), tyz = dmul(tz, q.qy), tzz = dmul(tz, q.qz);
  R[0] = dsub(1., dadd(tyy, tzz)); R[1] = dsub(txy, twz);          R[2] = dadd(txz, twy);
  R[3] = dadd(txy, twz);          R[4] = dsub(1., dadd(txx, tzz)); R[5] = dsub(tyz, twx);
  R[6] = dsub(txz, twy);          R[7] = dadd(tyz, twx);          R[8] = dsub(1., dadd(txx, tyy));
}

// One entry: the pose SetPose receives (row-major 4x4 f32), the camera centre it leaves, and Swi for the points.
CCM_SC_HD void entry_pose(const S3& corrected_Siw, float Tcw[16], float centre[3], S3* Swi) {
  double R[9];
  rotation_matrix(corrected_Siw, R);
  const double inv_s = ddiv(1., corrected_Siw.s);
  const double t[3] = {dmul(corrected_Siw.tx, inv_s), dmul(corrected_Siw.ty, inv_s), dmul(corrected_Siw.tz, inv_s)};
  for (int r = 0; r < 3; r++) {
    for (int c = 0; c < 3; c++) Tcw[4 * r + c] = nd::to_f32(R[3 * r + c]);
    Tcw[4 * r + 3] = nd::to_f32(t[r]);
  }
  Tcw[12] = 0.f; Tcw[13] = 0.f; Tcw[14] = 0.f; Tcw[15] = 1.f;
  float Twc[16];
  mu::pose_inverse(Tcw, Twc);
  centre[0] = Twc[3]; centre[1] = Twc[7]; centre[2] = Twc[11];
  *Swi = inverse(corrected_Siw);
}

// One point: project with the uncorrected pose, back with the corrected one
CCM_SC_HD void move_point(const S3& Siw, const S3& Swi, const float X[3], float out[3]) {
  const double x[3] = {(double)X[0], (double)X[1], (double)X[2]};
  double c[3], w[3];
  map(Siw, x, c);
  map(Swi, c, w);
  out[0] = nd::to_f32(w[0]); out[1] = nd::to_f32(w[1]); out[2] = nd::to_f32(w[2]);
}

// The centre rule for a point claimed by entry `claim`: a keyframe that is an entry before it reads its corrected centre, every other
// keyframe its pre-loop centre.  kf_entry [n_kf]: the entry of each keyframe row, -1 for one outside the list.
struct ClaimCentres {
  const float* old_centre;   // [n_kf][3]
  const float* new_centre;   // [n_e][3]
  const int32_t* kf_entry;   // [n_kf]
  int32_t claim;
  CCM_SC_HD void operator()(int32_t k, float O[3]) const {
    const int32_t e = kf_entry[k];
    if (e >= 0 && e < claim) nd::centre_of(new_centre, e, O);
    else nd::centre_of(old_centre, k, O);
  }
};

}  // namespace sc
}  // namespace ccm

// sim3_correction_oracle.cpp — TEST INFRASTRUCTURE: the checker's flat restatement of the Sim3 correction pass of
// LoopFinder::CorrectLoop (cslam/src/LoopFinder.cpp:568-613) and MapMerger::MergeMaps (cslam/src/MapMerger.cpp:349-395) over the arrays
// of ccm_sim3_correction (include/ccm_b200.h).  Written from the reference loop, not from the product's sim3_correction_math.cuh:
// it walks the entries in order exactly as the reference does, keeps a live table of camera centres, moves and tags each point the
// moment an entry reaches it, runs UpdateNormalAndDepth on it against the centres as they stand at that moment (orc_normal_depth of
// normal_depth_oracle.cpp, one point at a time), and overwrites the entry's centre only after its points.  Which entry claims a
// point and which centres its normal sees are therefore outcomes of the walk, not assumptions.
//   g2o::Sim3::map       s*(r*x) + t, r*x = Eigen's _transformVector: uv = 2 (q.vec x v); v + w uv + q.vec x uv
//   g2o::Sim3::inverse   (r.conjugate(), r.conjugate() * ((-1./s) * t), 1./s)
//   toRotationMatrix     Eigen's Quaternion::toRotationMatrix
//   eigt *= (1./s); toCvSE3; SetPose: Ow = -Rcw^T tcw summed left to right in f32
// Compiled by oracle/Makefile with -ffp-contract=off.
#include <cstdint>
#include <vector>

extern "C" int orc_normal_depth(int32_t n_kf, const float* kf_centre, const uint8_t* kf_bad, int32_t n_mp, const float* mp_pos,
                                const int64_t* obs_ptr, const int32_t* obs_kf, const int32_t* mp_ref, const float* mp_scale_ref,
                                const float* mp_scale_last, float* normal, float* max_dist, float* min_dist, uint8_t* status);

namespace {

struct Sim3 {
  double x, y, z, w;   // quaternion
  double t[3];
  double s;
};

Sim3 load(const double* p) { return Sim3{p[0], p[1], p[2], p[3], {p[4], p[5], p[6]}, p[7]}; }

void cross(const double a[3], const double b[3], double c[3]) {
  c[0] = a[1] * b[2] - a[2] * b[1];
  c[1] = a[2] * b[0] - a[0] * b[2];
  c[2] = a[0] * b[1] - a[1] * b[0];
}

void transform_vector(const Sim3& S, const double v[3], double o[3]) {
  const double q[3] = {S.x, S.y, S.z};
  double uv[3], c[3];
  cross(q, v, uv);
  for (int i = 0; i < 3; i++) uv[i] += uv[i];
  cross(q, uv, c);
  for (int i = 0; i < 3; i++) o[i] = v[i] + S.w * uv[i] + c[i];
}

void sim3_map(const Sim3& S, const double x[3], double o[3]) {
  double r[3];
  transform_vector(S, x, r);
  for (int i = 0; i < 3; i++) o[i] = S.s * r[i] + S.t[i];
}

Sim3 sim3_inverse(const Sim3& S) {
  Sim3 c{-S.x, -S.y, -S.z, S.w, {0, 0, 0}, 1. / S.s};
  const double k = -1. / S.s;
  const double kt[3] = {k * S.t[0], k * S.t[1], k * S.t[2]};
  transform_vector(c, kt, c.t);
  return c;
}

void to_rotation_matrix(const Sim3& q, double R[3][3]) {
  const double tx = 2 * q.x, ty = 2 * q.y, tz = 2 * q.z;
  const double twx = tx * q.w, twy = ty * q.w, twz = tz * q.w;
  const double txx = tx * q.x, txy = ty * q.x, txz = tz * q.x;
  const double tyy = ty * q.y, tyz = tz * q.y, tzz = tz * q.z;
  R[0][0] = 1 - (tyy + tzz); R[0][1] = txy - twz;       R[0][2] = txz + twy;
  R[1][0] = txy + twz;       R[1][1] = 1 - (txx + tzz); R[1][2] = tyz - twx;
  R[2][0] = txz - twy;       R[2][1] = tyz + twx;       R[2][2] = 1 - (txx + tyy);
}

}  // namespace

// Returns 0, or -1 on input the reference could not have produced (a row out of range, a keyframe listed twice).
extern "C" int orc_sim3_correction(int32_t n_kf, const float* kf_centre, const uint8_t* kf_bad, int32_t n_e, const int32_t* entry_kf,
                                   const double* entry_Siw_new, const double* entry_Siw_old, const int64_t* slot_ptr, const int32_t* slot_mp,
                                   int32_t n_mp, const float* mp_pos, const uint8_t* mp_skip, const int64_t* obs_ptr, const int32_t* obs_kf,
                                   const int32_t* mp_ref, const float* mp_scale_ref, const float* mp_scale_last, float* entry_Tcw,
                                   float* entry_centre, int32_t* mp_entry, float* mp_pos_out, float* normal, float* max_dist,
                                   float* min_dist, uint8_t* status) {
  if (n_kf < 0 || n_e < 0 || n_mp < 0) return -1;
  std::vector<uint8_t> listed((size_t)n_kf, 0);
  for (int32_t e = 0; e < n_e; e++) {
    if (entry_kf[e] < 0 || entry_kf[e] >= n_kf || listed[entry_kf[e]]) return -1;
    listed[entry_kf[e]] = 1;
  }
  std::vector<float> centre(kf_centre, kf_centre + 3 * (size_t)n_kf);     // GetCameraCenter() of every keyframe, live
  std::vector<uint8_t> tagged(mp_skip, mp_skip + n_mp);                     // isBad() or mCorrectedByKF == mId, live
  for (int32_t i = 0; i < n_mp; i++) {
    mp_entry[i] = -1;
    for (int c = 0; c < 3; c++) { mp_pos_out[3 * (size_t)i + c] = mp_pos[3 * (size_t)i + c]; normal[3 * (size_t)i + c] = 0.f; }
    max_dist[i] = min_dist[i] = 0.f; status[i] = 0;
  }
  for (int32_t e = 0; e < n_e; e++) {                                        // for(mit = CorrectedSim3.begin(); ...)
    const Sim3 CorrectedSiw = load(entry_Siw_new + 8 * (size_t)e);
    const Sim3 CorrectedSwi = sim3_inverse(CorrectedSiw);
    const Sim3 Siw = load(entry_Siw_old + 8 * (size_t)e);
    for (int64_t j = slot_ptr[e]; j < slot_ptr[e + 1]; j++) {                // vpMPsi = pKFi->GetMapPointMatches()
      const int32_t p = slot_mp[j];
      if (p < -1 || p >= n_mp) return -1;
      if (p < 0) continue;                                                   // if(!pMPi) continue;
      if (tagged[p]) continue;                                               // isBad() || mCorrectedByKF == mId
      const double P3Dw[3] = {(double)mp_pos[3 * (size_t)p], (double)mp_pos[3 * (size_t)p + 1], (double)mp_pos[3 * (size_t)p + 2]};
      double c[3], w[3];
      sim3_map(Siw, P3Dw, c);
      sim3_map(CorrectedSwi, c, w);
      float* X = mp_pos_out + 3 * (size_t)p;
      X[0] = (float)w[0]; X[1] = (float)w[1]; X[2] = (float)w[2];             // SetWorldPos(toCvMat(...))
      tagged[p] = 1;
      mp_entry[p] = e;
      const int64_t local_ptr[2] = {0, obs_ptr[p + 1] - obs_ptr[p]};          // UpdateNormalAndDepth() against the centres as they stand
      if (orc_normal_depth(n_kf, centre.data(), kf_bad, 1, X, local_ptr, obs_kf + obs_ptr[p], mp_ref + p, mp_scale_ref + p, mp_scale_last + p,
                           normal + 3 * (size_t)p, max_dist + p, min_dist + p, status + p) != 0)
        return -1;
    }
    double R[3][3];
    to_rotation_matrix(CorrectedSiw, R);
    double t[3] = {CorrectedSiw.t[0], CorrectedSiw.t[1], CorrectedSiw.t[2]};
    const double inv = 1. / CorrectedSiw.s;
    for (int i = 0; i < 3; i++) t[i] *= inv;                                  // eigt *= (1./s)
    float* T = entry_Tcw + 16 * (size_t)e;                                    // Converter::toCvSE3
    for (int r = 0; r < 4; r++)
      for (int k = 0; k < 4; k++) T[4 * r + k] = r == 3 ? (k == 3 ? 1.f : 0.f) : (k == 3 ? (float)t[r] : (float)R[r][k]);
    float Ow[3];                                                              // SetPose: Ow = -Rwc * tcw
    for (int r = 0; r < 3; r++) {
      float s = T[r] * T[3];
      s = s + T[4 + r] * T[7];
      s = s + T[8 + r] * T[11];
      Ow[r] = -s;
    }
    const int32_t k = entry_kf[e];
    for (int c = 0; c < 3; c++) { centre[3 * (size_t)k + c] = Ow[c]; entry_centre[3 * (size_t)e + c] = Ow[c]; }
  }
  return 0;
}

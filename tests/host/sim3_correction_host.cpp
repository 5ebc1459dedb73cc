// sim3_correction_host.cpp — TEST CODE: the arithmetic of ccm_sim3_correction (ccm_slam_b200/csrc/sim3_correction_math.cuh) run on
// the host: the bodies of k_sc_entries, k_sc_claim (the atomicMin as a plain minimum) and k_sc_points with their grid-stride loops
// turned into plain loops, the slots visited in reverse so that the claim cannot lean on the walk order.  Also exposes the explicitly
// rounded Sim3 operations next to sim3_math.cuh's, for a bitwise comparison.  Compiled by tests/test_sim3_correction.py with g++.
//
// -DMUT=n builds one deliberately wrong variant, which the tests require the oracle to tell apart:
//   1 the claim taken by the last entry        2 the claim by keyframe row instead of map order
//   3 every centre the pre-loop one (the plain table)   4 every entry's centre corrected   5 the claiming entry counted as corrected
//   6 t/s as a division                        7 the point map in f32        8 the quaternions normalised
#ifndef MUT
#define MUT 0
#endif
#include <climits>
#include <cmath>
#include <cstdint>
#include <vector>

#include "../../ccm_slam_b200/csrc/sim3_correction_math.cuh"

using namespace ccm;

extern "C" int sc_host_correct(int32_t n_kf, const float* kf_centre, const uint8_t* kf_bad, int32_t n_e, const int32_t* entry_kf,
                               const double* entry_Siw_new, const double* entry_Siw_old, const int64_t* slot_ptr, const int32_t* slot_mp,
                               int32_t n_mp, const float* mp_pos, const uint8_t* mp_skip, const int64_t* obs_ptr, const int32_t* obs_kf,
                               const int32_t* mp_ref, const float* mp_scale_ref, const float* mp_scale_last, float* entry_Tcw,
                               float* entry_centre, int32_t* mp_entry, float* mp_pos_out, float* normal, float* max_dist, float* min_dist,
                               uint8_t* status) {
  std::vector<int32_t> kf_entry((size_t)n_kf, -1);
  for (int32_t e = 0; e < n_e; e++) kf_entry[entry_kf[e]] = e;
  std::vector<double> swi(8 * (size_t)n_e);
  std::vector<double> siw_new(entry_Siw_new, entry_Siw_new + 8 * (size_t)n_e), siw_old(entry_Siw_old, entry_Siw_old + 8 * (size_t)n_e);
#if MUT == 8
  for (double* q : {siw_new.data(), siw_old.data()})
    for (int32_t e = 0; e < n_e; e++) {
      double* a = q + 8 * (size_t)e;
      const double n = std::sqrt(a[0] * a[0] + a[1] * a[1] + a[2] * a[2] + a[3] * a[3]);
      for (int c = 0; c < 4; c++) a[c] /= n;
    }
#endif
  entry_Siw_new = siw_new.data(); entry_Siw_old = siw_old.data();
  for (int32_t e = 0; e < n_e; e++) {                                   // k_sc_entries
    S3 w;
    sc::entry_pose(s3_load(entry_Siw_new + 8 * (size_t)e), entry_Tcw + 16 * (size_t)e, entry_centre + 3 * (size_t)e, &w);
    s3_store(w, swi.data() + 8 * (size_t)e);
#if MUT == 6
    const double* a = entry_Siw_new + 8 * (size_t)e;
    float* T = entry_Tcw + 16 * (size_t)e;
    for (int r = 0; r < 3; r++) T[4 * r + 3] = (float)(a[4 + r] / a[7]);
    float Twc[16];
    mu::pose_inverse(T, Twc);
    entry_centre[3 * (size_t)e] = Twc[3]; entry_centre[3 * (size_t)e + 1] = Twc[7]; entry_centre[3 * (size_t)e + 2] = Twc[11];
#endif
  }
  for (int32_t i = 0; i < n_mp; i++) mp_entry[i] = INT_MAX;
  const int64_t S = n_e ? slot_ptr[n_e] : 0;
  for (int64_t j = S - 1; j >= 0; j--) {                                // k_sc_claim
    const int32_t p = slot_mp[j];
    if (p < 0 || mp_skip[p]) continue;
    int32_t lo = 0, hi = n_e;
    while (hi - lo > 1) {
      const int32_t mid = (lo + hi) >> 1;
      if (slot_ptr[mid] <= j) lo = mid; else hi = mid;
    }
#if MUT == 1
    if (mp_entry[p] == INT_MAX || lo > mp_entry[p]) mp_entry[p] = lo;
#elif MUT == 2
    if (mp_entry[p] == INT_MAX || entry_kf[lo] < entry_kf[mp_entry[p]]) mp_entry[p] = lo;
#else
    if (lo < mp_entry[p]) mp_entry[p] = lo;
#endif
  }
  for (int32_t i = 0; i < n_mp; i++) {                                  // k_sc_points
    const int32_t c = mp_entry[i];
    float X[3] = {mp_pos[3 * (size_t)i], mp_pos[3 * (size_t)i + 1], mp_pos[3 * (size_t)i + 2]};
    float nv[3] = {0.f, 0.f, 0.f}, dmax = 0.f, dmin = 0.f;
    uint8_t st = 0;
    if (c != INT_MAX) {
      const float P[3] = {X[0], X[1], X[2]};
#if MUT == 7
      const S3 A = s3_load(entry_Siw_old + 8 * (size_t)c), B = s3_load(swi.data() + 8 * (size_t)c);
      float y[3];
      for (const S3* S : {&A, &B}) {
        const float q[3] = {(float)S->qx, (float)S->qy, (float)S->qz}, w = (float)S->qw;
        float u[3] = {q[1] * X[2] - q[2] * X[1], q[2] * X[0] - q[0] * X[2], q[0] * X[1] - q[1] * X[0]};
        for (float& v : u) v += v;
        const float c2[3] = {q[1] * u[2] - q[2] * u[1], q[2] * u[0] - q[0] * u[2], q[0] * u[1] - q[1] * u[0]};
        const float t[3] = {(float)S->tx, (float)S->ty, (float)S->tz};
        for (int k = 0; k < 3; k++) y[k] = (float)S->s * (X[k] + w * u[k] + c2[k]) + t[k];
        for (int k = 0; k < 3; k++) X[k] = y[k];
      }
      (void)P;
#else
      sc::move_point(s3_load(entry_Siw_old + 8 * (size_t)c), s3_load(swi.data() + 8 * (size_t)c), P, X);
#endif
#if MUT == 3
      const nd::TableCentres at{kf_centre};
#elif MUT == 4
      const sc::ClaimCentres at{kf_centre, entry_centre, kf_entry.data(), INT_MAX};
#elif MUT == 5
      const sc::ClaimCentres at{kf_centre, entry_centre, kf_entry.data(), c + 1};
#else
      const sc::ClaimCentres at{kf_centre, entry_centre, kf_entry.data(), c};
#endif
      st = nd::update_point(X, obs_kf, obs_ptr[i], obs_ptr[i + 1], at, kf_bad, mp_ref[i], mp_scale_ref[i], mp_scale_last[i], nv, &dmax, &dmin);
      if (!st) { nv[0] = nv[1] = nv[2] = 0.f; dmax = dmin = 0.f; }
    }
    mp_entry[i] = c == INT_MAX ? -1 : c;
    for (int k = 0; k < 3; k++) { mp_pos_out[3 * (size_t)i + k] = X[k]; normal[3 * (size_t)i + k] = nv[k]; }
    max_dist[i] = dmax; min_dist[i] = dmin; status[i] = st;
  }
  return 0;
}

// the explicitly rounded operations against sim3_math.cuh / ba_math.cuh on n Sim3s (8 doubles each) and n points (3 doubles each):
// out[n][4][8] = inverse (ours, theirs), map (ours, theirs) padded; R[n][2][9] = rotation matrix (ours, theirs)
extern "C" void sc_host_ops(int32_t n, const double* S, const double* x, double* out, double* R) {
  for (int32_t i = 0; i < n; i++) {
    const S3 a = s3_load(S + 8 * (size_t)i);
    double* o = out + 32 * (size_t)i;
    s3_store(sc::inverse(a), o);
    s3_store(s3_inv(a), o + 8);
    const double* v = x + 3 * (size_t)i;
    sc::map(a, v, o + 16);
    s3_map(a, v[0], v[1], v[2], o[24], o[25], o[26]);
    sc::rotation_matrix(a, R + 18 * (size_t)i);
    quat_to_R(a.qx, a.qy, a.qz, a.qw, R + 18 * (size_t)i + 9);
  }
}

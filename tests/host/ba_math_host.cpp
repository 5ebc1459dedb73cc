// Host build of the product's csrc/ba_math.cuh for tests/test_ba_math_host.py: the per-observation linearisation, the Huber weight
// and the pose update exp(x) * T that the BA kernels run, exported with a C ABI.  Compiled with g++ -ffp-contract=off.
#include "../../ccm_slam_b200/csrc/ba_math.cuh"

namespace {
ccm::Pose pose_of(const double* p) { return ccm::Pose{p[0], p[1], p[2], p[3], p[4], p[5], p[6]}; }
}  // namespace

extern "C" {

// out: ex ey chi2 Xc[3] Jl[6] Jp[12]  (24 doubles)
void bm_linearize(const double* T, const double* intr, const double* X, const double* uv, double w, double* out) {
  ccm::ObsLin L;
  ccm::linearize_obs(pose_of(T), intr, X[0], X[1], X[2], uv[0], uv[1], w, L);
  out[0] = L.ex; out[1] = L.ey; out[2] = L.chi2;
  for (int i = 0; i < 3; i++) out[3 + i] = L.Xc[i];
  for (int i = 0; i < 6; i++) out[6 + i] = L.Jl[i];
  for (int i = 0; i < 12; i++) out[12 + i] = L.Jp[i];
}

void bm_huber(double e, double delta, double* out) { ccm::huber(e, delta, out[0], out[1]); }

void bm_exp_times(const double* upd, const double* T, double* out) {
  const ccm::Pose o = ccm::se3_exp_times(upd, pose_of(T));
  out[0] = o.qx; out[1] = o.qy; out[2] = o.qz; out[3] = o.qw; out[4] = o.tx; out[5] = o.ty; out[6] = o.tz;
}

}  // extern "C"

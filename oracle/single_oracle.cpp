// single_oracle.cpp — CPU oracle for the two single-vertex optimisations of cslam::Optimizer (TEST INFRASTRUCTURE, NOT PRODUCT).
//
//   orc_pose_optimize : Optimizer::PoseOptimizationClient (S/Optimizer.cpp:215-347): one VertexSE3Expmap, N unary
//                       EdgeSE3ProjectXYZOnlyPose (G/types/types_six_dof_expmap.h:143-171, .cpp:266-296, analytic Jacobian),
//                       Huber sqrt(5.991), 4 rounds of {reset estimate, initializeOptimization(0), optimize(10), classify}.
//   orc_sim3_optimize : Optimizer::OptimizeSim3 (S/Optimizer.cpp:861-1056): one VertexSim3Expmap (fix_scale zeroes update[6],
//                       G/types/types_seven_dof_expmap.h:60-69), per correspondence an EdgeSim3ProjectXYZ and an
//                       EdgeInverseSim3ProjectXYZ against FIXED points (.h:130-172), NUMERIC Jacobians, central differences
//                       delta = 1e-9 (G/core/base_binary_edge.hpp:131-205), Huber sqrt(th2), optimize(5), drop pairs with
//                       chi2 > th2, optimize(5 or 10).
//
// Both run g2o's Levenberg loop (G/core/optimization_algorithm_levenberg.cpp:61-189) on a dense D x D system
// (LinearSolverDense = Eigen LDLT with isPositive check, G/solvers/linear_solver_dense.h:99-106; restated as an unpivoted
// Cholesky that fails on a non-positive pivot).  Edge errors are cached the way g2o caches them: classification after
// optimize() reads the error of the LAST evaluated state (a rejected trial leaves stale errors), except where the reference
// calls computeError() explicitly (S/Optimizer.cpp:310-313).
#include <cmath>
#include <cstring>
#include <limits>
#include <vector>

#include "lie.hpp"
#include "oracle.h"

namespace {
using namespace orc;

// LM trace of one optimize() call: {end, iterations, iteration limit, cached chi2, fresh chi2, stale edges, rejected} +
// TRACE_ITERS rows of TRACE_COLS
// (the layout of the device's trace, include/ccm_b200.h)
constexpr int TRACE_ITERS = 10, TRACE_COLS = 7, TRACE_HEAD = 7, TRACE_CALL = TRACE_HEAD + TRACE_ITERS * TRACE_COLS;

inline void huber1(double e, double delta, double rho[3]) {  // G/core/robust_kernel_impl.cpp:77-91
  const double dsqr = (double)(float)(delta * delta);  // float member, G/core/robust_kernel_impl.h:84
  if (e <= dsqr) {
    rho[0] = e; rho[1] = 1.; rho[2] = 0.;
  } else {
    const double sqrte = std::sqrt(e);
    rho[0] = 2 * sqrte * delta - dsqr;
    rho[1] = delta / sqrte;
    rho[2] = -0.5 * rho[1] / e;
  }
}

// dense SPD solve, row-major n x n (n <= 7); false when a pivot is not positive
template <int N>
bool chol_solve(const double* A, const double* b, double* x) {
  double L[N * N];
  for (int i = 0; i < N; i++)
    for (int j = 0; j <= i; j++) {
      double s = A[i * N + j];
      for (int k = 0; k < j; k++) s -= L[i * N + k] * L[j * N + k];
      if (i == j) {
        if (!(s > 0.0) || !std::isfinite(s)) return false;
        L[i * N + i] = std::sqrt(s);
      } else {
        L[i * N + j] = s / L[j * N + j];
      }
    }
  double y[N];
  for (int i = 0; i < N; i++) {
    double s = b[i];
    for (int k = 0; k < i; k++) s -= L[i * N + k] * y[k];
    y[i] = s / L[i * N + i];
  }
  for (int i = N - 1; i >= 0; i--) {
    double s = y[i];
    for (int k = i + 1; k < N; k++) s -= L[k * N + i] * x[k];
    x[i] = s / L[i * N + i];
  }
  return true;
}

// ---- the two models: state, error of edge e, Jacobian of edge e, oplus --------------------------------------------------
struct PoseModel {
  static constexpr int D = 6;
  static constexpr bool unary = true;   // EdgeSE3ProjectXYZOnlyPose is a BaseUnaryEdge
  typedef SE3 State;
  const orc_pose_opt_problem* p;
  int n_edges() const { return p->n; }
  double weight(int e) const { return (double)p->inv_sigma2[e]; }
  void error(const State& T, int e, double err[2]) const {  // types_six_dof_expmap.h:153-157
    const double X[3] = {(double)p->Xw[3 * e], (double)p->Xw[3 * e + 1], (double)p->Xw[3 * e + 2]};
    double xc[3];
    se3_map(T, X, xc);
    const double u = xc[0] / xc[2] * (double)p->fx + (double)p->cx, v = xc[1] / xc[2] * (double)p->fy + (double)p->cy;
    err[0] = (double)p->uv[2 * e] - u;
    err[1] = (double)p->uv[2 * e + 1] - v;
  }
  void jacobian(State& T, int e, const double* /*err*/, double J[2 * 6]) const {  // types_six_dof_expmap.cpp:266-288
    const double X[3] = {(double)p->Xw[3 * e], (double)p->Xw[3 * e + 1], (double)p->Xw[3 * e + 2]};
    double xc[3];
    se3_map(T, X, xc);
    const double x = xc[0], y = xc[1], invz = 1.0 / xc[2], invz_2 = invz * invz, fx = p->fx, fy = p->fy;
    J[0] = x * y * invz_2 * fx; J[1] = -(1 + (x * x * invz_2)) * fx; J[2] = y * invz * fx;
    J[3] = -invz * fx; J[4] = 0; J[5] = x * invz_2 * fx;
    J[6] = (1 + y * y * invz_2) * fy; J[7] = -x * y * invz_2 * fy; J[8] = -x * invz * fy;
    J[9] = 0; J[10] = -invz * fy; J[11] = y * invz_2 * fy;
  }
  static void oplus(State& T, const double* x) { T = se3_mul(se3_exp(x), T); }  // VertexSE3Expmap::oplusImpl
};

struct Sim3Model {
  static constexpr int D = 7;
  static constexpr bool unary = false;  // EdgeSim3ProjectXYZ / EdgeInverseSim3ProjectXYZ are binary edges with a fixed point vertex
  typedef Sim3 State;
  const orc_sim3_opt_problem* p;
  // edge 2i = EdgeSim3ProjectXYZ of pair i (x1 = S12 * X2c into camera 1), edge 2i+1 = EdgeInverseSim3ProjectXYZ (x2 = S12^-1 * X1c)
  int n_edges() const { return 2 * p->n; }
  double weight(int e) const { return (double)((e & 1) ? p->inv_sigma2_2[e >> 1] : p->inv_sigma2_1[e >> 1]); }
  void error(const State& S, int e, double err[2]) const {  // types_seven_dof_expmap.h:138-146,160-168
    const int i = e >> 1;
    double q[3];
    if (!(e & 1)) {
      const double X[3] = {(double)p->P2c[3 * i], (double)p->P2c[3 * i + 1], (double)p->P2c[3 * i + 2]};
      sim3_map(S, X, q);
      err[0] = (double)p->uv1[2 * i] - (q[0] / q[2] * (double)p->K1[0] + (double)p->K1[2]);
      err[1] = (double)p->uv1[2 * i + 1] - (q[1] / q[2] * (double)p->K1[1] + (double)p->K1[3]);
    } else {
      const double X[3] = {(double)p->P1c[3 * i], (double)p->P1c[3 * i + 1], (double)p->P1c[3 * i + 2]};
      sim3_map(sim3_inv(S), X, q);
      err[0] = (double)p->uv2[2 * i] - (q[0] / q[2] * (double)p->K2[0] + (double)p->K2[2]);
      err[1] = (double)p->uv2[2 * i + 1] - (q[1] / q[2] * (double)p->K2[1] + (double)p->K2[3]);
    }
  }
  void jacobian(State& S, int e, const double* /*err*/, double J[2 * 7]) const {  // base_binary_edge.hpp:131-205 (vertex 1 only)
    const double delta = 1e-9, scalar = 1.0 / (2 * delta);
    double add[7] = {0, 0, 0, 0, 0, 0, 0};
    for (int d = 0; d < 7; d++) {
      double ep[2], em[2];
      State bak = S;
      add[d] = delta;
      oplus_fs(S, add);
      error(S, e, ep);
      S = bak;
      add[d] = -delta;
      oplus_fs(S, add);
      error(S, e, em);
      S = bak;
      add[d] = 0.0;
      J[d] = scalar * (ep[0] - em[0]);
      J[7 + d] = scalar * (ep[1] - em[1]);
    }
  }
  void oplus_fs(State& S, const double* x) const {  // VertexSim3Expmap::oplusImpl
    double u[7];
    std::memcpy(u, x, sizeof(u));
    if (p->fix_scale) u[6] = 0;
    S = sim3_mul(sim3_exp(u), S);
  }
};

// ---- g2o Levenberg on one vertex ------------------------------------------------------------------------------------------
template <class M>
struct Single {
  static constexpr int D = M::D;
  M m;
  typename M::State est;
  std::vector<uint8_t> active, robust;  // per edge: level 0 ; has a Huber kernel
  std::vector<double> err;              // cached _error of every edge (2 per edge)
  double delta = 0;
  double* trace = nullptr;              // optional: the current call's trace slot (layout of ccm_single trace in ccm_b200.h)

  void oplus(const double* x) {
    if constexpr (D == 7) m.oplus_fs(est, x); else M::oplus(est, x);
  }
  double chi2_of(int e) const { const double w = m.weight(e); return err[2 * e] * (w * err[2 * e]) + err[2 * e + 1] * (w * err[2 * e + 1]); }
  void compute_active_errors() {
    for (int e = 0; e < m.n_edges(); e++) if (active[e]) m.error(est, e, &err[2 * e]);
  }
  double active_robust_chi2() const {
    double chi = 0;
    for (int e = 0; e < m.n_edges(); e++) {
      if (!active[e]) continue;
      if (robust[e]) { double rho[3]; huber1(chi2_of(e), delta, rho); chi += rho[0]; } else chi += chi2_of(e);
    }
    return chi;
  }
  void build(double* H, double* b) {  // BaseUnaryEdge / BaseBinaryEdge::constructQuadraticForm on the free vertex
    std::fill(H, H + D * D, 0.0); std::fill(b, b + D, 0.0);
    for (int e = 0; e < m.n_edges(); e++) {
      if (!active[e]) continue;
      double J[2 * D];
      m.jacobian(est, e, &err[2 * e], J);
      const double w = m.weight(e);
      double wo = w, wr = 1.0;
      if (robust[e]) { double rho[3]; huber1(chi2_of(e), delta, rho); wo = rho[1] * w; wr = rho[1]; }
      const double r0 = -(w * err[2 * e]) * wr, r1 = -(w * err[2 * e + 1]) * wr;  // omega_r = -Omega e, times rho[1] when robust
      for (int i = 0; i < D; i++) {
        if constexpr (M::unary) {
          // BaseUnaryEdge::constructQuadraticForm (base_unary_edge.hpp:63-70): b -= rho[1] * A^T * Omega * e, grouped left to right
          const double a0 = robust[e] ? wr * J[i] : J[i], a1 = robust[e] ? wr * J[D + i] : J[D + i];
          b[i] -= (a0 * w) * err[2 * e] + (a1 * w) * err[2 * e + 1];
        } else {
          b[i] += J[i] * r0 + J[D + i] * r1;        // BaseBinaryEdge: b += B^T * omega_r (base_binary_edge.hpp:74-76,86-104)
        }
        for (int j = 0; j < D; j++) H[i * D + j] += J[i] * wo * J[j] + J[D + i] * wo * J[D + j];
      }
    }
  }
  // SparseOptimizer::optimize + OptimizationAlgorithmLevenberg::solve; returns the number of LM iterations (-1: no active edge)
  int optimize(int iterations) {
    bool any = false;
    for (int e = 0; e < m.n_edges(); e++) any = any || active[e];
    if (!any) { if (trace) { trace[0] = -1; trace[1] = -1; trace[2] = iterations; } return -1; }
    double lambda = -1, ni = 2;
    int n_bad = 0, done = 0, end = 0;
    bool ok = true;
    for (int it = 0; it < iterations && ok; it++) {
      compute_active_errors();
      double currentChi = active_robust_chi2();
      const double iniChi = currentChi;
      double tempChi = currentChi;
      double H[D * D], b[D], x[D];
      build(H, b);
      if (it == 0) {
        double maxd = 0;
        for (int i = 0; i < D; i++) maxd = std::max(std::fabs(H[i * D + i]), maxd);
        lambda = 1e-5 * maxd; ni = 2; n_bad = 0;
      }
      const double lambda0 = lambda;
      int nfail = 0;
      double rho = 0;
      int qmax = 0;
      do {
        const typename M::State bak = est;  // push
        double Hd[D * D];
        std::memcpy(Hd, H, sizeof(Hd));
        for (int i = 0; i < D; i++) Hd[i * D + i] += lambda;
        const bool ok2 = chol_solve<D>(Hd, b, x);
        if (!ok2) std::fill(x, x + D, 0.0);
        oplus(x);
        compute_active_errors();
        tempChi = active_robust_chi2();
        if (!ok2) { tempChi = std::numeric_limits<double>::max(); nfail++; }
        rho = currentChi - tempChi;
        double scale = 0;
        for (int i = 0; i < D; i++) scale += x[i] * (lambda * x[i] + b[i]);
        scale += 1e-3;
        rho /= scale;
        if (rho > 0 && std::isfinite(tempChi)) {
          double alpha = 1. - std::pow((2 * rho - 1), 3);
          alpha = std::min(alpha, 2. / 3.);
          lambda *= std::max(1. / 3., alpha);
          ni = 2;
          currentChi = tempChi;
        } else {
          lambda *= ni; ni *= 2;
          est = bak;  // pop (the cached errors stay those of the rejected state)
        }
        qmax++;
      } while (rho < 0 && qmax < 10);
      if (trace && it < TRACE_ITERS) {
        double* r = trace + TRACE_HEAD + it * TRACE_COLS;
        r[0] = iniChi; r[1] = lambda0; r[2] = qmax; r[3] = rho; r[4] = currentChi; r[5] = (rho > 0 && std::isfinite(tempChi)) ? 1 : 0;
        r[6] = nfail;
      }
      done++;
      if (qmax == 10 || rho == 0) { ok = false; end = qmax == 10 ? 1 : 2; continue; }
      if ((iniChi - currentChi) * 1e3 < iniChi) n_bad++; else n_bad = 0;
      if (n_bad >= 3) { ok = false; end = 3; continue; }
    }
    if (trace) { trace[0] = end; trace[1] = done; trace[2] = iterations; }
    return done;
  }
  // trace only, over the edges with use(e): chi2 of the cached errors the classification read and of fresh errors at est, the
  // number of edges whose cached error is not bit-identical to the fresh one, and the classification's rejections
  template <class Use>
  void trace_chi2(Use use, int rejected) const {
    if (!trace) return;
    double cached = 0, fresh = 0, stale = 0;
    for (int e = 0; e < m.n_edges(); e++) {
      if (!use(e)) continue;
      double f[2];
      m.error(est, e, f);
      const double w = m.weight(e);
      cached += chi2_of(e);
      fresh += f[0] * (w * f[0]) + f[1] * (w * f[1]);
      stale += (err[2 * e] != f[0] || err[2 * e + 1] != f[1]) ? 1 : 0;
    }
    trace[3] = cached; trace[4] = fresh; trace[5] = stale; trace[6] = rejected;
  }
};


int pose_optimize(const orc_pose_opt_problem* p, double* Tcw_out, uint8_t* outlier, double* trace) {
  Single<PoseModel> s;
  s.m.p = p;
  const int N = p->n;
  if (N < 3) { std::memcpy(Tcw_out, p->Tcw, 7 * sizeof(double)); return 0; }  // S/Optimizer.cpp:290-291
  s.active.assign(N, 1); s.robust.assign(N, 1); s.err.assign(2 * N, 0.0);
  s.delta = (double)(float)std::sqrt(5.991);  // const float deltaMono = sqrt(5.991)
  std::fill(outlier, outlier + N, 0);
  const SE3 T0 = se3_load(p->Tcw);
  s.est = T0;
  int nBad = 0;
  for (int round = 0; round < 4; round++) {
    s.est = T0;          // vSE3->setEstimate(Converter::toSE3Quat(Frame.mTcw))
    s.trace = trace ? trace + (size_t)round * TRACE_CALL : nullptr;
    s.optimize(10);      // initializeOptimization(0) = the level-0 edges = s.active
    nBad = 0;
    for (int e = 0; e < N; e++) {
      if (outlier[e]) s.m.error(s.est, e, &s.err[2 * e]);  // e->computeError() for the edges left out of this round
      const float chi2 = (float)s.chi2_of(e);              // const float chi2 = e->chi2()
      if (chi2 > 5.991f) { outlier[e] = 1; s.active[e] = 0; nBad++; } else { outlier[e] = 0; s.active[e] = 1; }
      if (round == 2) s.robust[e] = 0;                     // e->setRobustKernel(0)
    }
    s.trace_chi2([](int) { return true; }, nBad);       // s.err now holds what the classification read, for every edge
    if (N < 10) break;  // optimizer.edges().size() < 10
  }
  se3_store(s.est, Tcw_out);
  return N - nBad;
}

int sim3_optimize(const orc_sim3_opt_problem* p, double* S12_out, uint8_t* inlier, double* trace) {
  Single<Sim3Model> s;
  s.m.p = p;
  const int N = p->n;
  s.active.assign(2 * N, 1); s.robust.assign(2 * N, 1); s.err.assign(4 * N, 0.0);
  s.delta = (double)(float)std::sqrt(p->th2);  // const float deltaHuber = sqrt(th2)
  s.est = sim3_load(p->S12);
  std::memcpy(S12_out, p->S12, 8 * sizeof(double));
  std::fill(inlier, inlier + N, 1);
  s.trace = trace;
  s.optimize(5);
  int nBad = 0;
  for (int i = 0; i < N; i++)
    if (s.chi2_of(2 * i) > (double)p->th2 || s.chi2_of(2 * i + 1) > (double)p->th2) {
      inlier[i] = 0; s.active[2 * i] = 0; s.active[2 * i + 1] = 0; nBad++;  // removeEdge(e12), removeEdge(e21)
    }
  s.trace_chi2([](int) { return true; }, nBad);
  const int more = nBad > 0 ? 10 : 5;
  if (N - nBad < 10) return 0;  // g2oS12 is left untouched
  s.trace = trace ? trace + TRACE_CALL : nullptr;
  s.optimize(more);
  int nIn = 0;
  for (int i = 0; i < N; i++) {
    if (!inlier[i]) continue;
    if (s.chi2_of(2 * i) > (double)p->th2 || s.chi2_of(2 * i + 1) > (double)p->th2) inlier[i] = 0; else nIn++;
  }
  s.trace_chi2([&](int e) { return s.active[e] != 0; }, N - nBad - nIn);  // the pairs that were still edges
  sim3_store(s.est, S12_out);
  return nIn;
}

}  // namespace

extern "C" int orc_pose_optimize(const orc_pose_opt_problem* p, double* Tcw_out, uint8_t* outlier) {
  return pose_optimize(p, Tcw_out, outlier, nullptr);
}
extern "C" int orc_sim3_optimize(const orc_sim3_opt_problem* p, double* S12_out, uint8_t* inlier) {
  return sim3_optimize(p, S12_out, inlier, nullptr);
}
// the same, recording g2o's Levenberg protocol of every optimize() call: 4 (pose) / 2 (Sim3) calls of TRACE_CALL doubles, NaN where
// a call or an iteration did not happen.  The trace only observes: the results are those of orc_pose_optimize / orc_sim3_optimize.
extern "C" int orc_pose_opt_trace(const orc_pose_opt_problem* p, double* Tcw_out, uint8_t* outlier, double* trace) {
  std::fill(trace, trace + 4 * TRACE_CALL, std::numeric_limits<double>::quiet_NaN());
  return pose_optimize(p, Tcw_out, outlier, trace);
}
extern "C" int orc_sim3_opt_trace(const orc_sim3_opt_problem* p, double* S12_out, uint8_t* inlier, double* trace) {
  std::fill(trace, trace + 2 * TRACE_CALL, std::numeric_limits<double>::quiet_NaN());
  return sim3_optimize(p, S12_out, inlier, trace);
}

// ---- pieces, for the reference pin of the edge types (tests/test_oracle_vs_reference_g2o.py) ------------------------------------
// quadratic form of every correspondence at the given estimate: H (D x D row-major), b (D), err (2 per edge)
extern "C" void orc_pose_opt_build(const orc_pose_opt_problem* p, const double* Tcw, int robust, double delta, double* H, double* b, double* err) {
  Single<PoseModel> s;
  s.m.p = p;
  s.active.assign(p->n, 1); s.robust.assign(p->n, robust ? 1 : 0); s.err.assign(2 * (size_t)p->n, 0.0);
  s.delta = delta;
  s.est = se3_load(Tcw);
  s.compute_active_errors();
  s.build(H, b);
  if (err) std::memcpy(err, s.err.data(), sizeof(double) * s.err.size());
}
extern "C" void orc_sim3_opt_build(const orc_sim3_opt_problem* p, const double* S12, int robust, double delta, double* H, double* b, double* err) {
  Single<Sim3Model> s;
  s.m.p = p;
  s.active.assign(2 * (size_t)p->n, 1); s.robust.assign(2 * (size_t)p->n, robust ? 1 : 0); s.err.assign(4 * (size_t)p->n, 0.0);
  s.delta = delta;
  s.est = sim3_load(S12);
  s.compute_active_errors();
  s.build(H, b);
  if (err) std::memcpy(err, s.err.data(), sizeof(double) * s.err.size());
}

// dense SPD solve for the LinearSolverDense stand-in (oracle/ref_stub_g2o): the same Cholesky the single-vertex optimisations above use
extern "C" int orc_chol_solve(int n, const double* A, const double* b, double* x) {
  if (n == 6) return chol_solve<6>(A, b, x) ? 0 : 1;
  if (n == 7) return chol_solve<7>(A, b, x) ? 0 : 1;
  std::vector<double> L((size_t)n * n, 0.0), y(n);          // any other size: the same recurrence, runtime-sized
  for (int i = 0; i < n; i++)
    for (int j = 0; j <= i; j++) {
      double s = A[(size_t)i * n + j];
      for (int k = 0; k < j; k++) s -= L[(size_t)i * n + k] * L[(size_t)j * n + k];
      if (i == j) { if (!(s > 0.0) || !std::isfinite(s)) return 1; L[(size_t)i * n + i] = std::sqrt(s); }
      else L[(size_t)i * n + j] = s / L[(size_t)j * n + j];
    }
  for (int i = 0; i < n; i++) { double s = b[i]; for (int k = 0; k < i; k++) s -= L[(size_t)i * n + k] * y[k]; y[i] = s / L[(size_t)i * n + i]; }
  for (int i = n - 1; i >= 0; i--) { double s = y[i]; for (int k = i + 1; k < n; k++) s -= L[(size_t)k * n + i] * x[k]; x[i] = s / L[(size_t)i * n + i]; }
  return 0;
}


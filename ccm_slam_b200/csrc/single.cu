// single.cu — the two single-vertex optimisations of cslam::Optimizer behind ccm_pose_optimize / ccm_sim3_optimize.
//
//   PoseOptimizationClient (S/Optimizer.cpp:215-347): VertexSE3Expmap + N unary EdgeSE3ProjectXYZOnlyPose (analytic Jacobian,
//     G/types/types_six_dof_expmap.cpp:266-288), Huber sqrt(5.991), 4 x {reset estimate, optimize(10), chi2 > 5.991 -> level 1},
//     kernel dropped after the third round.
//   OptimizeSim3 (S/Optimizer.cpp:861-1056): VertexSim3Expmap + per pair EdgeSim3ProjectXYZ / EdgeInverseSim3ProjectXYZ against
//     fixed points (G/types/types_seven_dof_expmap.h:130-172), numeric Jacobians (central differences, delta 1e-9,
//     G/core/base_binary_edge.hpp:131-205), optimize(5), drop pairs over th2, optimize(5 | 10).
//
// These are latency problems (one 6- or 7-dof vertex, <= a few thousand edges), so the whole protocol of one problem runs in ONE
// launch on ONE CTA: edges are strided over the threads, the dense normal equation is block-reduced in a fixed order, thread 0
// factorises it (LinearSolverDense -> unpivoted Cholesky with a positivity check) and every thread replays g2o's Levenberg
// decisions (G/core/optimization_algorithm_levenberg.cpp:61-189) on the same broadcast scalars.  A batch of problems
// (frames of several agents, loop / merge candidates of the place recogniser) is one CTA each in the same launch.
// g2o caches edge errors: after optimize() the reference classifies with the error of the LAST evaluated state (a rejected
// trial leaves stale errors) unless it calls computeError() itself; the err[] scratch array reproduces that.
#include <algorithm>
#include <cmath>
#include <cstring>
#include <vector>

#include "ba_math.cuh"
#include "common.cuh"
#include "sim3_math.cuh"

using namespace ccm;

namespace {

constexpr int ST = 256;      // threads per problem
constexpr int NRED = 40;     // >= 7*8/2 + 7

struct LMShared {
  double red[ST / 32][NRED];
  double out[NRED];
  double x[8];
  double st[8];              // current estimate: Pose (7) or S3 (8)
  double st_bak[8];
  double pert[14][8];        // estimates displaced by +-delta along each coordinate (numeric Jacobians)
  int flag;
  int cnt;
};

// sum `vals[0..K)` over the CTA in a fixed order; the totals land in sh.out[0..K) and are visible to every thread on return
template <int K>
__device__ void block_reduce_vec(double* vals, LMShared& sh) {
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
#pragma unroll
  for (int k = 0; k < K; k++) {
    double v = vals[k];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
    if (lane == 0) sh.red[wid][k] = v;
  }
  __syncthreads();
  if (threadIdx.x < K) {
    double s = 0.0;
#pragma unroll
    for (int w = 0; w < ST / 32; w++) s += sh.red[w][threadIdx.x];
    sh.out[threadIdx.x] = s;
  }
  __syncthreads();
}

template <int N>
__device__ bool chol_solve(const double* A, const double* b, double* x) {  // row-major SPD N x N; false: pivot not positive
  double L[N * N];
#pragma unroll
  for (int i = 0; i < N; i++)
#pragma unroll
    for (int j = 0; j <= i; j++) {
      double s = A[i * N + j];
      for (int k = 0; k < j; k++) s -= L[i * N + k] * L[j * N + k];
      if (i == j) {
        if (!(s > 0.0) || !isfinite(s)) return false;
        L[i * N + i] = sqrt(s);
      } else {
        L[i * N + j] = s / L[j * N + j];
      }
    }
  double y[N];
#pragma unroll
  for (int i = 0; i < N; i++) {
    double s = b[i];
    for (int k = 0; k < i; k++) s -= L[i * N + k] * y[k];
    y[i] = s / L[i * N + i];
  }
#pragma unroll
  for (int i = N - 1; i >= 0; i--) {
    double s = y[i];
    for (int k = i + 1; k < N; k++) s -= L[k * N + i] * x[k];
    x[i] = s / L[i * N + i];
  }
  return true;
}

// ---- models -----------------------------------------------------------------------------------------------------------------
struct PoseM {
  static constexpr int D = 6, NS = 7;
  int n;
  const float* Xw; const float* uv; const float* w;
  double fx, fy, cx, cy;
  __device__ int n_edges() const { return n; }
  __device__ double weight(int e) const { return (double)w[e]; }
  __device__ void camera_point(const double* st, int e, double& x, double& y, double& z) const {
    quat_rotate(st[0], st[1], st[2], st[3], (double)Xw[3 * e], (double)Xw[3 * e + 1], (double)Xw[3 * e + 2], x, y, z);
    x += st[4]; y += st[5]; z += st[6];
  }
  __device__ void error(const double* st, int e, double& e0, double& e1) const {  // types_six_dof_expmap.h:153-157
    double x, y, z;
    camera_point(st, e, x, y, z);
    e0 = (double)uv[2 * e] - (x / z * fx + cx);
    e1 = (double)uv[2 * e + 1] - (y / z * fy + cy);
  }
  __device__ void prepare(LMShared&) const {}
  __device__ void jacobian(const LMShared& sh, int e, double* J) const {  // types_six_dof_expmap.cpp:266-288
    double x, y, z;
    camera_point(sh.st, e, x, y, z);
    const double invz = 1.0 / z, invz_2 = invz * invz;
    J[0] = x * y * invz_2 * fx; J[1] = -(1 + (x * x * invz_2)) * fx; J[2] = y * invz * fx;
    J[3] = -invz * fx; J[4] = 0; J[5] = x * invz_2 * fx;
    J[6] = (1 + y * y * invz_2) * fy; J[7] = -x * y * invz_2 * fy; J[8] = -x * invz * fy;
    J[9] = 0; J[10] = -invz * fy; J[11] = y * invz_2 * fy;
  }
  __device__ void oplus(double* st, const double* x) const {  // VertexSE3Expmap::oplusImpl: exp(x) * T
    const Pose T{st[0], st[1], st[2], st[3], st[4], st[5], st[6]};
    const Pose o = se3_exp_times(x, T);
    st[0] = o.qx; st[1] = o.qy; st[2] = o.qz; st[3] = o.qw; st[4] = o.tx; st[5] = o.ty; st[6] = o.tz;
  }
};

struct Sim3M {
  static constexpr int D = 7, NS = 8;
  int n;  // pairs; edge 2i = EdgeSim3ProjectXYZ (camera 1 sees S12 * X2c), edge 2i+1 = EdgeInverseSim3ProjectXYZ
  const float* P1c; const float* P2c; const float* uv1; const float* uv2; const float* w1; const float* w2;
  double K1[4], K2[4];
  int fix_scale;
  __device__ int n_edges() const { return 2 * n; }
  __device__ double weight(int e) const { return (double)((e & 1) ? w2[e >> 1] : w1[e >> 1]); }
  __device__ void error(const double* st, int e, double& e0, double& e1) const {  // types_seven_dof_expmap.h:138-146,160-168
    const S3 S = s3_load(st);
    const int i = e >> 1;
    double x, y, z;
    if (!(e & 1)) {
      s3_map(S, (double)P2c[3 * i], (double)P2c[3 * i + 1], (double)P2c[3 * i + 2], x, y, z);
      e0 = (double)uv1[2 * i] - (x / z * K1[0] + K1[2]);
      e1 = (double)uv1[2 * i + 1] - (y / z * K1[1] + K1[3]);
    } else {
      s3_map(s3_inv(S), (double)P1c[3 * i], (double)P1c[3 * i + 1], (double)P1c[3 * i + 2], x, y, z);
      e0 = (double)uv2[2 * i] - (x / z * K2[0] + K2[2]);
      e1 = (double)uv2[2 * i + 1] - (y / z * K2[1] + K2[3]);
    }
  }
  __device__ void oplus(double* st, const double* x) const {  // VertexSim3Expmap::oplusImpl
    double u[7];
#pragma unroll
    for (int k = 0; k < 7; k++) u[k] = x[k];
    const S3 o = s3_oplus(s3_load(st), u, fix_scale);
    s3_store(o, st);
  }
  __device__ void prepare(LMShared& sh) const {  // the 14 displaced estimates are the same for every edge: build them once
    if (threadIdx.x < 14) {
      double u[7] = {0, 0, 0, 0, 0, 0, 0};
      u[threadIdx.x >> 1] = (threadIdx.x & 1) ? -1e-9 : 1e-9;
      double st[8];
#pragma unroll
      for (int k = 0; k < 8; k++) st[k] = sh.st[k];
      oplus(st, u);
#pragma unroll
      for (int k = 0; k < 8; k++) sh.pert[threadIdx.x][k] = st[k];
    }
    __syncthreads();
  }
  __device__ void jacobian(const LMShared& sh, int e, double* J) const {  // base_binary_edge.hpp:131-205, free vertex only
    const double scalar = 1.0 / (2 * 1e-9);
#pragma unroll 1
    for (int d = 0; d < 7; d++) {
      double p0, p1, m0, m1;
      error(sh.pert[2 * d], e, p0, p1);
      error(sh.pert[2 * d + 1], e, m0, m1);
      J[d] = scalar * (p0 - m0);
      J[7 + d] = scalar * (p1 - m1);
    }
  }
};

// computeActiveErrors + activeRobustChi2: refreshes err[] of the active edges at sh.st, returns the robust chi2 to every thread
template <class M>
__device__ double errors_and_chi(const M& m, LMShared& sh, const uint8_t* active, const uint8_t* robust, double* err, double delta) {
  double acc[1] = {0.0};
  for (int e = threadIdx.x; e < m.n_edges(); e += ST) {
    if (!active[e]) continue;
    double e0, e1;
    m.error(sh.st, e, e0, e1);
    err[2 * e] = e0; err[2 * e + 1] = e1;
    const double w = m.weight(e);
    const double c = e0 * (w * e0) + e1 * (w * e1);
    if (robust[e]) {
      double r0, r1;
      huber(c, delta, r0, r1);
      acc[0] += r0;
    } else {
      acc[0] += c;
    }
  }
  block_reduce_vec<1>(acc, sh);
  return sh.out[0];
}

// buildSystem at sh.st: JtWJ (H, full) and -JtWe (b) over the active edges, from the cached errors err[] of those edges.
// Every thread calls it and receives the same H and b.  lm_optimize and the test hook ccm_{pose,sim3}_debug_system share it.
template <class M>
__device__ void build_system(const M& m, LMShared& sh, const uint8_t* active, const uint8_t* robust, const double* err,
                             double delta, double* H, double* b) {
  constexpr int D = M::D, NH = D * (D + 1) / 2, NA = NH + D;
  m.prepare(sh);
  double acc[NA];
#pragma unroll
  for (int k = 0; k < NA; k++) acc[k] = 0.0;
  for (int e = threadIdx.x; e < m.n_edges(); e += ST) {
    if (!active[e]) continue;
    double J[2 * D];
    m.jacobian(sh, e, J);
    const double w = m.weight(e), e0 = err[2 * e], e1 = err[2 * e + 1];
    double wo = w, wr = 1.0;
    if (robust[e]) {
      double r0, r1;
      huber(e0 * (w * e0) + e1 * (w * e1), delta, r0, r1);
      wo = r1 * w; wr = r1;
    }
    const double b0 = -(w * e0) * wr, b1 = -(w * e1) * wr;
    int k = 0;
#pragma unroll
    for (int i = 0; i < D; i++)
#pragma unroll
      for (int j = i; j < D; j++) acc[k++] += J[i] * wo * J[j] + J[D + i] * wo * J[D + j];
#pragma unroll
    for (int i = 0; i < D; i++) acc[k++] += J[i] * b0 + J[D + i] * b1;
  }
  block_reduce_vec<NA>(acc, sh);
  int k = 0;
#pragma unroll
  for (int i = 0; i < D; i++)
#pragma unroll
    for (int j = i; j < D; j++) { H[i * D + j] = sh.out[k]; H[j * D + i] = sh.out[k]; k++; }
#pragma unroll
  for (int i = 0; i < D; i++) b[i] = sh.out[k++];
}

// ---- LM trace (test builds of the kernels only) ------------------------------------------------------------------------------
// The product kernels are instantiated with NoTrace, whose hooks are empty: they compile to the code they had before the trace
// existed.  LMTrace records, per optimize() call of one problem, a header {end, iterations, iteration limit, cached chi2, fresh
// chi2, stale edges, rejected} and per LM iteration the row {iniChi, lambda at the start, trials, rho of the last trial,
// currentChi at the end, accepted, failed Cholesky factorisations}.  end: 0 iteration limit, 1 ten rejected trials, 2 rho == 0,
// 3 three iterations without gain, -1 no active edge.  Only thread 0 writes.
constexpr int TR_ITERS = CCM_SINGLE_TRACE_ITERS, TR_COLS = CCM_SINGLE_TRACE_COLS, TR_HEAD = CCM_SINGLE_TRACE_HEAD;
constexpr int TR_CALL = TR_HEAD + TR_ITERS * TR_COLS;

struct NoTrace {
  static constexpr bool on = false;
  __device__ void iter(int, double, double, int, double, double, bool, int) const {}
  __device__ void end(int, int, int) const {}
  __device__ void chi2(double, double, double, int) const {}
  __device__ void next() {}
};

struct LMTrace {
  static constexpr bool on = true;
  double* p;  // this problem's calls, TR_CALL doubles each
  int call;
  __device__ double* c() const { return p + (size_t)call * TR_CALL; }
  __device__ void iter(int it, double ini, double lam, int q, double rho, double cur, bool acc, int nfail) const {
    if (threadIdx.x || it >= TR_ITERS) return;
    double* r = c() + TR_HEAD + it * TR_COLS;
    r[0] = ini; r[1] = lam; r[2] = q; r[3] = rho; r[4] = cur; r[5] = acc ? 1.0 : 0.0; r[6] = nfail;
  }
  __device__ void end(int code, int iters, int limit) const {
    if (!threadIdx.x) { c()[0] = code; c()[1] = iters; c()[2] = limit; }
  }
  __device__ void chi2(double cached, double fresh, double stale, int rejected) const {
    if (!threadIdx.x) { c()[3] = cached; c()[4] = fresh; c()[5] = stale; c()[6] = rejected; }
  }
  __device__ void next() { call++; }
};

// SparseOptimizer::optimize(iterations) with OptimizationAlgorithmLevenberg on the single free vertex held in sh.st.
// Every thread of the CTA calls it; returns the number of LM iterations (-1: no active edge).
template <class M, class Tr>
__device__ int lm_optimize(const M& m, LMShared& sh, const uint8_t* active, const uint8_t* robust, double* err, double delta,
                           int iterations, const Tr& tr) {
  constexpr int D = M::D;
  int any = 0;
  for (int e = threadIdx.x; e < m.n_edges(); e += ST) any |= active[e];
  if (!__syncthreads_or(any)) { tr.end(-1, -1, iterations); return -1; }
  double lambda = -1, ni = 2;
  int n_bad = 0, done = 0, end = 0;
  bool ok = true;
  for (int it = 0; it < iterations && ok; it++) {
    double currentChi = errors_and_chi(m, sh, active, robust, err, delta);
    const double iniChi = currentChi;
    double tempChi = currentChi;
    double H[D * D], b[D];
    build_system(m, sh, active, robust, err, delta, H, b);
    if (it == 0) {
      double maxd = 0;
#pragma unroll
      for (int i = 0; i < D; i++) {  // std::max(fabs(H_ii), maxd): a NaN diagonal entry replaces maxd (fmax would drop it)
        const double a = fabs(H[i * D + i]);
        maxd = (a < maxd) ? maxd : a;
      }
      lambda = 1e-5 * maxd; ni = 2; n_bad = 0;
    }
    const double lambda0 = lambda;
    int nfail = 0;
    double rho = 0;
    int qmax = 0;
    do {
      __syncthreads();  // everyone is done with sh.out / sh.st of the previous step
      if (threadIdx.x == 0) {
        for (int k = 0; k < M::NS; k++) sh.st_bak[k] = sh.st[k];  // push
        double Hd[D * D], x[D];
        for (int k = 0; k < D * D; k++) Hd[k] = H[k];
        for (int i = 0; i < D; i++) Hd[i * D + i] += lambda;
        const bool ok2 = chol_solve<D>(Hd, b, x);
        if (!ok2) for (int i = 0; i < D; i++) x[i] = 0.0;
        for (int i = 0; i < D; i++) sh.x[i] = x[i];
        sh.flag = ok2 ? 1 : 0;
        m.oplus(sh.st, x);
      }
      __syncthreads();
      tempChi = errors_and_chi(m, sh, active, robust, err, delta);
      const bool ok2 = sh.flag != 0;
      if (!ok2) { tempChi = 1.7976931348623157e308; nfail++; }
      rho = currentChi - tempChi;
      double scale = 0;
#pragma unroll
      for (int i = 0; i < D; i++) scale += sh.x[i] * (lambda * sh.x[i] + b[i]);
      scale += 1e-3;
      rho /= scale;
      if (rho > 0 && isfinite(tempChi)) {
        double alpha = 1. - pow((2 * rho - 1), 3);
        alpha = fmin(alpha, 2. / 3.);
        lambda *= fmax(1. / 3., alpha);
        ni = 2;
        currentChi = tempChi;
      } else {
        lambda *= ni; ni *= 2;
        __syncthreads();
        if (threadIdx.x == 0)
          for (int k = 0; k < M::NS; k++) sh.st[k] = sh.st_bak[k];  // pop: the cached errors stay those of the rejected state
      }
      qmax++;
    } while (rho < 0 && qmax < 10);
    __syncthreads();
    tr.iter(it, iniChi, lambda0, qmax, rho, currentChi, rho > 0 && isfinite(tempChi), nfail);
    done++;
    if (qmax == 10 || rho == 0) { ok = false; end = qmax == 10 ? 1 : 2; continue; }
    if ((iniChi - currentChi) * 1e3 < iniChi) n_bad++; else n_bad = 0;
    if (n_bad >= 3) { ok = false; end = 3; continue; }
  }
  tr.end(end, done, iterations);
  return done;
}

// trace only, over the edges with use(e): the chi2 of the cached errors err[] the classification read, the chi2 of fresh errors
// at sh.st, the number of edges whose cached error is not bit-identical to the fresh one, and the classification's rejections
template <class M, class Tr, class Use>
__device__ void trace_chi2(const M& m, LMShared& sh, const double* err, const Tr& tr, Use use, int rejected) {
  if constexpr (Tr::on) {
    double acc[3] = {0.0, 0.0, 0.0};
    for (int e = threadIdx.x; e < m.n_edges(); e += ST) {
      if (!use(e)) continue;
      const double w = m.weight(e);
      double f0, f1;
      m.error(sh.st, e, f0, f1);
      acc[0] += err[2 * e] * (w * err[2 * e]) + err[2 * e + 1] * (w * err[2 * e + 1]);
      acc[1] += f0 * (w * f0) + f1 * (w * f1);
      acc[2] += (err[2 * e] != f0 || err[2 * e + 1] != f1) ? 1.0 : 0.0;
    }
    __syncthreads();
    block_reduce_vec<3>(acc, sh);
    tr.chi2(sh.out[0], sh.out[1], sh.out[2], rejected);
    __syncthreads();
  }
}

// ---- PoseOptimizationClient -------------------------------------------------------------------------------------------------
struct PoseProb { int n; int off; double T0[7]; double fx, fy, cx, cy; };

template <class Tr>
__global__ void __launch_bounds__(ST) k_pose_optimize(const PoseProb* __restrict__ probs, const float* __restrict__ Xw,
                                                      const float* __restrict__ uv, const float* __restrict__ w,
                                                      double* __restrict__ err, uint8_t* __restrict__ flags,
                                                      uint8_t* __restrict__ outlier, double* __restrict__ T_out,
                                                      int* __restrict__ n_in, double* __restrict__ trace) {
  __shared__ LMShared sh;
  Tr tr{};
  if constexpr (Tr::on) { tr.p = trace + (size_t)blockIdx.x * CCM_SINGLE_TRACE_POSE_CALLS * TR_CALL; tr.call = 0; }
  const PoseProb p = probs[blockIdx.x];
  PoseM m;
  m.n = p.n; m.Xw = Xw + 3 * (size_t)p.off; m.uv = uv + 2 * (size_t)p.off; m.w = w + p.off;
  m.fx = p.fx; m.fy = p.fy; m.cx = p.cx; m.cy = p.cy;
  double* e_err = err + 2 * (size_t)p.off;
  uint8_t* active = flags + 2 * (size_t)p.off;
  uint8_t* robust = active + p.n;
  uint8_t* outl = outlier + p.off;
  const int N = p.n;
  if (N < 3) {  // S/Optimizer.cpp:290-291: return 0, Frame.mTcw untouched
    if (threadIdx.x < 7) T_out[7 * (size_t)blockIdx.x + threadIdx.x] = p.T0[threadIdx.x];
    if (threadIdx.x == 0) n_in[blockIdx.x] = 0;
    for (int e = threadIdx.x; e < N; e += ST) outl[e] = 0;
    return;
  }
  for (int e = threadIdx.x; e < N; e += ST) { active[e] = 1; robust[e] = 1; outl[e] = 0; e_err[2 * e] = 0; e_err[2 * e + 1] = 0; }
  const double delta = (double)(float)sqrt(5.991);  // const float deltaMono = sqrt(5.991)
  int nBad = 0;
  for (int round = 0; round < 4; round++) {
    __syncthreads();
    if (threadIdx.x < 7) sh.st[threadIdx.x] = p.T0[threadIdx.x];  // vSE3->setEstimate(Converter::toSE3Quat(Frame.mTcw))
    if (threadIdx.x == 0) sh.cnt = 0;
    __syncthreads();
    lm_optimize(m, sh, active, robust, e_err, delta, 10, tr);
    int bad = 0;
    for (int e = threadIdx.x; e < N; e += ST) {
      if (outl[e]) m.error(sh.st, e, e_err[2 * e], e_err[2 * e + 1]);  // e->computeError() for edges left out of the round
      const double wgt = m.weight(e);
      const float chi2 = (float)(e_err[2 * e] * (wgt * e_err[2 * e]) + e_err[2 * e + 1] * (wgt * e_err[2 * e + 1]));
      if (chi2 > 5.991f) { outl[e] = 1; active[e] = 0; bad++; } else { outl[e] = 0; active[e] = 1; }
      if (round == 2) robust[e] = 0;  // e->setRobustKernel(0)
    }
    atomicAdd(&sh.cnt, bad);
    __syncthreads();
    nBad = sh.cnt;
    trace_chi2(m, sh, e_err, tr, [](int) { return true; }, nBad);  // e_err holds what the classification read, every edge
    tr.next();
    if (N < 10) break;  // optimizer.edges().size() < 10
  }
  __syncthreads();
  if (threadIdx.x < 7) T_out[7 * (size_t)blockIdx.x + threadIdx.x] = sh.st[threadIdx.x];
  if (threadIdx.x == 0) n_in[blockIdx.x] = N - nBad;
}

// ---- OptimizeSim3 -----------------------------------------------------------------------------------------------------------
struct Sim3Prob { int n; int off; double S0[8]; double K1[4], K2[4]; float th2; int fix_scale; };

template <class Tr>
__global__ void __launch_bounds__(ST) k_sim3_optimize(const Sim3Prob* __restrict__ probs, const float* __restrict__ P1c,
                                                      const float* __restrict__ P2c, const float* __restrict__ uv1,
                                                      const float* __restrict__ uv2, const float* __restrict__ w1,
                                                      const float* __restrict__ w2, double* __restrict__ err,
                                                      uint8_t* __restrict__ flags, uint8_t* __restrict__ inlier,
                                                      double* __restrict__ S_out, int* __restrict__ n_in,
                                                      double* __restrict__ trace) {
  __shared__ LMShared sh;
  Tr tr{};
  if constexpr (Tr::on) { tr.p = trace + (size_t)blockIdx.x * CCM_SINGLE_TRACE_SIM3_CALLS * TR_CALL; tr.call = 0; }
  const Sim3Prob p = probs[blockIdx.x];
  Sim3M m;
  m.n = p.n; m.P1c = P1c + 3 * (size_t)p.off; m.P2c = P2c + 3 * (size_t)p.off; m.uv1 = uv1 + 2 * (size_t)p.off;
  m.uv2 = uv2 + 2 * (size_t)p.off; m.w1 = w1 + p.off; m.w2 = w2 + p.off; m.fix_scale = p.fix_scale;
#pragma unroll
  for (int k = 0; k < 4; k++) { m.K1[k] = p.K1[k]; m.K2[k] = p.K2[k]; }
  const int N = p.n, NE = 2 * N;
  double* e_err = err + 4 * (size_t)p.off;
  uint8_t* active = flags + 4 * (size_t)p.off;
  uint8_t* robust = active + NE;
  uint8_t* inl = inlier + p.off;
  for (int e = threadIdx.x; e < NE; e += ST) { active[e] = 1; robust[e] = 1; e_err[2 * e] = 0; e_err[2 * e + 1] = 0; }
  for (int i = threadIdx.x; i < N; i += ST) inl[i] = 1;
  if (threadIdx.x < 8) { sh.st[threadIdx.x] = p.S0[threadIdx.x]; S_out[8 * (size_t)blockIdx.x + threadIdx.x] = p.S0[threadIdx.x]; }
  if (threadIdx.x == 0) sh.cnt = 0;
  __syncthreads();
  const double th2 = (double)p.th2;
  const double delta = (double)sqrtf(p.th2);  // const float deltaHuber = sqrt(th2)
  auto pair_chi2_over = [&](int i) {
    const double wa = m.weight(2 * i), wb = m.weight(2 * i + 1);
    const double ca = e_err[4 * i] * (wa * e_err[4 * i]) + e_err[4 * i + 1] * (wa * e_err[4 * i + 1]);
    const double cb = e_err[4 * i + 2] * (wb * e_err[4 * i + 2]) + e_err[4 * i + 3] * (wb * e_err[4 * i + 3]);
    return ca > th2 || cb > th2;
  };
  lm_optimize(m, sh, active, robust, e_err, delta, 5, tr);
  int bad = 0;
  for (int i = threadIdx.x; i < N; i += ST)
    if (pair_chi2_over(i)) { inl[i] = 0; active[2 * i] = 0; active[2 * i + 1] = 0; bad++; }  // removeEdge(e12), removeEdge(e21)
  atomicAdd(&sh.cnt, bad);
  __syncthreads();
  const int nBad = sh.cnt;
  trace_chi2(m, sh, e_err, tr, [](int) { return true; }, nBad);
  tr.next();
  if (N - nBad < 10) {  // return 0 before g2oS12 is written
    if (threadIdx.x == 0) n_in[blockIdx.x] = 0;
    return;
  }
  __syncthreads();
  if (threadIdx.x == 0) sh.cnt = 0;
  __syncthreads();
  lm_optimize(m, sh, active, robust, e_err, delta, nBad > 0 ? 10 : 5, tr);
  int good = 0;
  for (int i = threadIdx.x; i < N; i += ST) {
    if (!inl[i]) continue;
    if (pair_chi2_over(i)) inl[i] = 0; else good++;
  }
  atomicAdd(&sh.cnt, good);
  __syncthreads();
  trace_chi2(m, sh, e_err, tr, [&](int e) { return active[e] != 0; }, N - nBad - sh.cnt);  // the pairs that were still edges
  if (threadIdx.x < 8) S_out[8 * (size_t)blockIdx.x + threadIdx.x] = sh.st[threadIdx.x];
  if (threadIdx.x == 0) n_in[blockIdx.x] = sh.cnt;
}

// ---- test hook: one linearisation and one damped solve per problem at a caller-given state ----------------------------------
// The same errors_and_chi / build_system / chol_solve as lm_optimize, on caller-given active and robust masks, Huber delta and
// lambda.  Per edge: the error and the Jacobian at the state (every edge, active or not); per problem: H (without lambda), b,
// the robust chi2 of the active edges, x of (H + lambda I) x = b (zeros when the factorisation fails) and the solved flag.
template <class M>
__device__ void debug_system(const M& m, LMShared& sh, const uint8_t* active, const uint8_t* robust, double* e_err, double delta,
                             double lambda, double* err_out, double* J_out, double* sys, int* solved) {
  constexpr int D = M::D;
  __syncthreads();
  const double chi = errors_and_chi(m, sh, active, robust, e_err, delta);
  double H[D * D], b[D];
  build_system(m, sh, active, robust, e_err, delta, H, b);  // leaves m.prepare's displaced states in sh
  for (int e = threadIdx.x; e < m.n_edges(); e += ST) {
    m.error(sh.st, e, err_out[2 * e], err_out[2 * e + 1]);
    m.jacobian(sh, e, J_out + (size_t)2 * D * e);
  }
  if (threadIdx.x == 0) {
    double Hd[D * D], x[D];
    for (int k = 0; k < D * D; k++) Hd[k] = H[k];
    for (int i = 0; i < D; i++) Hd[i * D + i] += lambda;
    const bool ok = chol_solve<D>(Hd, b, x);
    if (!ok) for (int i = 0; i < D; i++) x[i] = 0.0;
    for (int k = 0; k < D * D; k++) sys[k] = H[k];
    for (int i = 0; i < D; i++) { sys[D * D + i] = b[i]; sys[D * D + D + 1 + i] = x[i]; }
    sys[D * D + D] = chi;
    *solved = ok ? 1 : 0;
  }
}

__global__ void __launch_bounds__(ST) k_pose_debug_system(const PoseProb* __restrict__ probs, const float* __restrict__ Xw,
                                                          const float* __restrict__ uv, const float* __restrict__ w,
                                                          const uint8_t* __restrict__ active, const uint8_t* __restrict__ robust,
                                                          const double* __restrict__ dl, double* __restrict__ e_err,
                                                          double* __restrict__ err_out, double* __restrict__ J_out,
                                                          double* __restrict__ sys, int* __restrict__ solved) {
  __shared__ LMShared sh;
  const PoseProb p = probs[blockIdx.x];
  PoseM m;
  m.n = p.n; m.Xw = Xw + 3 * (size_t)p.off; m.uv = uv + 2 * (size_t)p.off; m.w = w + p.off;
  m.fx = p.fx; m.fy = p.fy; m.cx = p.cx; m.cy = p.cy;
  if (threadIdx.x < 7) sh.st[threadIdx.x] = p.T0[threadIdx.x];
  debug_system(m, sh, active + p.off, robust + p.off, e_err + 2 * (size_t)p.off, dl[2 * blockIdx.x], dl[2 * blockIdx.x + 1],
               err_out + 2 * (size_t)p.off, J_out + 12 * (size_t)p.off, sys + (size_t)blockIdx.x * (36 + 6 + 1 + 6),
               solved + blockIdx.x);
}

__global__ void __launch_bounds__(ST) k_sim3_debug_system(const Sim3Prob* __restrict__ probs, const float* __restrict__ P1c,
                                                          const float* __restrict__ P2c, const float* __restrict__ uv1,
                                                          const float* __restrict__ uv2, const float* __restrict__ w1,
                                                          const float* __restrict__ w2, const uint8_t* __restrict__ active,
                                                          const uint8_t* __restrict__ robust, const double* __restrict__ dl,
                                                          double* __restrict__ e_err, double* __restrict__ err_out,
                                                          double* __restrict__ J_out, double* __restrict__ sys,
                                                          int* __restrict__ solved) {
  __shared__ LMShared sh;
  const Sim3Prob p = probs[blockIdx.x];
  Sim3M m;
  m.n = p.n; m.P1c = P1c + 3 * (size_t)p.off; m.P2c = P2c + 3 * (size_t)p.off; m.uv1 = uv1 + 2 * (size_t)p.off;
  m.uv2 = uv2 + 2 * (size_t)p.off; m.w1 = w1 + p.off; m.w2 = w2 + p.off; m.fix_scale = p.fix_scale;
#pragma unroll
  for (int k = 0; k < 4; k++) { m.K1[k] = p.K1[k]; m.K2[k] = p.K2[k]; }
  if (threadIdx.x < 8) sh.st[threadIdx.x] = p.S0[threadIdx.x];
  debug_system(m, sh, active + 2 * (size_t)p.off, robust + 2 * (size_t)p.off, e_err + 4 * (size_t)p.off, dl[2 * blockIdx.x],
               dl[2 * blockIdx.x + 1], err_out + 4 * (size_t)p.off, J_out + 28 * (size_t)p.off,
               sys + (size_t)blockIdx.x * (49 + 7 + 1 + 7), solved + blockIdx.x);
}

template <typename T>
void append(std::vector<T>& dst, const T* src, size_t n) { dst.insert(dst.end(), src, src + n); }

struct StreamGuard {
  cudaStream_t s = nullptr;
  StreamGuard() { CCM_CUDA(cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking)); }
  ~StreamGuard() { if (s) cudaStreamDestroy(s); }
};

// a batch of pose problems on the device: one PoseProb per problem, the correspondences of all problems back to back
struct PoseBatch {
  std::vector<PoseProb> hp;
  size_t tot = 0;
  DevBuf<PoseProb> dp; DevBuf<float> dX, duv, dw;
  PoseBatch(const ccm_pose_opt_problem* probs, int batch, const ccm_pose_opt_result* res, const char* who, cudaStream_t s)
      : hp(batch) {
    std::vector<float> hX, huv, hw;
    for (int b = 0; b < batch; b++) {
      const ccm_pose_opt_problem& q = probs[b];
      CCM_REQUIRE(q.n >= 0 && q.Tcw && (q.n == 0 || (q.Xw && q.uv && q.inv_sigma2)) && (q.n == 0 || !res || res[b].outlier), who);
      PoseProb& d = hp[b];
      d.n = q.n; d.off = (int)tot;
      memcpy(d.T0, q.Tcw, sizeof(d.T0));
      d.fx = q.fx; d.fy = q.fy; d.cx = q.cx; d.cy = q.cy;
      append(hX, q.Xw, (size_t)3 * q.n); append(huv, q.uv, (size_t)2 * q.n); append(hw, q.inv_sigma2, (size_t)q.n);
      tot += q.n;
    }
    const size_t t1 = std::max(tot, (size_t)1);
    dp.upload(hp.data(), batch, s);
    dX.alloc(3 * t1); duv.alloc(2 * t1); dw.alloc(t1);
    if (tot) { dX.upload(hX.data(), hX.size(), s); duv.upload(huv.data(), huv.size(), s); dw.upload(hw.data(), hw.size(), s); }
  }
};

struct Sim3Batch {
  std::vector<Sim3Prob> hp;
  size_t tot = 0;
  DevBuf<Sim3Prob> dp; DevBuf<float> dP1, dP2, du1, du2, dw1, dw2;
  Sim3Batch(const ccm_sim3_opt_problem* probs, int batch, const ccm_sim3_opt_result* res, const char* who, cudaStream_t s)
      : hp(batch) {
    std::vector<float> hP1, hP2, hu1, hu2, hw1, hw2;
    for (int b = 0; b < batch; b++) {
      const ccm_sim3_opt_problem& q = probs[b];
      CCM_REQUIRE(q.n >= 0 && q.S12 &&
                      (q.n == 0 || (q.P1c && q.P2c && q.uv1 && q.uv2 && q.inv_sigma2_1 && q.inv_sigma2_2 && (!res || res[b].inlier))),
                  who);
      Sim3Prob& d = hp[b];
      d.n = q.n; d.off = (int)tot;
      memcpy(d.S0, q.S12, sizeof(d.S0));
      for (int k = 0; k < 4; k++) { d.K1[k] = q.K1[k]; d.K2[k] = q.K2[k]; }
      d.th2 = q.th2; d.fix_scale = q.fix_scale ? 1 : 0;
      append(hP1, q.P1c, (size_t)3 * q.n); append(hP2, q.P2c, (size_t)3 * q.n); append(hu1, q.uv1, (size_t)2 * q.n);
      append(hu2, q.uv2, (size_t)2 * q.n); append(hw1, q.inv_sigma2_1, (size_t)q.n); append(hw2, q.inv_sigma2_2, (size_t)q.n);
      tot += q.n;
    }
    const size_t t1 = std::max(tot, (size_t)1);
    dp.upload(hp.data(), batch, s);
    dP1.alloc(3 * t1); dP2.alloc(3 * t1); du1.alloc(2 * t1); du2.alloc(2 * t1); dw1.alloc(t1); dw2.alloc(t1);
    if (tot) {
      dP1.upload(hP1.data(), hP1.size(), s); dP2.upload(hP2.data(), hP2.size(), s); du1.upload(hu1.data(), hu1.size(), s);
      du2.upload(hu2.data(), hu2.size(), s); dw1.upload(hw1.data(), hw1.size(), s); dw2.upload(hw2.data(), hw2.size(), s);
    }
  }
};

// trace == nullptr: the product kernel; otherwise the traced instantiation writes batch * calls * TR_CALL doubles to trace
// (NaN where a call or an iteration did not happen)
void pose_optimize(const ccm_pose_opt_problem* probs, int batch, ccm_pose_opt_result* res, double* trace) {
  ensure_device();
  CCM_REQUIRE(batch >= 0 && (batch == 0 || (probs && res)), "ccm_pose_optimize: bad argument");
  if (batch == 0) return;
  StreamGuard sg;
  cudaStream_t s = sg.s;
  PoseBatch B(probs, batch, res, "ccm_pose_optimize: null array", s);
  const size_t tot = B.tot, t1 = std::max(tot, (size_t)1);
  DevBuf<double> derr, dT, dtr; DevBuf<uint8_t> dflags, dout; DevBuf<int> dn;
  derr.alloc(2 * t1); dflags.alloc(2 * t1); dout.alloc(t1); dT.alloc((size_t)7 * batch); dn.alloc(batch);
  const size_t ntr = (size_t)batch * CCM_SINGLE_TRACE_POSE_CALLS * TR_CALL;
  if (trace) {
    std::vector<double> nan(ntr, std::nan(""));
    dtr.upload(nan.data(), ntr, s);
    k_pose_optimize<LMTrace><<<batch, ST, 0, s>>>(B.dp.p, B.dX.p, B.duv.p, B.dw.p, derr.p, dflags.p, dout.p, dT.p, dn.p, dtr.p);
  } else {
    k_pose_optimize<NoTrace><<<batch, ST, 0, s>>>(B.dp.p, B.dX.p, B.duv.p, B.dw.p, derr.p, dflags.p, dout.p, dT.p, dn.p, nullptr);
  }
  CCM_LAUNCHED();
  std::vector<double> hT((size_t)7 * batch);
  std::vector<int> hn(batch);
  std::vector<uint8_t> ho(t1);
  dT.download(hT.data(), hT.size(), s); dn.download(hn.data(), hn.size(), s); dout.download(ho.data(), tot, s);
  if (trace) dtr.download(trace, ntr, s);
  CCM_CUDA(cudaStreamSynchronize(s));
  for (int b = 0; b < batch; b++) {
    memcpy(res[b].Tcw, hT.data() + 7 * (size_t)b, 7 * sizeof(double));
    res[b].n_inliers = hn[b];
    if (probs[b].n) memcpy(res[b].outlier, ho.data() + B.hp[b].off, (size_t)probs[b].n);
  }
}

void sim3_optimize(const ccm_sim3_opt_problem* probs, int batch, ccm_sim3_opt_result* res, double* trace) {
  ensure_device();
  CCM_REQUIRE(batch >= 0 && (batch == 0 || (probs && res)), "ccm_sim3_optimize: bad argument");
  if (batch == 0) return;
  StreamGuard sg;
  cudaStream_t s = sg.s;
  Sim3Batch B(probs, batch, res, "ccm_sim3_optimize: null array", s);
  const size_t tot = B.tot, t1 = std::max(tot, (size_t)1);
  DevBuf<double> derr, dS, dtr; DevBuf<uint8_t> dflags, dinl; DevBuf<int> dn;
  derr.alloc(4 * t1); dflags.alloc(4 * t1); dinl.alloc(t1); dS.alloc((size_t)8 * batch); dn.alloc(batch);
  const size_t ntr = (size_t)batch * CCM_SINGLE_TRACE_SIM3_CALLS * TR_CALL;
  if (trace) {
    std::vector<double> nan(ntr, std::nan(""));
    dtr.upload(nan.data(), ntr, s);
    k_sim3_optimize<LMTrace><<<batch, ST, 0, s>>>(B.dp.p, B.dP1.p, B.dP2.p, B.du1.p, B.du2.p, B.dw1.p, B.dw2.p, derr.p, dflags.p,
                                                 dinl.p, dS.p, dn.p, dtr.p);
  } else {
    k_sim3_optimize<NoTrace><<<batch, ST, 0, s>>>(B.dp.p, B.dP1.p, B.dP2.p, B.du1.p, B.du2.p, B.dw1.p, B.dw2.p, derr.p, dflags.p,
                                                 dinl.p, dS.p, dn.p, nullptr);
  }
  CCM_LAUNCHED();
  std::vector<double> hS((size_t)8 * batch);
  std::vector<int> hn(batch);
  std::vector<uint8_t> hi(t1);
  dS.download(hS.data(), hS.size(), s); dn.download(hn.data(), hn.size(), s); dinl.download(hi.data(), tot, s);
  if (trace) dtr.download(trace, ntr, s);
  CCM_CUDA(cudaStreamSynchronize(s));
  for (int b = 0; b < batch; b++) {
    memcpy(res[b].S12, hS.data() + 8 * (size_t)b, 8 * sizeof(double));
    res[b].n_inliers = hn[b];
    if (probs[b].n) memcpy(res[b].inlier, hi.data() + B.hp[b].off, (size_t)probs[b].n);
  }
}

void pose_debug_system(const ccm_pose_opt_problem* probs, int batch, const uint8_t* active, const uint8_t* robust,
                       const double* delta_lambda, double* err, double* J, double* sys, int32_t* solved) {
  ensure_device();
  CCM_REQUIRE(batch >= 0 && (batch == 0 || (probs && delta_lambda && sys && solved)), "ccm_pose_debug_system: bad argument");
  if (batch == 0) return;
  StreamGuard sg;
  cudaStream_t s = sg.s;
  PoseBatch B(probs, batch, nullptr, "ccm_pose_debug_system: null array", s);
  const size_t tot = B.tot, t1 = std::max(tot, (size_t)1);
  CCM_REQUIRE(tot == 0 || (active && robust && err && J), "ccm_pose_debug_system: null array");
  DevBuf<uint8_t> da, dr; DevBuf<double> ddl, de, derr, dJ, dsys; DevBuf<int> dsol;
  da.alloc(t1); dr.alloc(t1);
  if (tot) { da.upload(active, tot, s); dr.upload(robust, tot, s); }
  ddl.upload(delta_lambda, (size_t)2 * batch, s);
  de.alloc(2 * t1); derr.alloc(2 * t1); dJ.alloc(12 * t1); dsys.alloc((size_t)49 * batch); dsol.alloc(batch);
  k_pose_debug_system<<<batch, ST, 0, s>>>(B.dp.p, B.dX.p, B.duv.p, B.dw.p, da.p, dr.p, ddl.p, de.p, derr.p, dJ.p, dsys.p, dsol.p);
  CCM_LAUNCHED();
  if (tot) { derr.download(err, 2 * tot, s); dJ.download(J, 12 * tot, s); }
  dsys.download(sys, (size_t)49 * batch, s); dsol.download(solved, batch, s);
  CCM_CUDA(cudaStreamSynchronize(s));
}

void sim3_debug_system(const ccm_sim3_opt_problem* probs, int batch, const uint8_t* active, const uint8_t* robust,
                       const double* delta_lambda, double* err, double* J, double* sys, int32_t* solved) {
  ensure_device();
  CCM_REQUIRE(batch >= 0 && (batch == 0 || (probs && delta_lambda && sys && solved)), "ccm_sim3_debug_system: bad argument");
  if (batch == 0) return;
  StreamGuard sg;
  cudaStream_t s = sg.s;
  Sim3Batch B(probs, batch, nullptr, "ccm_sim3_debug_system: null array", s);
  const size_t tot = B.tot, t1 = std::max(tot, (size_t)1);
  CCM_REQUIRE(tot == 0 || (active && robust && err && J), "ccm_sim3_debug_system: null array");
  DevBuf<uint8_t> da, dr; DevBuf<double> ddl, de, derr, dJ, dsys; DevBuf<int> dsol;
  da.alloc(2 * t1); dr.alloc(2 * t1);
  if (tot) { da.upload(active, 2 * tot, s); dr.upload(robust, 2 * tot, s); }
  ddl.upload(delta_lambda, (size_t)2 * batch, s);
  de.alloc(4 * t1); derr.alloc(4 * t1); dJ.alloc(28 * t1); dsys.alloc((size_t)64 * batch); dsol.alloc(batch);
  k_sim3_debug_system<<<batch, ST, 0, s>>>(B.dp.p, B.dP1.p, B.dP2.p, B.du1.p, B.du2.p, B.dw1.p, B.dw2.p, da.p, dr.p, ddl.p, de.p,
                                           derr.p, dJ.p, dsys.p, dsol.p);
  CCM_LAUNCHED();
  if (tot) { derr.download(err, 4 * tot, s); dJ.download(J, 28 * tot, s); }
  dsys.download(sys, (size_t)64 * batch, s); dsol.download(solved, batch, s);
  CCM_CUDA(cudaStreamSynchronize(s));
}

}  // namespace

extern "C" int ccm_pose_optimize(const ccm_pose_opt_problem* probs, int32_t batch, ccm_pose_opt_result* res) {
  return guarded([&] { pose_optimize(probs, batch, res, nullptr); });
}

extern "C" int ccm_sim3_optimize(const ccm_sim3_opt_problem* probs, int32_t batch, ccm_sim3_opt_result* res) {
  return guarded([&] { sim3_optimize(probs, batch, res, nullptr); });
}

extern "C" int ccm_pose_optimize_traced(const ccm_pose_opt_problem* probs, int32_t batch, ccm_pose_opt_result* res, double* trace) {
  return guarded([&] {
    CCM_REQUIRE(trace || batch == 0, "ccm_pose_optimize_traced: bad argument");
    pose_optimize(probs, batch, res, trace);
  });
}

extern "C" int ccm_sim3_optimize_traced(const ccm_sim3_opt_problem* probs, int32_t batch, ccm_sim3_opt_result* res, double* trace) {
  return guarded([&] {
    CCM_REQUIRE(trace || batch == 0, "ccm_sim3_optimize_traced: bad argument");
    sim3_optimize(probs, batch, res, trace);
  });
}

extern "C" int ccm_pose_debug_system(const ccm_pose_opt_problem* probs, int32_t batch, const uint8_t* active, const uint8_t* robust,
                                     const double* delta_lambda, double* err, double* J, double* sys, int32_t* solved) {
  return guarded([&] { pose_debug_system(probs, batch, active, robust, delta_lambda, err, J, sys, solved); });
}

extern "C" int ccm_sim3_debug_system(const ccm_sim3_opt_problem* probs, int32_t batch, const uint8_t* active, const uint8_t* robust,
                                     const double* delta_lambda, double* err, double* J, double* sys, int32_t* solved) {
  return guarded([&] { sim3_debug_system(probs, batch, active, robust, delta_lambda, err, J, sys, solved); });
}

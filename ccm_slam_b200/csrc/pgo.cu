// pgo.cu — Sim3 essential-graph optimisation on the GPU behind ccm_pgo_solve (include/ccm_b200.h).
//
// Replaces optimizer.optimize(20) of Optimizer::OptimizeEssentialGraph{LoopClosure,MapFusion} (S/Optimizer.cpp:1277, :1513):
//   vertex  VertexSim3Expmap, oplus = Sim3(update) * estimate, update[6] := 0 when _fix_scale  (G/types/types_seven_dof_expmap.h:60-69)
//   edge    EdgeSim3, e = log(C * S_i * S_j^-1), information = I7                               (:105-114, S/Optimizer.cpp:1125)
//   solver  BlockSolver_7_3 without Schur, Levenberg with user lambda 1e-16                     (S/Optimizer.cpp:1066-1072)
// The reference differentiates numerically (central differences, delta = 1e-9, G/core/base_binary_edge.hpp:131-205);
// k_pgo_linearize does the same per edge (one thread per edge, 28 error evaluations) so that the Jacobians carry the same
// discretisation, then scatters J^T J / J^T e into the 7x7 block-CSR Hessian with red.add.f64.  The linear solve is the
// shared persistent PCG (pcg.cuh, BS = 7) instead of the reference's sparse LDL^T.
#include <algorithm>
#include <chrono>
#include <cmath>
#include <limits>

#include "ba_math.cuh"
#include "common.cuh"
#include "pcg.cuh"
#include "sim3_math.cuh"

using namespace ccm;

namespace {

struct PgoEdge { int i, j, ai, aj, idx_ii, idx_jj, idx_ij; int ij_transposed; };  // ai/aj: free index or -1

__global__ void __launch_bounds__(128) k_pgo_error(const double* __restrict__ v, const PgoEdge* __restrict__ edges,
                                                   const double* __restrict__ meas, int E, double* __restrict__ partials) {
  __shared__ double red[4];
  double acc = 0.0;
  for (int e = blockIdx.x * blockDim.x + threadIdx.x; e < E; e += gridDim.x * blockDim.x) {
    double err[7];
    edge_error(s3_load(meas + 8 * (size_t)e), s3_load(v + 8 * (size_t)edges[e].i), s3_load(v + 8 * (size_t)edges[e].j), err);
#pragma unroll
    for (int k = 0; k < 7; k++) acc += err[k] * err[k];
  }
  const double t = block_sum(acc, red);
  if (threadIdx.x == 0) partials[blockIdx.x] = t;
}

// One EdgeSim3: error e = log(C * vi * vj^-1) and its numeric Jacobians by central differences through oplus, delta = 1e-9
// (G/core/base_binary_edge.hpp:131-205).  J[r * 7 + d] = de_r / du_d; the Jacobian of a fixed side is exactly zero.
__device__ __forceinline__ void pgo_edge_linearize(const S3& C, const S3& vi, const S3& vj, bool free_i, bool free_j, int fix_scale,
                                                   double err[7], double Ji[49], double Jj[49]) {
  edge_error(C, vi, vj, err);
  const double delta = 1e-9, scalar = 1.0 / (2 * delta);
  for (int side = 0; side < 2; side++) {
    double* J = side ? Jj : Ji;
    const bool free_v = side ? free_j : free_i;
    for (int d = 0; d < 7; d++) {
      double ep[7], em[7], add[7] = {0, 0, 0, 0, 0, 0, 0};
      if (free_v) {
        add[d] = delta;
        if (side) edge_error(C, vi, s3_oplus(vj, add, fix_scale), ep); else edge_error(C, s3_oplus(vi, add, fix_scale), vj, ep);
        add[d] = -delta;
        if (side) edge_error(C, vi, s3_oplus(vj, add, fix_scale), em); else edge_error(C, s3_oplus(vi, add, fix_scale), vj, em);
      }
      for (int r = 0; r < 7; r++) J[r * 7 + d] = free_v ? scalar * (ep[r] - em[r]) : 0.0;
    }
  }
}

// one thread per edge: error, numeric Jacobians, scatter into H and b
__global__ void __launch_bounds__(64) k_pgo_linearize(const double* __restrict__ v, const PgoEdge* __restrict__ edges,
                                                      const double* __restrict__ meas, int E, int fix_scale,
                                                      double* __restrict__ H, double* __restrict__ b) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= E) return;
  const PgoEdge ed = edges[e];
  double err[7], Ji[49], Jj[49];
  pgo_edge_linearize(s3_load(meas + 8 * (size_t)e), s3_load(v + 8 * (size_t)ed.i), s3_load(v + 8 * (size_t)ed.j), ed.ai >= 0,
                     ed.aj >= 0, fix_scale, err, Ji, Jj);
  if (ed.ai >= 0) {
    for (int r = 0; r < 7; r++) {
      double g = 0;
      for (int k = 0; k < 7; k++) g -= Ji[k * 7 + r] * err[k];
      atomicAdd(b + (size_t)ed.ai * 7 + r, g);
      for (int c = 0; c < 7; c++) {
        double hh = 0;
        for (int k = 0; k < 7; k++) hh += Ji[k * 7 + r] * Ji[k * 7 + c];
        atomicAdd(H + (size_t)ed.idx_ii * 49 + r * 7 + c, hh);
      }
    }
  }
  if (ed.aj >= 0) {
    for (int r = 0; r < 7; r++) {
      double g = 0;
      for (int k = 0; k < 7; k++) g -= Jj[k * 7 + r] * err[k];
      atomicAdd(b + (size_t)ed.aj * 7 + r, g);
      for (int c = 0; c < 7; c++) {
        double hh = 0;
        for (int k = 0; k < 7; k++) hh += Jj[k * 7 + r] * Jj[k * 7 + c];
        atomicAdd(H + (size_t)ed.idx_jj * 49 + r * 7 + c, hh);
      }
    }
  }
  if (ed.ai >= 0 && ed.aj >= 0 && ed.ai != ed.aj) {
    // block (ai, aj) += Ji^T Jj and its mirror (aj, ai) += Jj^T Ji: the PCG works on the full symmetric block-CSR
    for (int r = 0; r < 7; r++)
      for (int c = 0; c < 7; c++) {
        double hh = 0;
        for (int k = 0; k < 7; k++) hh += Ji[k * 7 + r] * Jj[k * 7 + c];
        atomicAdd(H + (size_t)ed.idx_ij * 49 + r * 7 + c, hh);
        atomicAdd(H + (size_t)ed.ij_transposed * 49 + c * 7 + r, hh);
      }
  }
}

// per free vertex: Hd = H + lambda I on the diagonal block (written to Hs), Minv = inverse of that block (Gauss-Jordan)
__global__ void __launch_bounds__(64) k_pgo_damp(const double* __restrict__ H, double* __restrict__ Hs, long long nnz49,
                                                 const int* __restrict__ diag, int n, double lambda, double* __restrict__ Minv,
                                                 double* __restrict__ maxdiag_bits, int* __restrict__ fail) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  for (long long k = i; k < nnz49; k += (long long)gridDim.x * blockDim.x) Hs[k] = H[k];
  (void)maxdiag_bits;
  if (i >= n) return;
  double A[49], I[49];
  const double* src = H + (size_t)diag[i] * 49;
  for (int k = 0; k < 49; k++) { A[k] = src[k]; I[k] = 0.0; }
  for (int k = 0; k < 7; k++) { A[k * 8] += lambda; I[k * 8] = 1.0; }
  bool ok = true;
  for (int c = 0; c < 7; c++) {
    int piv = c;
    double best = fabs(A[c * 7 + c]);
    for (int r = c + 1; r < 7; r++)
      if (fabs(A[r * 7 + c]) > best) { best = fabs(A[r * 7 + c]); piv = r; }
    if (!(best > 0.0)) { ok = false; break; }
    if (piv != c)
      for (int k = 0; k < 7; k++) {
        double t = A[c * 7 + k]; A[c * 7 + k] = A[piv * 7 + k]; A[piv * 7 + k] = t;
        t = I[c * 7 + k]; I[c * 7 + k] = I[piv * 7 + k]; I[piv * 7 + k] = t;
      }
    const double ip = 1.0 / A[c * 7 + c];
    for (int k = 0; k < 7; k++) { A[c * 7 + k] *= ip; I[c * 7 + k] *= ip; }
    for (int r = 0; r < 7; r++) {
      if (r == c) continue;
      const double f = A[r * 7 + c];
      for (int k = 0; k < 7; k++) { A[r * 7 + k] -= f * A[c * 7 + k]; I[r * 7 + k] -= f * I[c * 7 + k]; }
    }
  }
  for (int k = 0; k < 49; k++) Minv[(size_t)i * 49 + k] = ok ? I[k] : (k % 8 == 0 ? 1.0 : 0.0);
  if (!ok) atomicExch(fail, 1);
}

__global__ void k_pgo_add_lambda(double* __restrict__ Hs, const int* __restrict__ diag, int n, double lambda) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n * 7) return;
  Hs[(size_t)diag[i / 7] * 49 + (i % 7) * 8] += lambda;
}

__global__ void __launch_bounds__(128) k_pgo_update(const double* __restrict__ v, const int* __restrict__ vidx,
                                                    const double* __restrict__ x, const double* __restrict__ b, int K,
                                                    int fix_scale, double lambda, double* __restrict__ vt,
                                                    double* __restrict__ partials) {
  __shared__ double red[4];
  double acc = 0.0;
  for (int k = blockIdx.x * blockDim.x + threadIdx.x; k < K; k += gridDim.x * blockDim.x) {
    S3 s = s3_load(v + 8 * (size_t)k);
    const int a = vidx[k];
    if (a >= 0) {
      double u[7];
      for (int d = 0; d < 7; d++) u[d] = x[(size_t)a * 7 + d];
      if (fix_scale) u[6] = 0;  // oplusImpl zeroes the solver's x[6] in place before computeScale reads it
      for (int d = 0; d < 7; d++) acc += u[d] * (lambda * u[d] + b[(size_t)a * 7 + d]);
      s = s3_oplus(s, u, fix_scale);
    }
    s3_store(s, vt + 8 * (size_t)k);
  }
  const double t = block_sum(acc, red);
  if (threadIdx.x == 0) partials[blockIdx.x] = t;
}

__global__ void __launch_bounds__(1024) k_sum(const double* __restrict__ p, int n, double* __restrict__ out) {
  __shared__ double red[32];
  double v = 0.0;
  for (int i = threadIdx.x; i < n; i += blockDim.x) v += p[i];
  const double t = block_sum(v, red);
  if (threadIdx.x == 0) out[0] = t;
}

__global__ void k_pgo_maxdiag(const double* __restrict__ H, const int* __restrict__ diag, int n, unsigned long long* out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n * 7) return;
  const double v = fabs(H[(size_t)diag[i / 7] * 49 + (i % 7) * 8]);
  atomicMax(out, (unsigned long long)__double_as_longlong(v));
}

// Coarse level of the PCG: below PGO_BIG free vertices, 64 nodes with piecewise-constant prolongation; from PGO_BIG on,
// PGO_BIG_NC nodes with piecewise-linear prolongation (CCM_PCG_NC / CCM_PCG_PROLONG override both).
constexpr int PGO_BIG = 4096;
constexpr int PGO_BIG_NC = 256;

// Host-side set-up shared by ccm_pgo_solve and ccm_pgo_debug_system: the active edges (at least one free end; an edge between two
// fixed vertices is dropped), the free-vertex index map vidx, the full symmetric block-CSR pattern of H (columns ascending), the
// scatter slots of every active edge, the PCG CTA and grid, and the coarse shape.  n == 0 (equivalently Ea == 0): nothing to solve.
struct PgoSetup {
  int K = 0, n = 0, Ea = 0;
  std::vector<int> vidx, rowptr, col, diag;
  std::vector<PgoEdge> edges;
  std::vector<double> meas;
  long long nnzb = 0;
  int gsm = 0, pcg_block = 0, pcg_grid = 0, c_agg = 0, c_nc = 0, c_prolong = 0;
  void* pcg_fn = nullptr;

  explicit PgoSetup(const ccm_pgo_problem* p) : K(p->K) {
    const int E = p->E;
    std::vector<char> has(K, 0);
    std::vector<int> act;
    for (int e = 0; e < E; e++) {
      const int i = p->edge_i[e], j = p->edge_j[e];
      CCM_REQUIRE(i >= 0 && i < K && j >= 0 && j < K, "ccm_pgo_solve: edge index out of range");
      if (p->fixed[i] && p->fixed[j]) continue;
      act.push_back(e);
      has[i] = has[j] = 1;
    }
    vidx.assign(K, -1);
    for (int k = 0; k < K; k++)
      if (has[k] && !p->fixed[k]) vidx[k] = n++;
    Ea = (int)act.size();
    rowptr.assign(n + 1, 0);
    if (n == 0 || Ea == 0) return;
    std::vector<std::vector<int>> rows(n);
    for (int a = 0; a < n; a++) rows[a].push_back(a);
    for (int e : act) {
      const int a = vidx[p->edge_i[e]], b = vidx[p->edge_j[e]];
      if (a >= 0 && b >= 0 && a != b) { rows[a].push_back(b); rows[b].push_back(a); }
    }
    diag.resize(n);
    for (int a = 0; a < n; a++) {
      std::sort(rows[a].begin(), rows[a].end());
      rows[a].erase(std::unique(rows[a].begin(), rows[a].end()), rows[a].end());
      col.insert(col.end(), rows[a].begin(), rows[a].end());
      rowptr[a + 1] = (int)col.size();
    }
    auto find = [&](int a, int b) {
      const int* bb = col.data() + rowptr[a];
      const int* ee = col.data() + rowptr[a + 1];
      return (int)(std::lower_bound(bb, ee, b) - col.data());
    };
    for (int a = 0; a < n; a++) diag[a] = find(a, a);
    edges.resize(Ea);
    meas.resize((size_t)Ea * 8);
    for (int k = 0; k < Ea; k++) {
      const int e = act[k];
      PgoEdge& ed = edges[k];
      ed.i = p->edge_i[e]; ed.j = p->edge_j[e]; ed.ai = vidx[ed.i]; ed.aj = vidx[ed.j];
      ed.idx_ii = ed.ai >= 0 ? diag[ed.ai] : 0; ed.idx_jj = ed.aj >= 0 ? diag[ed.aj] : 0;
      ed.idx_ij = (ed.ai >= 0 && ed.aj >= 0 && ed.ai != ed.aj) ? find(ed.ai, ed.aj) : 0;
      ed.ij_transposed = (ed.ai >= 0 && ed.aj >= 0 && ed.ai != ed.aj) ? find(ed.aj, ed.ai) : 0;
      memcpy(&meas[(size_t)k * 8], p->meas + 8 * (size_t)e, 8 * sizeof(double));
    }
    nnzb = (long long)col.size();
    gsm = sm_count();
    pcg_block = ((long long)n * 32 >= (long long)gsm * PCG_TPB) ? 512 : 256;
    pcg_fn = pcg_block == 512 ? (void*)k_pcg<7, 512, 1> : (void*)k_pcg<7, 256, 2>;
    int per_sm = 0;
    CCM_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, (const void*)pcg_fn, pcg_block, 0));
    CCM_REQUIRE(per_sm >= 1, "k_pcg does not fit on an SM");
    per_sm = std::min(per_sm, pcg_block == 256 ? 2 : 1);
    pcg_grid = std::max(1, std::min(gsm * per_sm, div_up((long long)n * 32, pcg_block)));
    const char* env_nc = getenv("CCM_PCG_NC");
    const char* env_pl = getenv("CCM_PCG_PROLONG");
    const bool big = n >= PGO_BIG;
    c_prolong = env_pl ? (atoi(env_pl) ? 1 : 0) : (big ? 1 : 0);
    pcg_coarse_shape(n, env_nc ? atoi(env_nc) : (big ? PGO_BIG_NC : 64), &c_agg, &c_nc);
  }
};

// Device buffers of one solve and the launches ccm_pgo_solve and ccm_pgo_debug_system share.
struct PgoDevice {
  const PgoSetup& S;
  cudaStream_t s;
  DevBuf<double> d_v, d_vt, d_meas, H, Hs, b, Minv, x, pr, pz, pp, pq, partials, scal, pcg_partials, pcg_status, cAc, crc, cyc;
  DevBuf<int> d_vidx, d_rowptr, d_col, d_diag, fail;
  DevBuf<PgoEdge> d_edges;
  DevBuf<unsigned> bar;

  PgoDevice(const PgoSetup& setup, const double* sim3, cudaStream_t stream) : S(setup), s(stream) {
    const int K = S.K, n = S.n;
    const long long nnzb = S.nnzb;
    d_v.upload(sim3, (size_t)K * 8, s); d_vt.alloc((size_t)K * 8);
    d_meas.upload(S.meas.data(), S.meas.size(), s); d_edges.upload(S.edges.data(), S.Ea, s);
    d_vidx.upload(S.vidx.data(), K, s); d_rowptr.upload(S.rowptr.data(), n + 1, s); d_col.upload(S.col.data(), nnzb, s);
    d_diag.upload(S.diag.data(), n, s);
    H.alloc(nnzb * 49); Hs.alloc(nnzb * 49); b.alloc((size_t)n * 7); Minv.alloc((size_t)n * 49);
    x.alloc_zero((size_t)n * 7, s); pr.alloc((size_t)n * 7); pz.alloc((size_t)n * 7); pp.alloc((size_t)2 * n * 7); pq.alloc((size_t)n * 7);
    partials.alloc((size_t)S.gsm * 8 + 8); scal.alloc_zero(8, s); pcg_status.alloc_zero(4, s); bar.alloc_zero(2, s); fail.alloc_zero(1, s);
    pcg_partials.alloc((size_t)3 * S.pcg_grid);
    const size_t nC = (size_t)7 * S.c_nc;
    cAc.alloc(std::max(2 * nC * nC, (size_t)1)); crc.alloc(std::max(2 * nC, (size_t)1)); cyc.alloc(std::max(nC, (size_t)1));
  }

  // chi2 of `state` (sum of e'e over the active edges) into dev_out
  void chi2_of(const double* state, double* dev_out) {
    const int g = std::max(1, std::min(div_up(S.Ea, 128), S.gsm * 8));
    k_pgo_error<<<g, 128, 0, s>>>(state, d_edges.p, d_meas.p, S.Ea, partials.p);
    CCM_LAUNCHED();
    k_sum<<<1, 1024, 0, s>>>(partials.p, g, dev_out);
    CCM_LAUNCHED();
  }

  // H and b (undamped) at `state`
  void linearize(const double* state, int fix_scale) {
    CCM_CUDA(cudaMemsetAsync(H.p, 0, H.bytes(), s));
    CCM_CUDA(cudaMemsetAsync(b.p, 0, b.bytes(), s));
    k_pgo_linearize<<<div_up(S.Ea, 64), 64, 0, s>>>(state, d_edges.p, d_meas.p, S.Ea, fix_scale, H.p, b.p);
    CCM_LAUNCHED();
  }

  // x = (H + lambda I)^-1 b by PCG: Hs = H + lambda I, Minv = block-Jacobi inverse (fail set when a block is singular),
  // pcg_status = [iterations, relres, flag, coarse size]
  void damped_pcg(double lambda, double tol, int max_iter) {
    const int n = S.n;
    const long long nnzb = S.nnzb;
    CCM_CUDA(cudaMemsetAsync(fail.p, 0, sizeof(int), s));
    k_pgo_damp<<<std::max(div_up(n, 64), std::min(div_up(nnzb * 49, 64), S.gsm * 16)), 64, 0, s>>>(
        H.p, Hs.p, nnzb * 49, d_diag.p, n, lambda, Minv.p, nullptr, fail.p);
    CCM_LAUNCHED();
    k_pgo_add_lambda<<<div_up(n * 7, 128), 128, 0, s>>>(Hs.p, d_diag.p, n, lambda);
    CCM_LAUNCHED();
    CCM_CUDA(cudaMemsetAsync(bar.p, 0, 2 * sizeof(unsigned), s));
    PcgArgs a;
    a.n = n; a.rowptr = d_rowptr.p; a.col = d_col.p; a.val = Hs.p; a.Minv = Minv.p; a.b = b.p;
    a.x = x.p; a.r = pr.p; a.z = pz.p; a.p = pp.p; a.q = pq.p; a.partials = pcg_partials.p; a.bar = bar.p;
    a.tol = tol; a.max_iter = max_iter; a.status = pcg_status.p;
    a.agg = S.c_agg; a.nc = S.c_nc; a.Ac = cAc.p; a.rc = crc.p; a.yc = cyc.p; a.coarse_mode = 1; a.prof = nullptr; a.prolong = S.c_prolong;
    void* args[] = {&a};
    CCM_CUDA(cudaLaunchCooperativeKernel(S.pcg_fn, dim3(S.pcg_grid), dim3(S.pcg_block), args, 0, s));
    CCM_LAUNCHED();
  }
};

int pcg_max_of(const ccm_pgo_options* o) { return o->pcg_max_iter > 0 ? o->pcg_max_iter : 5000; }
double pcg_tol_of(const ccm_pgo_options* o) { return o->pcg_tol > 0 ? o->pcg_tol : 1e-10; }

void pgo_solve(const ccm_pgo_problem* p, const ccm_pgo_options* o, ccm_pgo_result* r) {
  const auto T0 = std::chrono::steady_clock::now();
  ensure_device();
  CCM_REQUIRE(p && o && r && p->K > 0 && p->E >= 0 && p->sim3 && p->fixed && r->sim3, "ccm_pgo_solve: bad argument");
  const CallStream sg;
  const cudaStream_t s = sg.s;
  const int K = p->K;
  const PgoSetup S(p);
  const int n = S.n;
  r->trace_len = 0; r->iters_done = 0; r->chi2_initial = r->chi2_final = 0; r->lambda_final = 0;
  memcpy(r->sim3, p->sim3, sizeof(double) * 8 * K);
  if (n == 0 || S.Ea == 0) { r->iters_done = -1; return; }
  PgoDevice D(S, p->sim3, s);
  double* h_scal = nullptr;
  CCM_CUDA(cudaMallocHost((void**)&h_scal, 8 * sizeof(double)));
  struct HostGuard { double* p; ~HostGuard() { cudaFreeHost(p); } } hg{h_scal};
  double *cur = D.d_v.p, *trial = D.d_vt.p;
  const int pcg_max = pcg_max_of(o);
  const double pcg_tol = pcg_tol_of(o);
  auto terminate = [&] { return o->stop && *o->stop; };
  double lambda = -1, ni = 2;
  int nBad = 0, ret = 0;
  bool ok = true;
  for (int it = 0; it < o->iterations && !terminate() && ok; it++) {
    D.chi2_of(cur, D.scal.p);
    D.linearize(cur, p->fix_scale);
    if (it == 0 && !(o->lambda_init > 0)) {
      CCM_CUDA(cudaMemsetAsync(D.scal.p + 4, 0, sizeof(double), s));
      k_pgo_maxdiag<<<div_up(n * 7, 128), 128, 0, s>>>(D.H.p, D.d_diag.p, n, reinterpret_cast<unsigned long long*>(D.scal.p + 4));
      CCM_LAUNCHED();
    }
    CCM_CUDA(cudaMemcpyAsync(h_scal, D.scal.p, 5 * sizeof(double), cudaMemcpyDeviceToHost, s));
    CCM_CUDA(cudaStreamSynchronize(s));
    double currentChi = h_scal[0];
    const double iniChi = currentChi;
    if (it == 0) {
      r->chi2_initial = currentChi;
      lambda = o->lambda_init > 0 ? o->lambda_init : 1e-5 * h_scal[4];
      ni = 2; nBad = 0;
    }
    double rho = 0, tempChi = currentChi, lambda_used = lambda, relres = 0;
    int qmax = 0, pcg_it = 0;
    do {
      lambda_used = lambda;
      D.damped_pcg(lambda, pcg_tol, pcg_max);
      const int g = std::max(1, std::min(div_up(K, 128), S.gsm * 8));
      k_pgo_update<<<g, 128, 0, s>>>(cur, D.d_vidx.p, D.x.p, D.b.p, K, p->fix_scale, lambda, trial, D.partials.p);
      CCM_LAUNCHED();
      k_sum<<<1, 1024, 0, s>>>(D.partials.p, g, D.scal.p + 1);
      CCM_LAUNCHED();
      D.chi2_of(trial, D.scal.p + 2);
      CCM_CUDA(cudaMemcpyAsync(h_scal, D.scal.p, 3 * sizeof(double), cudaMemcpyDeviceToHost, s));
      CCM_CUDA(cudaMemcpyAsync(h_scal + 3, D.pcg_status.p, 3 * sizeof(double), cudaMemcpyDeviceToHost, s));
      CCM_CUDA(cudaMemcpyAsync(h_scal + 6, D.fail.p, sizeof(int), cudaMemcpyDeviceToHost, s));
      CCM_CUDA(cudaStreamSynchronize(s));
      int jfail;
      memcpy(&jfail, h_scal + 6, sizeof(int));
      tempChi = h_scal[2];
      pcg_it = (int)h_scal[3]; relres = h_scal[4];
      const bool ok2 = !((int)h_scal[5] == 2 || jfail);
      if (!ok2) tempChi = std::numeric_limits<double>::max();
      rho = currentChi - tempChi;
      double scale = h_scal[1];
      scale += 1e-3;
      rho /= scale;
      if (rho > 0 && std::isfinite(tempChi)) {
        double alpha = 1. - std::pow((2 * rho - 1), 3);
        alpha = std::min(alpha, 2. / 3.);
        lambda *= std::max(1. / 3., alpha);
        ni = 2;
        currentChi = tempChi;
        std::swap(cur, trial);
      } else {
        lambda *= ni;
        ni *= 2;
      }
      qmax++;
    } while (rho < 0 && qmax < 10 && !terminate());
    ret++;
    if (r->trace && r->trace_len < r->trace_cap) {
      double* tr = r->trace + (size_t)r->trace_len * CCM_TRACE_COLS;
      tr[0] = it; tr[1] = lambda_used; tr[2] = currentChi; tr[3] = rho; tr[4] = qmax; tr[5] = lambda; tr[6] = pcg_it; tr[7] = relres;
      r->trace_len++;
    }
    r->chi2_final = currentChi; r->lambda_final = lambda;
    if (qmax == 10 || rho == 0) { ok = false; continue; }
    if ((iniChi - currentChi) * 1e3 < iniChi) nBad++; else nBad = 0;
    if (nBad >= 3) { ok = false; continue; }
  }
  r->iters_done = ret;
  CCM_CUDA(cudaMemcpyAsync(r->sim3, cur, sizeof(double) * 8 * K, cudaMemcpyDeviceToHost, s));
  CCM_CUDA(cudaStreamSynchronize(s));
  r->t_total_ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - T0).count();
}

// ---- test-only entry points: the product's own device code on caller-chosen inputs ----------------------------------------

__global__ void k_sim3_debug_ops(int n, const double* __restrict__ u, const double* __restrict__ a, const double* __restrict__ b,
                                 int fix_scale, double* __restrict__ exp_u, double* __restrict__ log_a, double* __restrict__ mul_ab,
                                 double* __restrict__ inv_a, double* __restrict__ oplus_u_a) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  double uu[7];
  for (int d = 0; d < 7; d++) uu[d] = u[(size_t)i * 7 + d];
  const S3 A = s3_load(a + 8 * (size_t)i), B = s3_load(b + 8 * (size_t)i);
  s3_store(s3_exp(uu), exp_u + 8 * (size_t)i);
  s3_log(A, log_a + 7 * (size_t)i);
  s3_store(s3_mul(A, B), mul_ab + 8 * (size_t)i);
  s3_store(s3_inv(A), inv_a + 8 * (size_t)i);
  s3_store(s3_oplus(A, uu, fix_scale), oplus_u_a + 8 * (size_t)i);
}

__global__ void __launch_bounds__(64) k_pgo_debug_edges(int n, const double* __restrict__ meas, const double* __restrict__ si,
                                                        const double* __restrict__ sj, const int* __restrict__ free_ij, int fix_scale,
                                                        double* __restrict__ err, double* __restrict__ Ji, double* __restrict__ Jj) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= n) return;
  double er[7], ji[49], jj[49];
  pgo_edge_linearize(s3_load(meas + 8 * (size_t)e), s3_load(si + 8 * (size_t)e), s3_load(sj + 8 * (size_t)e), free_ij[2 * e] != 0,
                     free_ij[2 * e + 1] != 0, fix_scale, er, ji, jj);
  for (int k = 0; k < 7; k++) err[(size_t)e * 7 + k] = er[k];
  for (int k = 0; k < 49; k++) { Ji[(size_t)e * 49 + k] = ji[k]; Jj[(size_t)e * 49 + k] = jj[k]; }
}

void sim3_debug_ops(int n, const double* u, const double* a, const double* b, int fix_scale, double* exp_u, double* log_a,
                    double* mul_ab, double* inv_a, double* oplus_u_a) {
  ensure_device();
  CCM_REQUIRE(n >= 0 && (n == 0 || (u && a && b && exp_u && log_a && mul_ab && inv_a && oplus_u_a)), "ccm_sim3_debug_ops: bad argument");
  if (n == 0) return;
  const CallStream sg;
  DevBuf<double> du, da, db, o_exp, o_log, o_mul, o_inv, o_oplus;
  du.upload(u, (size_t)n * 7, sg.s); da.upload(a, (size_t)n * 8, sg.s); db.upload(b, (size_t)n * 8, sg.s);
  o_exp.alloc((size_t)n * 8); o_log.alloc((size_t)n * 7); o_mul.alloc((size_t)n * 8); o_inv.alloc((size_t)n * 8); o_oplus.alloc((size_t)n * 8);
  k_sim3_debug_ops<<<div_up(n, 64), 64, 0, sg.s>>>(n, du.p, da.p, db.p, fix_scale, o_exp.p, o_log.p, o_mul.p, o_inv.p, o_oplus.p);
  CCM_LAUNCHED();
  o_exp.download(exp_u, (size_t)n * 8, sg.s); o_log.download(log_a, (size_t)n * 7, sg.s); o_mul.download(mul_ab, (size_t)n * 8, sg.s);
  o_inv.download(inv_a, (size_t)n * 8, sg.s); o_oplus.download(oplus_u_a, (size_t)n * 8, sg.s);
  CCM_CUDA(cudaStreamSynchronize(sg.s));
}

void pgo_debug_edges(int n, const double* meas, const double* si, const double* sj, const int32_t* free_ij, int fix_scale, double* err,
                     double* Ji, double* Jj) {
  ensure_device();
  CCM_REQUIRE(n >= 0 && (n == 0 || (meas && si && sj && free_ij && err && Ji && Jj)), "ccm_pgo_debug_edges: bad argument");
  if (n == 0) return;
  const CallStream sg;
  DevBuf<double> dm, di, dj, de, dJi, dJj;
  DevBuf<int> df;
  dm.upload(meas, (size_t)n * 8, sg.s); di.upload(si, (size_t)n * 8, sg.s); dj.upload(sj, (size_t)n * 8, sg.s);
  df.upload(free_ij, (size_t)n * 2, sg.s);
  de.alloc((size_t)n * 7); dJi.alloc((size_t)n * 49); dJj.alloc((size_t)n * 49);
  k_pgo_debug_edges<<<div_up(n, 64), 64, 0, sg.s>>>(n, dm.p, di.p, dj.p, df.p, fix_scale, de.p, dJi.p, dJj.p);
  CCM_LAUNCHED();
  de.download(err, (size_t)n * 7, sg.s); dJi.download(Ji, (size_t)n * 49, sg.s); dJj.download(Jj, (size_t)n * 49, sg.s);
  CCM_CUDA(cudaStreamSynchronize(sg.s));
}

void pgo_debug_system(const ccm_pgo_problem* p, const ccm_pgo_options* o, double lambda, int32_t* n_free, int64_t* nnzb,
                      int32_t* vidx, int32_t* rowptr, int32_t* col, double* H, double* b, double* Minv, double* x, double* chi2,
                      double* pcg, int32_t* paths) {
  ensure_device();
  CCM_REQUIRE(p && o && n_free && nnzb && p->K > 0 && p->E >= 0 && p->sim3 && p->fixed, "ccm_pgo_debug_system: bad argument");
  const PgoSetup S(p);
  *n_free = S.n; *nnzb = S.nnzb;
  if (vidx) memcpy(vidx, S.vidx.data(), sizeof(int32_t) * S.K);
  if (rowptr) memcpy(rowptr, S.rowptr.data(), sizeof(int32_t) * (S.n + 1));
  if (col && S.nnzb) memcpy(col, S.col.data(), sizeof(int32_t) * S.nnzb);
  if (paths) { paths[0] = S.pcg_block; paths[1] = S.c_agg; paths[2] = S.c_nc; paths[3] = 0; }
  if (!H || S.n == 0) return;
  CCM_REQUIRE(b && Minv && x && chi2 && pcg, "ccm_pgo_debug_system: bad argument");
  const CallStream sg;
  PgoDevice D(S, p->sim3, sg.s);
  D.chi2_of(D.d_v.p, D.scal.p);
  D.linearize(D.d_v.p, p->fix_scale);
  D.damped_pcg(lambda, pcg_tol_of(o), pcg_max_of(o));
  D.H.download(H, (size_t)S.nnzb * 49, sg.s); D.b.download(b, (size_t)S.n * 7, sg.s); D.Minv.download(Minv, (size_t)S.n * 49, sg.s);
  D.x.download(x, (size_t)S.n * 7, sg.s); D.scal.download(chi2, 1, sg.s); D.pcg_status.download(pcg, 4, sg.s);
  CCM_CUDA(cudaStreamSynchronize(sg.s));
  if (paths) paths[3] = pcg[3] > 0;
}

}  // namespace

extern "C" int ccm_pgo_solve(const ccm_pgo_problem* p, const ccm_pgo_options* o, ccm_pgo_result* r) {
  return guarded([&] { pgo_solve(p, o, r); });
}

extern "C" int ccm_sim3_debug_ops(int32_t n, const double* u, const double* a, const double* b, int32_t fix_scale, double* exp_u,
                                  double* log_a, double* mul_ab, double* inv_a, double* oplus_u_a) {
  return guarded([&] { sim3_debug_ops(n, u, a, b, fix_scale, exp_u, log_a, mul_ab, inv_a, oplus_u_a); });
}

extern "C" int ccm_pgo_debug_edges(int32_t n, const double* meas, const double* si, const double* sj, const int32_t* free_ij,
                                   int32_t fix_scale, double* err, double* Ji, double* Jj) {
  return guarded([&] { pgo_debug_edges(n, meas, si, sj, free_ij, fix_scale, err, Ji, Jj); });
}

extern "C" int ccm_pgo_debug_system(const ccm_pgo_problem* p, const ccm_pgo_options* o, double lambda, int32_t* n_free, int64_t* nnzb,
                                    int32_t* vidx, int32_t* rowptr, int32_t* col, double* H, double* b, double* Minv, double* x,
                                    double* chi2, double* pcg, int32_t* paths) {
  return guarded([&] { pgo_debug_system(p, o, lambda, n_free, nnzb, vidx, rowptr, col, H, b, Minv, x, chi2, pcg, paths); });
}

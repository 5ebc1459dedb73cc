// pcg.cuh — persistent cooperative preconditioned conjugate gradients on a block-CSR SPD system (block size BS).
//
// Replaces the direct sparse LDL^T of g2o's LinearSolverEigen (G/solvers/linear_solver_eigen.h:106-133) on the reduced
// camera system (BS = 6, bundle adjustment) and on the Sim3 pose-graph Hessian (BS = 7, essential graph).  One warp per
// block row; the whole solve runs inside one kernel launched with cudaLaunchCooperativeKernel, grid-wide barriers go
// through a global counter, dot products are reduced in a fixed order so that every CTA sees identical scalars.
//
// Preconditioner: two-level additive Schwarz,  M^-1 = blockdiag(S)^-1 + P (P^T S P)^-1 P^T.
//   * fine level: block-Jacobi (inverse diagonal blocks, computed by the caller);
//   * coarse level (prolong = 0; the pose graph's BS = 7 solve and CCM_PCG_PROLONG=0): aggregates of `agg` consecutive block rows (keyframes are ordered along each agent's trajectory, so
//     index neighbours are co-visible), piecewise-constant prolongation per degree of freedom -> a dense (BS*nc)^2
//     Galerkin matrix, nc <= 128, assembled and inverted (ping-pong Gauss-Jordan, one grid barrier per pivot) inside the
//     same kernel before the iteration starts.  It removes the smooth error modes along the trajectory that make
//     block-Jacobi PCG iteration counts grow with the number of keyframes.
//   * prolong = 1 (bundle adjustment's default): the same coarse nodes, but P interpolates linearly between aggregate centres.  On the
//     cfg5 chain this cuts the iteration count 2.2-2.9x at equal coarse size and a linear P over 192 nodes beats a constant P
//     over 768 (tools/pcg_precond_study.py).  The default (cfg5: 1538 -> 617 iterations at 192 nodes, 496 at 256 nodes).
#pragma once
#include <cuda_runtime.h>

namespace ccm {

constexpr int TPB = 256;
// Coarse-matrix inversion: GJB pivots per Gauss-Jordan sweep, so one grid barrier and one pass over the matrix per GJB pivots.
// Both products of a sweep run on the f64 tensor cores.  On cfg5 (nC = 1536: 48 sweeps) the set-up launch (assembly + inverse)
// takes 2.0 ms; at 8 pivots per sweep on the CUDA cores it took 4.9 ms (H100 80GB HBM3, 700 W).
constexpr int GJB = 32;
constexpr int GJ_CW = 128;     // column chunk a CTA stages per sweep
constexpr int GJ_LDP = GJB + 4;     // padded row strides of the shared pivot inverse / pivot rows: the B fragments of
constexpr int GJ_LDR = GJ_CW + 4;   // mma.m8n8k4 read 4 rows x 8 columns, unpadded those 4 rows fall into the same banks
constexpr int PCG_TPB = 1024;  // one fat CTA per SM keeps the grid barrier at one participant per SM (132 on an H100 SXM)

// The ping-pong buffer of Ac (2 (BS nc)^2 doubles) that holds the coarse inverse after the set-up: the sweep count's parity.
__host__ __device__ inline double* coarse_inverse(double* Ac, int nC) {
  return (((nC + GJB - 1) / GJB) & 1) ? Ac + (size_t)nC * nC : Ac;
}

// D += A B on one 8x8x4 f64 tensor-core tile.  A (8x4 row-major): lane t holds A[t/4][t%4]; B (4x8 col-major): lane t holds
// B[t%4][t/4]; C / D (8x8): lane t holds C[t/4][2 (t%4)] and C[t/4][2 (t%4) + 1].
__device__ __forceinline__ void dmma_884(double& c0, double& c1, double a, double b) {
  asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0, %1}, {%2}, {%3}, {%0, %1};"
               : "+d"(c0), "+d"(c1)
               : "d"(a), "d"(b));
}

__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// block-wide sum; result valid in thread 0.  smem must hold blockDim/32 doubles.
__device__ __forceinline__ double block_sum(double v, double* smem) {
  v = warp_sum(v);
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  __syncthreads();
  if (lane == 0) smem[wid] = v;
  __syncthreads();
  double r = 0;
  if (wid == 0) {
    r = lane < (blockDim.x >> 5) ? smem[lane] : 0.0;
    r = warp_sum(r);
  }
  return r;
}

struct PcgArgs {
  int n;  // block rows
  const int* rowptr; const int* col; const double* val; const double* Minv; const double* b;
  double *x, *r, *z, *p, *q;  // p: 2 * n*BS (double buffered search direction)
  double* partials;  // 3 * gridDim.x
  unsigned* bar;     // zeroed before launch
  double tol; int max_iter;
  double* status;    // [iters, relres, flag(0 converged, 1 max_iter, 2 breakdown: p'Sp <= 0), coarse_used]
  // coarse level (agg <= 0 disables it)
  int agg, nc;       // rows per aggregate, number of aggregates
  int coarse_mode;   // 1: assemble + invert now, 2: reuse the inverse a previous launch left in Ac (still a valid SPD preconditioner),
                     // 3: assemble into Ac and return (debug export)
  int prolong = 0;   // 0: piecewise-constant prolongation (one coarse node per aggregate), 1: piecewise linear between aggregate centres
  double* Ac;        // 2 * (BS*nc)^2 ping-pong buffers
  double* rc;        // 2 * BS*nc restricted residual (double buffered)
  double* yc;        // BS*nc coarse correction
  long long* prof;   // optional: 8 cycle counters filled by CTA 0 (setup, spmv, update+restrict, coarse, precond, unused) or NULL
};

// One counter, every CTA polls it.  (Round 2 tried the variant k_pcg2 uses -- the last arriver releases a separate generation word
// the others poll -- here too: with two CTAs of 256 threads per SM it was slower on cfg4: the extra hop costs more than the
// contention it removes.)
__device__ __forceinline__ void grid_barrier(unsigned* bar, unsigned& target) {
  __syncthreads();
  if (threadIdx.x == 0) {
    target += gridDim.x;
    __threadfence();
    atomicAdd(bar, 1u);
    while (*(volatile unsigned*)bar < target) {}
    __threadfence();
  }
  __syncthreads();
}

// Coarse parents of fine block row a.  Piecewise constant: the aggregate a / agg with weight 1.  Piecewise linear: the two
// aggregate centres ((g + 1/2) agg - 1/2) that bracket a, hat-function weights; rows outside the first / last centre take the
// end node with weight 1.  The columns of P stay a partition of unity, so P^T S P is SPD whenever S is.
struct CoarseParents { int lo, hi; double w0, w1; };
__device__ __forceinline__ CoarseParents coarse_parents(int a, int agg, int nc, int prolong) {
  CoarseParents c;
  if (!prolong || nc < 2) {
    c.lo = c.hi = a / agg; c.w0 = 1.0; c.w1 = 0.0;
    return c;
  }
  double pos = ((double)a + 0.5) / (double)agg - 0.5;
  pos = fmin(fmax(pos, 0.0), (double)(nc - 1));
  int lo = (int)pos;  // pos >= 0: truncation is floor
  if (lo > nc - 2) lo = nc - 2;
  const double f = fmin(fmax(pos - (double)lo, 0.0), 1.0);
  c.lo = lo; c.hi = lo + 1; c.w0 = 1.0 - f; c.w1 = f;
  return c;
}

// sum of partials[0..g) in a fixed order, same value in every thread of the calling warp
__device__ __forceinline__ double sum_partials_dev(const double* partials, int g) {
  double v = 0.0;
  for (int i = threadIdx.x & 31; i < g; i += 32) v += __ldcg(partials + i);
  return warp_sum(v);
}

// MAXT/MINB: launch bounds of the variant (1024x1 leaves 64 registers per thread, 512x1 and 256x2 leave 128)
template <int BS, int MAXT = PCG_TPB, int MINB = 1>
__global__ void __launch_bounds__(MAXT, MINB) k_pcg(PcgArgs A) {
  constexpr int BB = BS * BS;
  __shared__ double red[PCG_TPB / 32];
  __shared__ double gj_rows[GJB * GJ_LDR];
  __shared__ double gj_pi[GJB * GJ_LDP];
  __shared__ double gj_vr[2][GJB], gj_vc[2][GJB];
  __shared__ int gj_bad;
  const int bdim = blockDim.x;  // 256 (small systems: spread over more SMs) or PCG_TPB
  const int lane = threadIdx.x & 31;
  const int gw = (blockIdx.x * bdim + threadIdx.x) >> 5;
  const int nw = (gridDim.x * bdim) >> 5;
  const int G = gridDim.x;
  const long long gtid = (long long)blockIdx.x * bdim + threadIdx.x, gthreads = (long long)gridDim.x * bdim;
  unsigned target = 0;
  double* part0 = A.partials;
  double* part1 = A.partials + G;
  double* part2 = A.partials + 2 * G;
  const int nC = A.agg > 0 ? BS * A.nc : 0;
  bool coarse = nC > 0;
  const double* Ainv = nullptr;

  // ---- coarse level set-up: Ac = P^T S P, then Ac^-1 by ping-pong Gauss-Jordan -------------------------------------
  if (coarse && A.coarse_mode == 2) {
    Ainv = coarse_inverse(A.Ac, nC);
    for (long long i = gtid; i < 2ll * nC; i += gthreads) A.rc[i] = 0.0;
    grid_barrier(A.bar, target);
  } else if (coarse) {
    double* A0 = A.Ac;
    double* A1 = A.Ac + (size_t)nC * nC;
    for (long long i = gtid; i < (long long)nC * nC; i += gthreads) A0[i] = 0.0;
    for (long long i = gtid; i < 2ll * nC; i += gthreads) A.rc[i] = 0.0;
    grid_barrier(A.bar, target);
    // assembly: the warp walks one block row, accumulates the blocks of one aggregate column in registers, flushes with
    // red.add when the aggregate changes (columns are sorted, so a row flushes once per touched aggregate)
    if (A.prolong) {
      // piecewise-linear P: block S_ab feeds the coarse columns lo(b) and lo(b)+1.  Columns are sorted, so lo(b) never decreases
      // along the row: keep the running sums for nodes `cur` (L) and `cur + 1` (H), shift H -> L when lo(b) advances by one, and
      // flush a finished column sum T_J = sum_b w_J(b) S_ab into the coarse rows of both parents of a, weighted.
      for (int a = gw; a < A.n; a += nw) {
        const CoarseParents pa = coarse_parents(a, A.agg, A.nc, 1);
        double l0 = 0.0, l1 = 0.0, h0 = 0.0, h1 = 0.0;
        int cur = -1;
        auto flush = [&](int J, double t0, double t1) {
          if (J < 0 || J >= A.nc) return;
          if (lane < BB) {
            const size_t c = (size_t)J * BS + lane % BS;
            atomicAdd(A0 + (size_t)(pa.lo * BS + lane / BS) * nC + c, pa.w0 * t0);
            if (pa.w1 != 0.0) atomicAdd(A0 + (size_t)(pa.hi * BS + lane / BS) * nC + c, pa.w1 * t0);
          }
          if (lane + 32 < BB) {
            const size_t c = (size_t)J * BS + (lane + 32) % BS;
            atomicAdd(A0 + (size_t)(pa.lo * BS + (lane + 32) / BS) * nC + c, pa.w0 * t1);
            if (pa.w1 != 0.0) atomicAdd(A0 + (size_t)(pa.hi * BS + (lane + 32) / BS) * nC + c, pa.w1 * t1);
          }
        };
        const int beg = A.rowptr[a], end = A.rowptr[a + 1];
        for (int j = beg; j < end; j++) {
          const CoarseParents pb = coarse_parents(A.col[j], A.agg, A.nc, 1);
          if (pb.lo != cur) {
            if (cur >= 0) {
              flush(cur, l0, l1);
              if (pb.lo == cur + 1) { l0 = h0; l1 = h1; }
              else { flush(cur + 1, h0, h1); l0 = 0.0; l1 = 0.0; }
            }
            h0 = 0.0; h1 = 0.0;
            cur = pb.lo;
          }
          const double* v = A.val + (size_t)j * BB;
          const double s0 = lane < BB ? __ldg(v + lane) : 0.0;
          const double s1 = lane + 32 < BB ? __ldg(v + lane + 32) : 0.0;
          l0 += pb.w0 * s0; l1 += pb.w0 * s1;
          h0 += pb.w1 * s0; h1 += pb.w1 * s1;
        }
        if (cur >= 0) { flush(cur, l0, l1); flush(cur + 1, h0, h1); }
      }
    } else
    for (int a = gw; a < A.n; a += nw) {
      const int ra = a / A.agg;
      double acc0 = 0.0, acc1 = 0.0;
      int cur = -1;
      const int beg = A.rowptr[a], end = A.rowptr[a + 1];
      for (int j = beg; j <= end; j++) {
        const int cb = j < end ? A.col[j] / A.agg : -2;
        if (cb != cur) {
          if (cur >= 0) {
            if (lane < BB) atomicAdd(A0 + (size_t)(ra * BS + lane / BS) * nC + cur * BS + lane % BS, acc0);
            if (lane + 32 < BB) atomicAdd(A0 + (size_t)(ra * BS + (lane + 32) / BS) * nC + cur * BS + (lane + 32) % BS, acc1);
          }
          cur = cb; acc0 = 0.0; acc1 = 0.0;
        }
        if (j < end) {
          const double* v = A.val + (size_t)j * BB;
          if (lane < BB) acc0 += __ldg(v + lane);
          if (lane + 32 < BB) acc1 += __ldg(v + lane + 32);
        }
      }
    }
    grid_barrier(A.bar, target);
    if (A.coarse_mode == 3) return;  // assembly only (ccm_ba_debug_coarse): A0 holds P^T S P
    // Block Gauss-Jordan without pivoting (the matrix is SPD, so every pivot block is too): sweep t eliminates GJB pivots at
    // once (rank-GJB update), reads buffer t&1 and writes buffer (t+1)&1.  With A = [[P, R], [C, D]] the sweep writes
    // [[P^-1, P^-1 R], [-C P^-1, D - C P^-1 R]], one formula for every entry:
    //   dst[i][j] = base[i][j] + H[i] . Rr[:, j],   H[i] = X[i] P^-1,
    //   X[i] = -src[i][piv] (pivot rows: the unit vector e_{i-k0}),  Rr[l][j] = src[k0+l][j] (pivot columns: delta(l, j-k0)),
    //   base = src off the pivot rows and columns, 0 on them.
    // Both products run as mma.m8n8k4.f64 tiles, one warp per slab of 8 rows.  Work split of one sweep: the matrix is cut into
    // column chunks of GJ_CW; a CTA stages Rr of its chunk in shared memory and its warps stream slabs through it (H is formed
    // again per chunk: GJB / GJ_CW more flops, no extra barrier); the L2 traffic per sweep is about one read + one write of
    // the matrix.
    bool bad = false;
    int sweep = 0;
    const int wid = threadIdx.x >> 5, wpc = bdim >> 5;
    const int qr = lane >> 2, qc = lane & 3;  // mma fragment coordinates (see dmma_884)
    const int nch = (nC + GJ_CW - 1) / GJ_CW;
    const int rgs = G / nch > 0 ? G / nch : 1;  // CTAs sharing one column chunk
    const int nslab = (nC + 7) >> 3;
    constexpr int PE = (GJB * GJB + MAXT - 1) / MAXT;  // pivot-block entries per thread (every launch uses MAXT threads)
    for (int k0 = 0; k0 < nC; k0 += GJB, sweep++) {
      const int kb = nC - k0 < GJB ? nC - k0 : GJB;
      const double* src = (sweep & 1) ? A1 : A0;
      double* dst = (sweep & 1) ? A0 : A1;
      // P^-1 (identity past kb) by Gauss-Jordan, identical in every CTA: each thread keeps its entries in registers, the
      // pivot row and column of the next step go through the ping-pong vectors gj_vr / gj_vc -> one __syncthreads per pivot
      double e[PE];
#pragma unroll
      for (int u = 0; u < PE; u++) {
        const int t = threadIdx.x + u * bdim, r2 = t / GJB, c2 = t % GJB;
        e[u] = 0.0;
        if (t < GJB * GJB) {
          e[u] = (r2 < kb && c2 < kb) ? __ldcg(src + (size_t)(k0 + r2) * nC + k0 + c2) : (r2 == c2 ? 1.0 : 0.0);
          if (r2 == 0) gj_vr[0][c2] = e[u];
          if (c2 == 0) gj_vc[0][r2] = e[u];
        }
      }
      if (threadIdx.x == 0) gj_bad = 0;
      __syncthreads();
      for (int q = 0; q < kb; q++) {  // the identity past kb has unit pivots and changes nothing
        const double* vr = gj_vr[q & 1];
        const double* vc = gj_vc[q & 1];
        const double piv = vr[q];
        const double ip = 1.0 / piv;
#pragma unroll
        for (int u = 0; u < PE; u++) {
          const int t = threadIdx.x + u * bdim, r2 = t / GJB, c2 = t % GJB;
          if (t < GJB * GJB) {
            const double prq = vc[r2], pqc = vr[c2];
            e[u] = r2 == q ? (c2 == q ? ip : pqc * ip) : (c2 == q ? -prq * ip : e[u] - prq * (pqc * ip));
            if (r2 == q + 1) gj_vr[(q + 1) & 1][c2] = e[u];
            if (c2 == q + 1) gj_vc[(q + 1) & 1][r2] = e[u];
          }
        }
        if (threadIdx.x == 0 && (!(piv > 0.0) || !isfinite(piv))) gj_bad = 1;
        __syncthreads();
      }
      if (gj_bad) { bad = true; break; }  // uniform over the grid: every CTA inverted the same pivot block
#pragma unroll
      for (int u = 0; u < PE; u++) {
        const int t = threadIdx.x + u * bdim;
        if (t < GJB * GJB) gj_pi[(t / GJB) * GJ_LDP + t % GJB] = e[u];
      }
      for (int item = blockIdx.x; item < nch * rgs; item += G) {
        const int c0 = (item % nch) * GJ_CW, rg = item / nch;
        for (int t = threadIdx.x; t < GJB * GJ_CW; t += bdim) {
          const int l = t / GJ_CW, j = c0 + t % GJ_CW;
          gj_rows[l * GJ_LDR + t % GJ_CW] = (l >= kb || j >= nC) ? 0.0
                                            : (j >= k0 && j < k0 + kb) ? (j - k0 == l ? 1.0 : 0.0)
                                                                       : __ldcg(src + (size_t)(k0 + l) * nC + j);
        }
        __syncthreads();  // gj_rows and gj_pi complete
        for (int s = rg * wpc + wid; s < nslab; s += rgs * wpc) {
          const int i0 = s * 8, ia = i0 + qr;  // this lane's row in the A and C fragments
          const bool pslab = i0 >= k0 && i0 < k0 + GJB;  // k0 and i0 are multiples of 8: a slab is all pivot rows or none
          double a[GJB / 4];  // X[ia][4 ks + qc]
#pragma unroll
          for (int ks = 0; ks < GJB / 4; ks++) {
            const int m = 4 * ks + qc;
            a[ks] = pslab ? (ia - k0 == m ? 1.0 : 0.0) : (ia < nC && m < kb) ? -__ldcg(src + (size_t)ia * nC + k0 + m) : 0.0;
          }
          double h[GJB / 8][2];  // H = X P^-1, C layout
#pragma unroll
          for (int nt = 0; nt < GJB / 8; nt++) h[nt][0] = h[nt][1] = 0.0;
#pragma unroll
          for (int ks = 0; ks < GJB / 4; ks++)
#pragma unroll
            for (int nt = 0; nt < GJB / 8; nt++) dmma_884(h[nt][0], h[nt][1], a[ks], gj_pi[(4 * ks + qc) * GJ_LDP + 8 * nt + qr]);
          // C layout -> A layout: A[qr][4 ks + qc] sits in lane (qr, (4 (ks & 1) + qc) / 2), element qc & 1 of tile ks / 2
#pragma unroll
          for (int ks = 0; ks < GJB / 4; ks++) {
            const int sl = (lane & ~3) | ((4 * (ks & 1) + qc) >> 1);
            const double v0 = __shfl_sync(0xffffffffu, h[ks >> 1][0], sl);
            const double v1 = __shfl_sync(0xffffffffu, h[ks >> 1][1], sl);
            a[ks] = (qc & 1) ? v1 : v0;
          }
          const bool rowok = ia < nC;
          const double* srow = src + (size_t)ia * nC;
          double* drow = dst + (size_t)ia * nC;
          constexpr int NT = 4;  // column tiles in flight: independent accumulator chains, their base loads issued together
          for (int n0 = 0; n0 < GJ_CW / 8 && c0 + 8 * n0 < nC; n0 += NT) {
            double d[NT][2];
#pragma unroll
            for (int w = 0; w < NT; w++) {
              const int j = c0 + 8 * (n0 + w) + 2 * qc;
#pragma unroll
              for (int x = 0; x < 2; x++) {
                const int jx = j + x;
                d[w][x] = (!pslab && rowok && jx < nC && !(jx >= k0 && jx < k0 + kb)) ? __ldcg(srow + jx) : 0.0;
              }
            }
#pragma unroll
            for (int ks = 0; ks < GJB / 4; ks++)
#pragma unroll
              for (int w = 0; w < NT; w++)
                dmma_884(d[w][0], d[w][1], a[ks], gj_rows[(4 * ks + qc) * GJ_LDR + 8 * (n0 + w) + qr]);
            if (rowok) {
#pragma unroll
              for (int w = 0; w < NT; w++) {
                const int j = c0 + 8 * (n0 + w) + 2 * qc;
                if (j < nC) drow[j] = d[w][0];
                if (j + 1 < nC) drow[j + 1] = d[w][1];
              }
            }
          }
        }
        __syncthreads();  // readers of gj_rows are done before the next item restages it
      }
      grid_barrier(A.bar, target);
    }
    if (bad) coarse = false;
    Ainv = coarse_inverse(A.Ac, nC);
  }

  // z = Minv r for the rows of this warp; with the coarse level: += (P yc)[row]
  auto precond_rows = [&](double& acc_rz, double& acc_rr) {
    for (int a = gw; a < A.n; a += nw) {
      double rv = 0.0;
      if (lane < BS) rv = A.r[(size_t)a * BS + lane];
      double r6[BS];
#pragma unroll
      for (int k = 0; k < BS; k++) r6[k] = __shfl_sync(0xffffffffu, rv, k);
      if (lane < BS) {
        const double* M = A.Minv + (size_t)a * BB + lane * BS;
        double zv = 0.0;
#pragma unroll
        for (int k = 0; k < BS; k++) zv += M[k] * r6[k];
        if (coarse) {
          if (A.prolong) {
            const CoarseParents pa = coarse_parents(a, A.agg, A.nc, 1);
            zv += pa.w0 * __ldcg(A.yc + (size_t)pa.lo * BS + lane) + pa.w1 * __ldcg(A.yc + (size_t)pa.hi * BS + lane);
          } else {
            zv += __ldcg(A.yc + (size_t)(a / A.agg) * BS + lane);
          }
        }
        A.z[(size_t)a * BS + lane] = zv;
        acc_rz += rv * zv;
        acc_rr += rv * rv;
      }
    }
  };
  // rc[buf] += P^T r over the rows of this warp (red.add), then (after a barrier) yc = Ainv rc[buf]
  auto restrict_rows = [&](int buf) {
    if (A.prolong) {
      for (int a = gw; a < A.n; a += nw)
        if (lane < BS) {
          const CoarseParents pa = coarse_parents(a, A.agg, A.nc, 1);
          const double rv = A.r[(size_t)a * BS + lane];
          atomicAdd(A.rc + (size_t)buf * nC + (size_t)pa.lo * BS + lane, pa.w0 * rv);
          if (pa.w1 != 0.0) atomicAdd(A.rc + (size_t)buf * nC + (size_t)pa.hi * BS + lane, pa.w1 * rv);
        }
      return;
    }
    for (int a = gw; a < A.n; a += nw)
      if (lane < BS) atomicAdd(A.rc + (size_t)buf * nC + (size_t)(a / A.agg) * BS + lane, A.r[(size_t)a * BS + lane]);
  };
  auto coarse_solve = [&](int buf) {
    const double* rcv = A.rc + (size_t)buf * nC;
    for (int i = gw; i < nC; i += nw) {
      double s = 0.0;
      for (int j = lane; j < nC; j += 32) s += __ldcg(Ainv + (size_t)i * nC + j) * __ldcg(rcv + j);
      s = warp_sum(s);
      if (lane == 0) A.yc[i] = s;
    }
    // clear the other buffer for the next iteration (nobody reads or writes it in this phase)
    if (blockIdx.x == 0) for (int i = threadIdx.x; i < nC; i += bdim) A.rc[(size_t)(buf ^ 1) * nC + i] = 0.0;
  };

  const bool prof_on = A.prof != nullptr && blockIdx.x == 0 && threadIdx.x == 0;
  long long tprev = clock64();
  auto lap = [&](int slot) { if (prof_on) { const long long t = clock64(); A.prof[slot] += t - tprev; tprev = t; } };
  lap(0);
  // ---- x = 0, r = b ----------------------------------------------------------------------------------------------------
  for (int a = gw; a < A.n; a += nw)
    if (lane < BS) {
      A.x[(size_t)a * BS + lane] = 0.0;
      A.r[(size_t)a * BS + lane] = A.b[(size_t)a * BS + lane];
      A.p[(size_t)a * BS + lane] = 0.0;  // p_old of the first iteration (beta = 0)
    }
  int buf = 0;
  if (coarse) {
    restrict_rows(buf);
    grid_barrier(A.bar, target);
    coarse_solve(buf);
    grid_barrier(A.bar, target);
    buf ^= 1;
  }
  double acc_rz = 0.0, acc_bb = 0.0;
  precond_rows(acc_rz, acc_bb);
  {
    const double t0 = block_sum(acc_rz, red);
    const double t1 = block_sum(acc_bb, red);
    if (threadIdx.x == 0) { part0[blockIdx.x] = t0; part1[blockIdx.x] = t1; }
  }
  grid_barrier(A.bar, target);
  double rz = sum_partials_dev(part0, G);
  const double bb = sum_partials_dev(part1, G);
  const double stop2 = A.tol * A.tol * bb;
  int it = 0, flag = 1;
  double rr = bb;
  if (!(bb > 0.0)) {
    flag = 0;
  } else {
    // The direction update p = z + beta p_old is folded into the product: every reader forms the entries of p it needs from
    // z and p_old with the same fma the row owner uses (bit-identical), the owner stores its rows into the other p buffer.
    // This removes the p-update phase and its grid barrier (4 barriers per iteration).
    const size_t nv = (size_t)A.n * BS;
    double beta = 0.0;
    int pc = 0;
    for (it = 0; it < A.max_iter; it++, pc ^= 1) {
      const double* pold = A.p + (size_t)pc * nv;
      double* pnew = A.p + (size_t)(pc ^ 1) * nv;
      // q = S p ; pq = p.q
      double acc_pq = 0.0;
      for (int a = gw; a < A.n; a += nw) {
        double y[BS];
#pragma unroll
        for (int k = 0; k < BS; k++) y[k] = 0.0;
        const int beg = A.rowptr[a], end = A.rowptr[a + 1];
        for (int j = beg + lane; j < end; j += 32) {
          const double* v = A.val + (size_t)j * BB;
          const size_t cj = (size_t)A.col[j] * BS;
          double pv[BS];
#pragma unroll
          for (int k = 0; k < BS; k++) pv[k] = fma(beta, __ldcg(pold + cj + k), __ldcg(A.z + cj + k));
          if constexpr (BS % 2 == 0) {
            const double2* v2 = reinterpret_cast<const double2*>(v);
#pragma unroll
            for (int rI = 0; rI < BS; rI++)
#pragma unroll
              for (int c = 0; c < BS / 2; c++) {
                const double2 t = __ldg(v2 + rI * (BS / 2) + c);  // (bypassing L1 here measured 18 % slower: neighbouring loads share lines)
                y[rI] += t.x * pv[2 * c] + t.y * pv[2 * c + 1];
              }
          } else {
#pragma unroll
            for (int rI = 0; rI < BS; rI++)
#pragma unroll
              for (int c = 0; c < BS; c++) y[rI] += __ldg(v + rI * BS + c) * pv[c];
          }
        }
#pragma unroll
        for (int k = 0; k < BS; k++) y[k] = warp_sum(y[k]);
        if (lane < BS) {
          double yl = y[0];
#pragma unroll
          for (int k = 1; k < BS; k++) yl = lane == k ? y[k] : yl;
          const double pn = fma(beta, __ldcg(pold + (size_t)a * BS + lane), __ldcg(A.z + (size_t)a * BS + lane));
          pnew[(size_t)a * BS + lane] = pn;
          A.q[(size_t)a * BS + lane] = yl;
          acc_pq += yl * pn;
        }
      }
      {
        const double t0 = block_sum(acc_pq, red);
        if (threadIdx.x == 0) part0[blockIdx.x] = t0;
      }
      grid_barrier(A.bar, target);
      lap(1);
      const double pq = sum_partials_dev(part0, G);
      if (!(pq > 0.0) || !isfinite(pq)) { flag = 2; break; }
      const double alpha = rz / pq;
      // x += alpha p ; r -= alpha q   (rows owned by this warp)
      for (int a = gw; a < A.n; a += nw)
        if (lane < BS) {
          A.x[(size_t)a * BS + lane] += alpha * pnew[(size_t)a * BS + lane];
          A.r[(size_t)a * BS + lane] -= alpha * A.q[(size_t)a * BS + lane];
        }
      if (coarse) {
        restrict_rows(buf);
        grid_barrier(A.bar, target);
        lap(2);
        coarse_solve(buf);
        grid_barrier(A.bar, target);
        lap(3);
        buf ^= 1;
      }
      double acc_rz2 = 0.0, acc_rr = 0.0;
      precond_rows(acc_rz2, acc_rr);
      {
        const double t0 = block_sum(acc_rz2, red);
        const double t1 = block_sum(acc_rr, red);
        if (threadIdx.x == 0) { part1[blockIdx.x] = t0; part2[blockIdx.x] = t1; }
      }
      grid_barrier(A.bar, target);
      lap(4);
      const double rz_new = sum_partials_dev(part1, G);
      rr = sum_partials_dev(part2, G);
      if (rr <= stop2) { flag = 0; it++; break; }
      beta = rz_new / rz;
      rz = rz_new;
    }
  }
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    A.status[0] = (double)it;
    A.status[1] = bb > 0.0 ? sqrt(rr / bb) : 0.0;
    A.status[2] = (double)flag;
    A.status[3] = coarse ? (double)nC : 0.0;
  }
}

// aggregate size for n block rows so that at most nc_max aggregates exist
inline void pcg_coarse_shape(int n, int nc_max, int* agg, int* nc) {
  if (nc_max <= 0 || n <= 0) { *agg = 0; *nc = 0; return; }
  *agg = (n + nc_max - 1) / nc_max;
  if (*agg < 1) *agg = 1;
  *nc = (n + *agg - 1) / *agg;
}

}  // namespace ccm

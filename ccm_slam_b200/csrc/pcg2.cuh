// pcg2.cuh — the preconditioned conjugate-gradient solve of the reduced camera system, second generation (BS = 6).
//
// Replaces g2o's LinearSolverEigen::solve (G/solvers/linear_solver_eigen.h:106-133) like k_pcg (pcg.cuh) does, with the same
// mathematics — M^-1 = blockdiag(S)^-1 + P (P^T S P)^-1 P^T, the coarse inverse built by k_pcg's set-up phase (launched with
// max_iter = 0) — but one kernel for one GPU and for the block rows distributed over the ranks of an NVLink node, and shaped
// around what bounds it:
//
//  * S is streamed, never gathered.  Block rows are cut into ITEMS of <= 16 consecutive blocks (<= 4608 contiguous bytes of
//    s_val).  Every CTA owns a contiguous run of rows (balanced by item count), every warp a contiguous run of the CTA's items,
//    and pulls them through its own two-stage shared-memory ring with cp.async.bulk (TMA 1-D copies) completing on an mbarrier;
//    the copy of item m + 2 is issued as soon as item m has been consumed, and the ring is cyclic over the warp's items, so the
//    first two items of the NEXT product are already in flight while the other phases of the iteration run (S is constant
//    during a solve).  A lane pair multiplies one 6x6 block (18 doubles per lane, conflict-free 16-byte shared loads).  Inside
//    the CTA's own rows an upper block is applied twice from one copy (S_ab p_b and S_ab^T p_a) and its mirror is not streamed
//    (pcg2_plan, below); the transposed products gather in per-warp shared-memory slabs that complete the rows after the product.
//  * the search direction p = z + beta p_old of the CTA's row window (own rows +- halo, <= 512 rows) is formed once per
//    product in shared memory; only columns outside the window (loop closures, merged maps) are gathered from L2.
//  * three grid-wide synchronisations per iteration instead of four: the restricted residual follows the recurrence
//    rc -= alpha P^T q, and P^T q is accumulated while q = S p is produced (phase 1).  Phase 2 (alpha known): x, r update of the
//    own rows, rc update (every CTA keeps rc in shared memory), the CTA's slice of the dense coarse product yc = Ainv rc.
//    Phase 3: z = Minv r + P yc, r.z, r.r.
//  * N ranks: rank k owns the block rows [r0, r1) (S is present on every rank after the all-reduce of the Schur blocks).
//    Synchronisations A (after phase 1) and B (after phase 3) stay local grid barriers; what crosses NVLink rides next to them:
//    once the local CTAs have arrived, CTA 0 sums the CTA partials in a fixed order and stores them — and after phase 1 its
//    P^T q partial — straight into every peer's exchange window (cudaIpc-mapped) as 16-byte low-latency packets
//    {lo32, epoch, hi32, epoch}: each 8-byte half is delivered atomically, so a reader that finds the epoch of this
//    synchronisation in both halves has the value — one NVLink traversal, no system-scope fence, no separate flag
//    (flag words + fence.sys measured slower).  z is not pushed at all: an owner writes its rows into
//    its own window, and a peer that needs a row of another rank (band rows next to the cut, loop closures) loads it over
//    NVLink after the owner's B packet has arrived.  Every rank forms the same scalars from the same numbers in rank order and
//    takes the same branches: no broadcast, no host round trip, no NCCL launch inside the solve.  Every spin carries a
//    clock64 time-out that raises a node-wide abort word (status 3) instead of hanging the GPU.
//
// Exchange-window hazards: everything in a window is double-buffered by iteration parity; a region written in iteration i is
// next written in iteration i + 2, and a rank gets there only through two node-wide barriers that every rank joins after it
// finished reading iteration i.
#pragma once
#include <stdint.h>

#include <algorithm>
#include <vector>

#include "pcg.cuh"

namespace ccm {

constexpr int P2_TPB = 512;
constexpr int P2_W = P2_TPB / 32;
constexpr int P2_ITEM_BLOCKS = 16;                    // blocks per item: one lane pair per block
constexpr int P2_ITEM_DOUBLES = P2_ITEM_BLOCKS * 36;  // 576 doubles = 4608 bytes
constexpr int P2_REC = 20;                            // ints per item record: first block, #blocks, row, flags, col[16]
constexpr int P2_WIN_ROWS = 512;                      // rows of the direction vector cached in shared memory
constexpr int P2_MAX_NC = 2304;                       // coarse unknowns the shared-memory copy of rc holds (384 nodes x 6)
constexpr int P2_SLAB_ROWS = 48;                      // rows of a warp's transposed-product slab (what is left of 227 KB)
constexpr int P2_NO_SLAB = -(1 << 30);                // slab_lo of a warp without transposed blocks
constexpr size_t P2_SMEM_BYTES = (size_t)(P2_W * 2 * P2_ITEM_DOUBLES + P2_MAX_NC + P2_WIN_ROWS * 6 + P2_W * 2 * 6 +
                                          P2_W * P2_SLAB_ROWS * 6) * sizeof(double) +
                                 (size_t)(P2_W * 2 + P2_W) * sizeof(int) + (size_t)(P2_W * 2) * sizeof(uint64_t);

struct Pcg2Args {
  int n;                       // block rows of S
  const double* val;           // block-CSR values (all rows)
  const int* items;            // item records of the OWN rows, P2_REC ints each, row-major order (pcg2_plan)
  const int* cta_row;          // [grid + 1] first own row of every CTA (absolute row indices), cta_row[grid] = r1
  const int* cta_item;         // [grid + 1] first item of every CTA
  const int* slab_lo;          // [grid * P2_W] first row of every warp's transposed-product slab, P2_NO_SLAB if it has none
  const double* Minv; const double* b;
  double *x, *r, *q, *p;       // p: 2 * n * 6
  double* partials;            // 3 * grid
  unsigned* bar;               // [0] arrival counter, [1] release generation; zeroed before launch
  double tol; int max_iter;
  double* status;              // [iters, relres, flag (0 converged, 1 max_iter, 2 breakdown, 3 peer time-out), coarse unknowns used]
  int agg, nc, prolong;
  const double* Ainv;          // (6 nc)^2, valid iff status[3] > 0 (left there by k_pcg's set-up launch or by the previous solve)
  double* yc;                  // 2 * 6 nc
  double* tpart;               // 2 * 6 nc, zeroed before launch: this rank's P^T q (parity-buffered)
  int rank, nranks, r0, r1;
  char* const* win;            // [nranks] exchange windows as mapped in this process; win[rank] is local
  size_t off_z, off_x, off_flags, off_ctl;
  size_t off_lls, off_llt;     // low-latency packets: scalars [2][nranks][4], P^T q [2][nranks][6 nc], 16 bytes each
  const int* rank_row;         // [nranks + 1] first block row of every rank
  const unsigned char* need;   // [n] 1 where some block of this rank's rows sits in that block column (the rows of p / z this rank reads)
  unsigned ll_epoch0;          // packets of this launch carry ll_epoch0 + 2 (it + 1) + {0: A, 1: B}; never 0
  unsigned long long epoch0;   // node barrier epochs of this launch start here (flags only ever grow)
  long long timeout_cycles;
  long long* prof;             // optional 8 cycle counters (CTA 0): [0] set-up, [1] product, [2] coarse, [3] precondition
};

__device__ __forceinline__ uint32_t p2_smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void p2_mbar_init(uint64_t* bar, int count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(p2_smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void p2_mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(p2_smem_u32(bar)), "r"(bytes) : "memory");
}
// S is read once per product and evicted first, so that the coarse inverse and the vectors, read every iteration, stay in L2
__device__ __forceinline__ uint64_t p2_evict_first_policy() {
  uint64_t pol;
  asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(pol));
  return pol;
}
__device__ __forceinline__ void p2_bulk_g2s(void* dst, const void* src, uint32_t bytes, uint64_t* bar, uint64_t pol) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], %4;" ::"r"(
                   p2_smem_u32(dst)),
               "l"(src), "r"(bytes), "r"(p2_smem_u32(bar)), "l"(pol)
               : "memory");
}
__device__ __forceinline__ bool p2_mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n .reg .pred p;\n mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n selp.u32 %0, 1, 0, p;\n}"
      : "=r"(ok)
      : "r"(p2_smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
// bounded wait: a copy that never lands (a bug, not a run-time condition) must end the kernel with an error, not hang the GPU
__device__ __forceinline__ void p2_mbar_wait(uint64_t* bar, uint32_t parity, long long timeout_cycles) {
  if (p2_mbar_try_wait(bar, parity)) return;
  const long long t0 = clock64();
  while (!p2_mbar_try_wait(bar, parity))
    if (clock64() - t0 > timeout_cycles) __trap();
}
__device__ __forceinline__ unsigned p2_ld_acquire_gpu(const unsigned* p) {
  unsigned v;
  asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void p2_st_release_gpu(unsigned* p, unsigned v) {
  asm volatile("st.release.gpu.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ unsigned long long p2_ld_acquire_sys(const unsigned long long* p) {
  unsigned long long v;
  asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void p2_st_release_sys(unsigned long long* p, unsigned long long v) {
  asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}

// low-latency packet: a double as two (32-bit half, 32-bit epoch) pairs; NVLink delivers every aligned 8-byte unit atomically
__device__ __forceinline__ void p2_ll_store(void* slot, double v, unsigned flag) {
  const unsigned long long b = (unsigned long long)__double_as_longlong(v);
  asm volatile("st.volatile.global.v4.u32 [%0], {%1, %2, %3, %4};" ::"l"(slot), "r"((unsigned)b), "r"(flag), "r"((unsigned)(b >> 32)), "r"(flag)
               : "memory");
}
__device__ __forceinline__ bool p2_ll_try(const void* slot, unsigned flag, double& v) {
  unsigned a, f1, b, f2;
  asm volatile("ld.volatile.global.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(a), "=r"(f1), "=r"(b), "=r"(f2) : "l"(slot) : "memory");
  if (f1 != flag || f2 != flag) return false;
  v = __longlong_as_double((long long)(((unsigned long long)b << 32) | a));
  return true;
}
__device__ __forceinline__ double p2_ld_volatile(const double* p) {
  double v;
  asm volatile("ld.volatile.global.f64 %0, [%1];" : "=d"(v) : "l"(p) : "memory");
  return v;
}

// Grid-wide (cross = false) or node-wide (cross = true and nranks > 1) barrier.  Every CTA arrives at a counter; CTA 0 waits for
// the arrivals, runs publish() with all its threads (partials -> exchange windows), meets the peers' CTA 0s at the flag words
// when the barrier is node-wide, and releases the local CTAs through a generation word.  Returns false after a time-out / abort.
// remote: the CTAs stored into peer windows since the last barrier (their arrival then needs a system-scope fence, which waits for
// the NVLink write acknowledgements; a GPU-scope fence otherwise).
template <typename F>
__device__ __forceinline__ bool p2_barrier(const Pcg2Args& A, unsigned& gen, unsigned long long& epoch, bool cross, bool remote, int* s_ok,
                                           F&& publish) {
  __syncthreads();
  gen += 1;
  const bool multi = A.nranks > 1;
  const bool node = cross && multi;
  if (node) epoch += 1;
  volatile unsigned* ctl = reinterpret_cast<volatile unsigned*>(A.win[A.rank] + A.off_ctl);
  if (!multi && !node) {
    // one GPU: nothing to publish between arrival and release, so the LAST arriver releases the others (one hop less than routing
    // the release through CTA 0)
    if (threadIdx.x == 0) {
      int ok = 1;
      __threadfence();
      if (atomicAdd(A.bar, 1u) + 1u == gen * gridDim.x) {
        p2_st_release_gpu(A.bar + 1, gen);
      } else {
        const long long t0 = clock64();
        unsigned g;
        while ((g = p2_ld_acquire_gpu(A.bar + 1)) < gen)
          if (clock64() - t0 > A.timeout_cycles) { ok = 0; break; }
        if (g == 0xFFFFFFFFu) ok = 0;
      }
      *s_ok = ok;
    }
    __syncthreads();
    return *s_ok != 0;
  }
  if (threadIdx.x == 0) {
    if (multi && remote) __threadfence_system(); else __threadfence();
    atomicAdd(A.bar, 1u);
  }
  if (blockIdx.x == 0) {
    if (threadIdx.x == 0) {
      int ok = 1;
      const long long t0 = clock64();
      const unsigned target = gen * gridDim.x;
      while (p2_ld_acquire_gpu(A.bar) < target)
        if (*ctl || clock64() - t0 > A.timeout_cycles) { ok = 0; break; }
      *s_ok = ok;
    }
    __syncthreads();
    if (*s_ok) publish();
    if (node) __threadfence_system(); else __threadfence();
    __syncthreads();
    if (threadIdx.x == 0) {
      int ok = *s_ok;
      if (node && ok) {
        const long long t0 = clock64();
        for (int k = 0; k < A.nranks; k++)
          p2_st_release_sys(reinterpret_cast<unsigned long long*>(A.win[k] + A.off_flags) + A.rank, epoch);
        const unsigned long long* mine = reinterpret_cast<const unsigned long long*>(A.win[A.rank] + A.off_flags);
        for (int k = 0; k < A.nranks && ok; k++)
          while (p2_ld_acquire_sys(mine + k) < epoch)
            if (*ctl || clock64() - t0 > A.timeout_cycles) { ok = 0; break; }
      }
      if (!ok) {  // tell every rank and every local CTA to leave
        for (int k = 0; k < A.nranks; k++) *reinterpret_cast<volatile unsigned*>(A.win[k] + A.off_ctl) = 1u;
        __threadfence_system();
      }
      *s_ok = ok;
      p2_st_release_gpu(A.bar + 1, ok ? gen : 0xFFFFFFFFu);
    }
  } else if (threadIdx.x == 0) {
    int ok = 1;
    const long long t0 = clock64();
    unsigned g;
    while ((g = p2_ld_acquire_gpu(A.bar + 1)) < gen)
      if (*ctl || clock64() - t0 > A.timeout_cycles) { ok = 0; break; }
    if (g == 0xFFFFFFFFu || *ctl) ok = 0;
    *s_ok = ok;
  }
  __syncthreads();
  return *s_ok != 0;
}

// running sums of P^T v over consecutive rows: rows arrive in increasing order, so the lower parent never decreases; `l` collects
// node cur, `h` node cur + 1; a finished node is flushed with one red.add per component (lanes 0..5 hold the components)
struct P2CoarseAcc { int cur; double l, h; };
__device__ __forceinline__ void p2_cflush(const Pcg2Args& A, double* tp, int J, double v, int lane) {
  if (J >= 0 && J < A.nc && lane < 6 && v != 0.0) atomicAdd(tp + (size_t)J * 6 + lane, v);
}
__device__ __forceinline__ void p2_cadd(const Pcg2Args& A, P2CoarseAcc& s, double* tp, int a, double v, int lane) {
  const CoarseParents pa = coarse_parents(a, A.agg, A.nc, A.prolong);
  if (pa.lo != s.cur) {
    if (s.cur >= 0) {
      p2_cflush(A, tp, s.cur, s.l, lane);
      if (pa.lo == s.cur + 1) s.l = s.h;
      else { p2_cflush(A, tp, s.cur + 1, s.h, lane); s.l = 0.0; }
    } else s.l = 0.0;
    s.h = 0.0;
    s.cur = pa.lo;
  }
  s.l += pa.w0 * v;
  s.h += pa.w1 * v;
}

__global__ void __launch_bounds__(P2_TPB, 1) k_pcg2(Pcg2Args A) {
  constexpr int BS = 6, BB = 36;
  extern __shared__ __align__(128) unsigned char p2_smem[];
  double* sm_ring = reinterpret_cast<double*>(p2_smem);   // [W][2][576]
  double* sm_rc = sm_ring + P2_W * 2 * P2_ITEM_DOUBLES;   // [P2_MAX_NC]
  double* sm_pwin = sm_rc + P2_MAX_NC;                    // [P2_WIN_ROWS * 6]
  double* sm_bval = sm_pwin + P2_WIN_ROWS * 6;            // [W][2][6] partial rows at the ends of the warps' runs
  int* sm_brow = reinterpret_cast<int*>(sm_bval + P2_W * 2 * 6);  // [W][2]
  int* sm_bcnt = sm_brow + P2_W * 2;                      // [W]
  uint64_t* sm_mbar = reinterpret_cast<uint64_t*>(sm_bcnt + P2_W);  // [W][2]
  double* sm_slab = reinterpret_cast<double*>(sm_mbar + P2_W * 2);   // [W][P2_SLAB_ROWS * 6] transposed products S_ab^T p_a at row b
  __shared__ int s_slo[P2_W];
  __shared__ double red[P2_TPB / 32];
  __shared__ int s_ok;

  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  const int G = gridDim.x, N = A.nranks, me = A.rank;
  const size_t nv = (size_t)A.n * BS;
  const int nC = A.agg > 0 ? BS * A.nc : 0;
  unsigned gen = 0;
  unsigned long long epoch = A.epoch0;
  double* part0 = A.partials;
  double* part1 = A.partials + G;
  double* part2 = A.partials + 2 * G;
  auto zbuf = [&](int k, int par) { return reinterpret_cast<double*>(A.win[k] + A.off_z) + (size_t)par * nv; };
  // low-latency packet slots in rank k's window, written by rank src: 4 scalars ([0] p.q, [1] coarse flag, [2] r.z, [3] r.r), 6 nc of P^T q
  auto lls = [&](int k, int par, int src, int which) { return A.win[k] + A.off_lls + (((size_t)par * N + src) * 4 + which) * 16; };
  auto llt = [&](int k, int par, int src, int j) { return A.win[k] + A.off_llt + (((size_t)par * N + src) * (size_t)nC + j) * 16; };
  volatile unsigned* ctl_word = reinterpret_cast<volatile unsigned*>(A.win[me] + A.off_ctl);
  bool ll_ok = true;   // cleared when a packet did not arrive in time (a peer aborted or died): the solve ends with status 3
  auto ll_wait = [&](const void* slot, unsigned ep) -> double {
    double v = 0.0;
    if (p2_ll_try(slot, ep, v)) return v;
    const long long t0 = clock64();
    while (!p2_ll_try(slot, ep, v))
      if (*ctl_word || clock64() - t0 > A.timeout_cycles) {
        for (int k = 0; k < N; k++) *reinterpret_cast<volatile unsigned*>(A.win[k] + A.off_ctl) = 1u;
        ll_ok = false;
        return 0.0;
      }
    return v;
  };
  // owner of block row a, and z of any row: own rows from the local window, rows of another rank over NVLink from its window
  auto owner_of = [&](int a) { int k = 0; while (k + 1 < N && a >= A.rank_row[k + 1]) k++; return k; };
  auto load_z = [&](int par, size_t g) -> double {
    const int a = (int)(g / BS);
    if (N == 1 || (a >= A.r0 && a < A.r1)) return __ldcg(zbuf(me, par) + g);
    return p2_ld_volatile(zbuf(owner_of(a), par) + g);
  };
  __shared__ double sm_ll[8][4];
  // coarse unknowns [t_lo(k), t_hi(k)) that the rows of rank k restrict to (both parents of its first and last row)
  auto t_lo = [&](int k) { const int a0 = A.rank_row[k]; return a0 >= A.rank_row[k + 1] ? 0 : coarse_parents(a0, A.agg, A.nc, A.prolong).lo * BS; };
  auto t_hi = [&](int k) {
    const int a1 = A.rank_row[k + 1] - 1;
    return a1 < A.rank_row[k] ? 0 : (coarse_parents(a1, A.agg, A.nc, A.prolong).hi + 1) * BS;
  };

  // ---- this CTA's rows and items, this warp's run of items, its ring ------------------------------------------------------
  const int c0 = A.cta_row[blockIdx.x], c1 = A.cta_row[blockIdx.x + 1];
  const int it0 = A.cta_item[blockIdx.x], it1 = A.cta_item[blockIdx.x + 1];
  const int wb = it0 + (int)((long long)(it1 - it0) * wid / P2_W);
  const int we = it0 + (int)((long long)(it1 - it0) * (wid + 1) / P2_W);
  const int nwi = we - wb;
  double* ring = sm_ring + (size_t)wid * 2 * P2_ITEM_DOUBLES;
  uint64_t* mb = sm_mbar + wid * 2;
  double* slab = sm_slab + (size_t)wid * P2_SLAB_ROWS * 6;
  const int slo = A.slab_lo[(size_t)blockIdx.x * P2_W + wid];
  if (lane == 0) s_slo[wid] = slo;
  // direction window: the block columns this CTA's items touch (one pass over its records), at most P2_WIN_ROWS rows around its own rows
  __shared__ int s_cmin, s_cmax;
  if (tid == 0) { s_cmin = A.n; s_cmax = -1; }
  __syncthreads();
  {
    int cmin = A.n, cmax = -1;
    for (int k = wb; k < we; k++) {
      const int* rec = A.items + (size_t)k * P2_REC;
      const int nb = __ldg(rec + 1);
      if (lane < nb) { const int c = __ldg(rec + 4 + lane); cmin = c < cmin ? c : cmin; cmax = c > cmax ? c : cmax; }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const int a = __shfl_xor_sync(0xffffffffu, cmin, o), b = __shfl_xor_sync(0xffffffffu, cmax, o);
      cmin = a < cmin ? a : cmin; cmax = b > cmax ? b : cmax;
    }
    if (lane == 0 && cmax >= 0) { atomicMin(&s_cmin, cmin); atomicMax(&s_cmax, cmax); }
  }
  __syncthreads();
  int wlo = c0, whi = c1;
  if (c1 > c0) {
    if (c1 - c0 >= P2_WIN_ROWS) whi = c0 + P2_WIN_ROWS;
    else {
      const int halo = (P2_WIN_ROWS - (c1 - c0)) / 2;
      wlo = c0 - halo < 0 ? 0 : c0 - halo;
      whi = c1 + halo > A.n ? A.n : c1 + halo;
      if (s_cmax >= 0) {   // no wider than what the items read
        wlo = wlo < s_cmin ? (s_cmin < c0 ? s_cmin : c0) : wlo;
        whi = whi > s_cmax + 1 ? (s_cmax + 1 > c1 ? s_cmax + 1 : c1) : whi;
      }
    }
  }
  if (lane == 0) { p2_mbar_init(mb, 1); p2_mbar_init(mb + 1, 1); }
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  __syncwarp();
  // item records travel in registers: lane l < 20 holds word l.  rec0 = item of running index m, rec1 = m + 1, rec2 = m + 2.
  auto load_rec = [&](unsigned m) -> int {
    if (nwi <= 0 || lane >= P2_REC) return 0;
    return __ldg(A.items + (size_t)(wb + (int)(m % (unsigned)nwi)) * P2_REC + lane);
  };
  const uint64_t pol = p2_evict_first_policy();
  auto issue = [&](unsigned m, int rec) {  // copy of running index m into ring buffer m & 1; lane 0 issues
    const int j0 = __shfl_sync(0xffffffffu, rec, 0), nb = __shfl_sync(0xffffffffu, rec, 1);
    if (lane == 0) {
      const uint32_t bytes = (uint32_t)nb * BB * sizeof(double);
      p2_mbar_expect_tx(mb + (m & 1u), bytes);
      p2_bulk_g2s(ring + (size_t)(m & 1u) * P2_ITEM_DOUBLES, A.val + (size_t)j0 * BB, bytes, mb + (m & 1u), pol);
    }
  };
  unsigned mrun = 0;  // running index of the next item this warp consumes
  int rec0 = load_rec(0), rec1 = load_rec(1), rec2 = load_rec(2);
  if (nwi > 0) { issue(0, rec0); issue(1, rec1); }

  const bool prof_on = A.prof != nullptr && blockIdx.x == 0 && tid == 0;
  long long tprev = clock64();
  auto lap = [&](int slot) { if (prof_on) { const long long t = clock64(); A.prof[slot] += t - tprev; tprev = t; } };

  // ---- x = 0, r = b on the CTA's rows; p_old = 0 everywhere; rc = 0 ---------------------------------------------------------
  for (int i = tid; i < (c1 - c0) * BS; i += P2_TPB) {
    const size_t g = (size_t)c0 * BS + i;
    A.x[g] = 0.0;
    A.r[g] = A.b[g];
  }
  for (size_t i = (size_t)blockIdx.x * P2_TPB + tid; i < nv; i += (size_t)G * P2_TPB) A.p[i] = 0.0;
  for (int j = tid; j < nC; j += P2_TPB) sm_rc[j] = 0.0;
  for (int i = tid; i < P2_W; i += P2_TPB) sm_bcnt[i] = 0;

  bool coarse = nC > 0 && A.status[3] > 0.0;
  double rz = 0.0, bb = 0.0, rr = 0.0, beta = 0.0, stop2 = 0.0;
  int it, flag = 1, pc = 0;
  bool alive = true;
  auto no_publish = [] {};

  // it = -1 is the set-up pass: the same three phases with "q" = -b, alpha = 1 (rc = P^T b), no product, no x / r update
  for (it = -1; it < A.max_iter; it++) {
    const int par = it & 1;
    double* tp = A.tpart + (size_t)par * nC;
    double acc_pq = 0.0;
    if (it >= 0) {
      const double* pold = A.p + (size_t)pc * nv;
      double* pnew = A.p + (size_t)(pc ^ 1) * nv;
      const double* z = zbuf(me, par);
      // ---------------- phase 1: q = S p on the own rows, p.q, P^T q ----------------------------------------------------
      // every rank keeps the whole direction p: the rows of other ranks are updated from their owners' z (pulled over NVLink); the
      // first element of every thread is requested now and consumed after the product, so the round trip hides behind it
      const size_t gstride = (size_t)G * P2_TPB, g_first = (size_t)blockIdx.x * P2_TPB + tid;
      double z_first = 0.0;
      const bool first_remote = N > 1 && g_first < nv && ((int)(g_first / BS) < A.r0 || (int)(g_first / BS) >= A.r1) && A.need[g_first / BS];
      if (first_remote) z_first = load_z(par, g_first);
      for (int i = tid; i < (whi - wlo) * BS; i += P2_TPB) {
        const size_t g = (size_t)wlo * BS + i;
        const int a = wlo + i / BS;
        const bool mine = N == 1 || (a >= A.r0 && a < A.r1);
        sm_pwin[i] = (mine || A.need[a]) ? fma(beta, __ldcg(pold + g), load_z(par, g)) : 0.0;   // rows of other ranks only where some block reads them
      }
      __syncthreads();
      auto pvec = [&](int col, int k) -> double {  // component k of p at block column col
        if (col >= wlo && col < whi) return sm_pwin[(size_t)(col - wlo) * BS + k];
        const size_t g = (size_t)col * BS + k;
        return fma(beta, __ldcg(pold + g), load_z(par, g));
      };
      for (int i = lane; i < P2_SLAB_ROWS * 6; i += 32) slab[i] = 0.0;
      __syncwarp();
      auto row_part = [&](int a, double yv) {  // lanes 0..5: the streamed part of (S p)_a, completed after the CTA's product
        if (lane < BS) A.q[(size_t)a * BS + lane] = yv;
      };
      P2CoarseAcc cs{-1, 0.0, 0.0};
      auto row_done = [&](int a, double yv) {  // lanes 0..5 hold the components of (S p)_a
        if (lane < BS) {
          const size_t g = (size_t)a * BS + lane;
          const double pn = pvec(a, lane);
          pnew[g] = pn;
          A.q[g] = yv;
          acc_pq += yv * pn;
        }
        if (coarse) p2_cadd(A, cs, tp, a, yv, lane);
      };
      const int half = lane & 1, blk = lane >> 1;
      double y0 = 0.0, y1 = 0.0, y2 = 0.0;
      bool started = false;
      int npart = 0;
      // the three direction components of this lane's half of its block, for the first item
      double pa0 = 0.0, pa1 = 0.0, pa2 = 0.0;
      if (nwi > 0) {
        const int nb = __shfl_sync(0xffffffffu, rec0, 1);
        const int col = __shfl_sync(0xffffffffu, rec0, 4 + blk);
        if (blk < nb) { pa0 = pvec(col, 3 * half); pa1 = pvec(col, 3 * half + 1); pa2 = pvec(col, 3 * half + 2); }
      }
      for (int k = 0; k < nwi; k++, mrun++) {
        const int nb = __shfl_sync(0xffffffffu, rec0, 1), row = __shfl_sync(0xffffffffu, rec0, 2);
        const int flags = __shfl_sync(0xffffffffu, rec0, 3);
        const int colb = __shfl_sync(0xffffffffu, rec0, 4 + blk);
        // next item's direction components and the record three items ahead, requested before the wait
        double pn0 = 0.0, pn1 = 0.0, pn2 = 0.0;
        if (k + 1 < nwi) {
          const int nb1 = __shfl_sync(0xffffffffu, rec1, 1);
          const int col1 = __shfl_sync(0xffffffffu, rec1, 4 + blk);
          if (blk < nb1) { pn0 = pvec(col1, 3 * half); pn1 = pvec(col1, 3 * half + 1); pn2 = pvec(col1, 3 * half + 2); }
        }
        const int rec3 = load_rec(mrun + 3);
        const unsigned buf = mrun & 1u;
        p2_mbar_wait(mb + buf, (mrun >> 1) & 1u, A.timeout_cycles);
        // partner's half of the direction
        const double qb0 = __shfl_xor_sync(0xffffffffu, pa0, 1), qb1 = __shfl_xor_sync(0xffffffffu, pa1, 1),
                     qb2 = __shfl_xor_sync(0xffffffffu, pa2, 1);
        const double v0 = half ? qb0 : pa0, v1 = half ? qb1 : pa1, v2 = half ? qb2 : pa2;
        const double v3 = half ? pa0 : qb0, v4 = half ? pa1 : qb1, v5 = half ? pa2 : qb2;
        if (flags & 1) started = true;
        if (blk < nb) {
          const double2* sb = reinterpret_cast<const double2*>(ring + (size_t)buf * P2_ITEM_DOUBLES + (size_t)blk * BB + half * 18);
          const double2 a0 = sb[0], a1 = sb[1], a2 = sb[2], b0 = sb[3], b1 = sb[4], b2 = sb[5], d0 = sb[6], d1 = sb[7], d2 = sb[8];
          y0 += a0.x * v0 + a0.y * v1 + a1.x * v2 + a1.y * v3 + a2.x * v4 + a2.y * v5;
          y1 += b0.x * v0 + b0.y * v1 + b1.x * v2 + b1.y * v3 + b2.x * v4 + b2.y * v5;
          y2 += d0.x * v0 + d0.y * v1 + d1.x * v2 + d1.y * v3 + d2.x * v4 + d2.y * v5;
        }
        if (flags >> 4) {  // S_ab^T p_a for row b from the same copy: this half sums its three rows, the pair swaps halves of the result
          const bool tr = blk < nb && ((flags >> (4 + blk)) & 1);
          double t0 = 0.0, t1 = 0.0, t2 = 0.0, t3 = 0.0, t4 = 0.0, t5 = 0.0;
          if (tr) {
            const double2* sb = reinterpret_cast<const double2*>(ring + (size_t)buf * P2_ITEM_DOUBLES + (size_t)blk * BB + half * 18);
            const double2 a0 = sb[0], a1 = sb[1], a2 = sb[2], b0 = sb[3], b1 = sb[4], b2 = sb[5], d0 = sb[6], d1 = sb[7], d2 = sb[8];
            const double r0 = pvec(row, 3 * half), r1 = pvec(row, 3 * half + 1), r2 = pvec(row, 3 * half + 2);
            t0 = a0.x * r0 + b0.x * r1 + d0.x * r2; t1 = a0.y * r0 + b0.y * r1 + d0.y * r2;
            t2 = a1.x * r0 + b1.x * r1 + d1.x * r2; t3 = a1.y * r0 + b1.y * r1 + d1.y * r2;
            t4 = a2.x * r0 + b2.x * r1 + d2.x * r2; t5 = a2.y * r0 + b2.y * r1 + d2.y * r2;
          }
          const double s0 = __shfl_xor_sync(0xffffffffu, half ? t0 : t3, 1), s1 = __shfl_xor_sync(0xffffffffu, half ? t1 : t4, 1),
                       s2 = __shfl_xor_sync(0xffffffffu, half ? t2 : t5, 1);
          if (tr) {  // the blocks of an item sit in distinct columns: no two lane pairs add into the same row
            double* d = slab + (size_t)(colb - slo) * BS + 3 * half;
            d[0] += (half ? t3 : t0) + s0;
            d[1] += (half ? t4 : t1) + s1;
            d[2] += (half ? t5 : t2) + s2;
          }
        }
        __syncwarp();
        issue(mrun + 2, rec2);  // the buffer just consumed takes the item two ahead (cyclic: wraps into the next product)
        if ((flags & 2) || k == nwi - 1) {
#pragma unroll
          for (int o = 2; o < 32; o <<= 1) {
            y0 += __shfl_xor_sync(0xffffffffu, y0, o);
            y1 += __shfl_xor_sync(0xffffffffu, y1, o);
            y2 += __shfl_xor_sync(0xffffffffu, y2, o);
          }
          const int src = lane < BS ? lane / 3 : 0;
          const double t0 = __shfl_sync(0xffffffffu, y0, src), t1 = __shfl_sync(0xffffffffu, y1, src), t2 = __shfl_sync(0xffffffffu, y2, src);
          const double yv = (lane % 3 == 0) ? t0 : (lane % 3 == 1) ? t1 : t2;
          if (started && (flags & 2)) {
            row_part(row, yv);
          } else {  // the row continues in a neighbouring warp's run: leave the partial sum for the merge below
            if (lane < BS) sm_bval[(size_t)(wid * 2 + npart) * BS + lane] = yv;
            if (lane == 0) sm_brow[wid * 2 + npart] = row;
            npart++;
          }
          y0 = y1 = y2 = 0.0;
          started = false;
        }
        rec0 = rec1; rec1 = rec2; rec2 = rec3;
        pa0 = pn0; pa1 = pn1; pa2 = pn2;
      }
      if (lane == 0) sm_bcnt[wid] = npart;
      __syncthreads();
      {  // rows cut by run boundaries: the warp that holds the first piece of a row sums the pieces in run order
        const int mycnt = sm_bcnt[wid];
        for (int e = 0; e < mycnt; e++) {
          const int row = sm_brow[wid * 2 + e];
          int prow = -1;
          if (e > 0) prow = sm_brow[wid * 2 + e - 1];
          else
            for (int w = wid - 1; w >= 0; w--)
              if (sm_bcnt[w] > 0) { prow = sm_brow[w * 2 + sm_bcnt[w] - 1]; break; }
          if (prow == row) continue;  // an earlier warp holds the first piece
          double accv = lane < BS ? sm_bval[(size_t)(wid * 2 + e) * BS + lane] : 0.0;
          int w = wid, f = e + 1;
          while (w < P2_W) {
            if (f >= sm_bcnt[w]) { w++; f = 0; continue; }
            if (sm_brow[w * 2 + f] != row) break;
            if (lane < BS) accv += sm_bval[(size_t)(w * 2 + f) * BS + lane];
            f++;
          }
          row_part(row, accv);
        }
      }
      __syncthreads();
      // every row of the CTA: its streamed part plus the warps' transposed products in warp order (a fixed order); rows in
      // increasing order per warp, so the running sums of P^T q apply
      for (int a = c0 + wid; a < c1; a += P2_W) {
        double v = 0.0;
        if (lane < BS) {
          v = A.q[(size_t)a * BS + lane];
          for (int w = 0; w < P2_W; w++) {
            const int o = a - s_slo[w];
            if (o >= 0 && o < P2_SLAB_ROWS) v += sm_slab[((size_t)w * P2_SLAB_ROWS + o) * BS + lane];
          }
        }
        row_done(a, v);
      }
      if (coarse) { p2_cflush(A, tp, cs.cur, cs.l, lane); p2_cflush(A, tp, cs.cur + 1, cs.h, lane); }
      if (N > 1)
        for (size_t i = g_first; i < nv; i += gstride) {
          const int a = (int)(i / BS);
          if ((a < A.r0 || a >= A.r1) && A.need[a]) pnew[i] = fma(beta, __ldcg(pold + i), i == g_first ? z_first : load_z(par, i));
        }
    } else if (coarse) {
      // set-up pass: P^T b of the CTA's rows (rows in increasing order per warp: the running sums still apply)
      P2CoarseAcc cs{-1, 0.0, 0.0};
      for (int a = c0 + wid; a < c1; a += P2_W) {
        const double v = lane < BS ? A.b[(size_t)a * BS + lane] : 0.0;
        p2_cadd(A, cs, tp, a, v, lane);
      }
      p2_cflush(A, tp, cs.cur, cs.l, lane);
      p2_cflush(A, tp, cs.cur + 1, cs.h, lane);
    }
    {
      const double t0 = block_sum(acc_pq, red);
      if (tid == 0) part0[blockIdx.x] = t0;
    }
    // ---------------- synchronisation A: p.q and P^T q of every rank ---------------------------------------------------------
    const unsigned epA = A.ll_epoch0 + 2u * (unsigned)(it + 1), epB = epA + 1u;
    alive = p2_barrier(A, gen, epoch, false, false, &s_ok, [&] {
      if (N == 1) return;
      const double v = sum_partials_dev(part0, G);   // every warp of CTA 0 forms the same sum
      if (tid < N && tid != me) {
        p2_ll_store(lls(tid, par, me, 0), v, epA);
        if (it < 0) p2_ll_store(lls(tid, par, me, 1), coarse ? 1.0 : 0.0, epA);
      }
      // a rank's P^T q partial is non-zero only on the coarse nodes its own rows hang on: [trange(me).lo, trange(me).hi)
      const int jlo = t_lo(me), jn = t_hi(me) - jlo;
      for (int i = tid; i < jn * N; i += P2_TPB) {
        const int k = i / jn, j = jlo + (i - k * jn);
        if (k != me) p2_ll_store(llt(k, par, me, j), __ldcg(tp + j), epA);
      }
    });
    if (!alive) break;
    if (N > 1) {  // the peers' packets: thread k < N fetches rank k's scalars for the whole CTA
      if (wid == 0) {
        const double own = sum_partials_dev(part0, G);
        if (lane < N) {
          sm_ll[lane][0] = lane == me ? own : ll_wait(lls(me, par, lane, 0), epA);
          sm_ll[lane][1] = (it < 0 && lane != me) ? ll_wait(lls(me, par, lane, 1), epA) : 1.0;
        }
      }
      if (__syncthreads_or(!ll_ok)) { alive = false; break; }
    }
    lap(it < 0 ? 0 : 1);
    // ---------------- phase 2: alpha; x, r on the CTA's rows; rc; the CTA's slice of yc = Ainv rc -----------------------------
    double alpha = 1.0;
    if (it >= 0) {
      double pq;
      if (N == 1) pq = sum_partials_dev(part0, G);
      else { pq = 0.0; for (int k = 0; k < N; k++) pq += sm_ll[k][0]; }
      if (!(pq > 0.0) || !isfinite(pq)) { flag = 2; break; }
      alpha = rz / pq;
      const double* pnew = A.p + (size_t)(pc ^ 1) * nv;
      for (int i = tid; i < (c1 - c0) * BS; i += P2_TPB) {
        const size_t g = (size_t)c0 * BS + i;
        A.x[g] += alpha * pnew[g];
        A.r[g] -= alpha * A.q[g];
      }
    } else if (N > 1) {  // the ranks invert their coarse matrices independently: use the coarse level only if all of them can
      double all = 1.0;
      for (int k = 0; k < N; k++) all = fmin(all, sm_ll[k][1]);
      coarse = coarse && all > 0.0;
    }
    if (coarse) {
      const double sgn = it < 0 ? 1.0 : -alpha;
      for (int j = tid; j < nC; j += P2_TPB) {
        double t;
        if (N == 1) t = __ldcg(tp + j);
        else {
          t = 0.0;
          for (int k = 0; k < N; k++)
            if (k == me) t += __ldcg(tp + j);
            else if (j >= t_lo(k) && j < t_hi(k)) t += ll_wait(llt(me, par, k, j), epA);
        }
        sm_rc[j] = fma(sgn, t, sm_rc[j]);
      }
      if (__syncthreads_or(!ll_ok)) { alive = false; break; }
      const int i0 = (int)((long long)nC * blockIdx.x / G), i1 = (int)((long long)nC * (blockIdx.x + 1) / G);
      for (int i = i0 + wid; i < i1; i += P2_W) {
        const double* arow = A.Ainv + (size_t)i * nC;
        double s = 0.0;
        for (int j = lane; j < nC; j += 32) s += __ldg(arow + j) * sm_rc[j];
        s = warp_sum(s);
        if (lane == 0) A.yc[(size_t)par * nC + i] = s;
      }
    }
    // ---------------- synchronisation Y (this GPU only): yc complete ---------------------------------------------------------
    alive = p2_barrier(A, gen, epoch, false, false, &s_ok, no_publish);
    if (!alive) break;
    lap(it < 0 ? 0 : 2);
    // ---------------- phase 3: z = Minv r + P yc on the CTA's rows -> every rank's z buffer of the other parity; r.z, r.r -----
    double acc_rz = 0.0, acc_rr = 0.0;
    for (int i = tid; i < (c1 - c0) * BS; i += P2_TPB) {
      const int a = c0 + i / BS, c = i % BS;
      const double* rrow = A.r + (size_t)a * BS;
      const double* M = A.Minv + (size_t)a * BB + c * BS;
      double zv = 0.0;
#pragma unroll
      for (int k = 0; k < BS; k++) zv += __ldg(M + k) * rrow[k];
      if (coarse) {
        const CoarseParents pa = coarse_parents(a, A.agg, A.nc, A.prolong);
        zv += pa.w0 * __ldcg(A.yc + (size_t)par * nC + (size_t)pa.lo * BS + c);
        if (pa.w1 != 0.0) zv += pa.w1 * __ldcg(A.yc + (size_t)par * nC + (size_t)pa.hi * BS + c);
      }
      const double rv = rrow[c];
      zbuf(me, par ^ 1)[(size_t)a * BS + c] = zv;   // own window only: peers pull the rows they need
      acc_rz += rv * zv;
      acc_rr += rv * rv;
    }
    // the P^T q buffer of the other parity is idle here (last read after A of the previous iteration, next filled after B)
    for (size_t j = (size_t)blockIdx.x * P2_TPB + tid; j < (size_t)nC; j += (size_t)G * P2_TPB) A.tpart[(size_t)(par ^ 1) * nC + j] = 0.0;
    {
      const double t0 = block_sum(acc_rz, red);
      const double t1 = block_sum(acc_rr, red);
      if (tid == 0) { part1[blockIdx.x] = t0; part2[blockIdx.x] = t1; }
    }
    // ---------------- synchronisation B: r.z, r.r of every rank; the z slices are in place --------------------------------------
    alive = p2_barrier(A, gen, epoch, false, false, &s_ok, [&] {
      if (N == 1) return;
      __threadfence_system();   // this rank's z rows (all CTAs have arrived) are ordered before the packets that announce them
      const double v1 = sum_partials_dev(part1, G);
      const double v2 = sum_partials_dev(part2, G);
      if (tid < N && tid != me) { p2_ll_store(lls(tid, par, me, 2), v1, epB); p2_ll_store(lls(tid, par, me, 3), v2, epB); }
    });
    if (!alive) break;
    if (N > 1) {
      if (wid == 0) {
        const double o1 = sum_partials_dev(part1, G), o2 = sum_partials_dev(part2, G);
        if (lane < N) {
          sm_ll[lane][2] = lane == me ? o1 : ll_wait(lls(me, par, lane, 2), epB);
          sm_ll[lane][3] = lane == me ? o2 : ll_wait(lls(me, par, lane, 3), epB);
        }
      }
      if (__syncthreads_or(!ll_ok)) { alive = false; break; }
    }
    lap(it < 0 ? 0 : 3);
    double rz_new, rr_new;
    if (N == 1) { rz_new = sum_partials_dev(part1, G); rr_new = sum_partials_dev(part2, G); }
    else {
      rz_new = 0.0; rr_new = 0.0;
      for (int k = 0; k < N; k++) { rz_new += sm_ll[k][2]; rr_new += sm_ll[k][3]; }
    }
    if (it < 0) {
      rz = rz_new; bb = rr_new; rr = bb;
      stop2 = A.tol * A.tol * bb;
      if (!(bb > 0.0)) { flag = 0; it = 0; break; }
    } else {
      rr = rr_new;
      pc ^= 1;
      if (rr <= stop2) { flag = 0; it++; break; }
      beta = rz_new / rz;
      rz = rz_new;
    }
  }
  if (it < 0) it = 0;
  // ---- N ranks: every rank returns the whole x ------------------------------------------------------------------------------
  if (alive && N > 1) {
    for (int i = tid; i < (c1 - c0) * BS; i += P2_TPB) {
      const size_t g = (size_t)c0 * BS + i;
      const double xv = A.x[g];
      for (int k = 0; k < N; k++) reinterpret_cast<double*>(A.win[k] + A.off_x)[g] = xv;
    }
    alive = p2_barrier(A, gen, epoch, true, true, &s_ok, no_publish);
    if (alive) {
      const double* xs = reinterpret_cast<const double*>(A.win[me] + A.off_x);
      for (size_t i = (size_t)blockIdx.x * P2_TPB + tid; i < nv; i += (size_t)G * P2_TPB) A.x[i] = __ldcg(xs + i);
    }
  }
  // the two copies every warp still has in flight must land before the CTA (and its shared memory) goes away
  if (nwi > 0) {
    p2_mbar_wait(mb + (mrun & 1u), (mrun >> 1) & 1u, A.timeout_cycles);
    p2_mbar_wait(mb + ((mrun + 1) & 1u), ((mrun + 1) >> 1) & 1u, A.timeout_cycles);
  }
  if (blockIdx.x == 0 && tid == 0) {
    A.status[0] = (double)it;
    A.status[1] = bb > 0.0 ? sqrt(rr / bb) : 0.0;
    A.status[2] = alive ? (double)flag : 3.0;
    A.status[3] = coarse ? (double)nC : 0.0;
  }
}

// byte layout of one exchange window
struct Pcg2Layout {
  size_t off_z, off_x, off_flags, off_ctl, off_lls, off_llt, bytes;
};
inline Pcg2Layout pcg2_layout(int n, int nranks, int nC) {
  Pcg2Layout L;
  size_t o = 0;
  auto take = [&](size_t bytes) { const size_t at = o; o += (bytes + 255) & ~(size_t)255; return at; };
  const size_t nv = (size_t)n * 6;
  L.off_z = take(2 * nv * sizeof(double));
  L.off_x = take(nv * sizeof(double));
  L.off_flags = take((size_t)nranks * sizeof(unsigned long long));
  L.off_ctl = take(sizeof(unsigned));
  L.off_lls = take((size_t)2 * nranks * 4 * 16);
  L.off_llt = take((size_t)2 * nranks * (nC > 0 ? nC : 1) * 16);
  L.bytes = o;
  return L;
}

// The item records of the rows [cta_row[0], cta_row[grid]) as k_pcg2 streams them (tools/pcg2_bytes.py restates this in numpy).
// A CTA owns the rows [c0, c1).  The lane pair that holds an upper block (a, b) with a < b < c1 applies it twice: S_ab p_b for row a
// and S_ab^T p_a for row b, into its warp's slab (flag bit 4 + k of the item).  The mirror (b, a) is then not streamed, so row b
// streams two contiguous runs of s_val: [rowptr[b], first block at column >= c0) and [first block at column >= b, rowptr[b + 1]).
// A warp's slab covers P2_SLAB_ROWS rows from the lowest row it adds into; a block whose row b falls beyond it is not applied
// transposed and its mirror is streamed as before.  That changes the item counts and so the warps' runs, so the CTA's plan is
// redone until no block falls out (blocks only ever go back to the full stream: it ends).  Nothing of it crosses a CTA, so the
// CTAs are planned one after the other, each to its own fixed point.
struct Pcg2Plan {
  std::vector<int> items, cta_item, slab_lo;
  long long streamed = 0;   // blocks streamed per product
};
// one CTA's rows [c0, c1): its items (appended to items), its warps' slabs (slab_lo[P2_W]); returns the blocks it streams.
// mirror / skip / cur are scratch, reused from CTA to CTA.
inline long long pcg2_plan_cta(const std::vector<int>& rowptr, const int* cl, int c0, int c1, std::vector<int>& items, int* slab_lo,
                               std::vector<int>& mirror, std::vector<unsigned char>& skip, std::vector<int>& cur) {
  const int base = rowptr[c0];
  const size_t item0 = items.size();
  // mirror[j - base]: the index of the mirror of upper block j when j is applied transposed, else -1; skip: that mirror
  mirror.assign((size_t)(rowptr[c1] - base), -1);
  skip.assign(mirror.size(), 0);
  // merge walk: as the rows a are visited in increasing order, the mirrors (b, a) with c0 <= a < b come in increasing order in
  // row b, so a cursor per row, started at its first column >= c0, finds each in one step
  cur.resize((size_t)(c1 - c0));
  for (int b = c0; b < c1; b++) cur[b - c0] = (int)(std::lower_bound(cl + rowptr[b], cl + rowptr[b + 1], c0) - cl);
  for (int a = c0; a < c1; a++)
    for (int j = rowptr[a]; j < rowptr[a + 1]; j++) {
      const int b = cl[j];
      if (b <= a) continue;
      if (b >= c1) break;
      const int m = cur[b - c0]++;
      mirror[j - base] = m;
      skip[m - base] = 1;
    }
  for (;;) {
    items.resize(item0);
    long long streamed = 0;
    for (int a = c0; a < c1; a++) {
      const size_t first = items.size();
      for (int j = rowptr[a]; j < rowptr[a + 1];) {
        if (skip[j - base]) { j++; continue; }
        int e = j;
        while (e < rowptr[a + 1] && e - j < P2_ITEM_BLOCKS && !skip[e - base]) e++;
        const size_t o = items.size();
        items.resize(o + P2_REC, 0);
        int* rec = &items[o];
        rec[0] = j; rec[1] = e - j; rec[2] = a;
        for (int k = 0; k < e - j; k++) {
          rec[4 + k] = cl[j + k];
          if (mirror[j + k - base] >= 0) rec[3] |= 1 << (4 + k);
        }
        streamed += e - j;
        j = e;
      }
      if (items.size() > first) {
        items[first + 3] |= 1;
        items[items.size() - P2_REC + 3] |= 2;
      }
    }
    // the warps' runs as k_pcg2 cuts them, their slabs, and the blocks that fall out of them
    const int n = (int)((items.size() - item0) / P2_REC);
    const int* recs = items.data() + item0;
    bool changed = false;
    for (int w = 0; w < P2_W; w++) {
      const int wb = (int)((long long)n * w / P2_W), we = (int)((long long)n * (w + 1) / P2_W);
      int lo = INT32_MAX;
      for (int m = wb; m < we; m++) {
        const int* rec = recs + (size_t)m * P2_REC;
        for (int k = 0; k < rec[1]; k++)
          if ((rec[3] >> (4 + k)) & 1) lo = std::min(lo, rec[4 + k]);
      }
      slab_lo[w] = lo == INT32_MAX ? P2_NO_SLAB : lo;
      if (lo == INT32_MAX) continue;
      for (int m = wb; m < we; m++) {
        const int* rec = recs + (size_t)m * P2_REC;
        for (int k = 0; k < rec[1]; k++)
          if (((rec[3] >> (4 + k)) & 1) && rec[4 + k] - lo >= P2_SLAB_ROWS) {
            int& mj = mirror[rec[0] + k - base];
            skip[mj - base] = 0;
            mj = -1;
            changed = true;
          }
      }
    }
    if (!changed) return streamed;
  }
}
inline Pcg2Plan pcg2_plan(const std::vector<int>& rowptr, const std::vector<int>& col, const std::vector<int>& cta_row) {
  const int grid = (int)cta_row.size() - 1;
  Pcg2Plan P;
  P.items.reserve(((size_t)(rowptr[cta_row[grid]] - rowptr[cta_row[0]]) / P2_ITEM_BLOCKS + 2 * (size_t)(cta_row[grid] - cta_row[0]) + 1) *
                  P2_REC);
  P.cta_item.assign((size_t)grid + 1, 0);
  P.slab_lo.assign((size_t)grid * P2_W, P2_NO_SLAB);
  std::vector<int> mirror, cur;
  std::vector<unsigned char> skip;
  for (int c = 0; c < grid; c++) {
    P.cta_item[c] = (int)(P.items.size() / P2_REC);
    P.streamed += pcg2_plan_cta(rowptr, col.data(), cta_row[c], cta_row[c + 1], P.items, &P.slab_lo[(size_t)c * P2_W], mirror, skip, cur);
  }
  P.cta_item[grid] = (int)(P.items.size() / P2_REC);
  return P;
}

}  // namespace ccm

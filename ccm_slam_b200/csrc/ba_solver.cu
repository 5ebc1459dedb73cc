// ba_solver.cu — host driver of the bundle-adjustment path + its C ABI (include/ccm_b200.h).
//
// Control flow restates g2o's OptimizationAlgorithmLevenberg::solve + SparseOptimizer::optimize
// (G/core/optimization_algorithm_levenberg.cpp:61-164, G/core/sparse_optimizer.cpp:354-419): the scalar LM schedule
// (lm_schedule.h; force-stop flag polling here) runs on the host, every O(E)/O(P)/O(K) step is a kernel from
// ba_kernels.cuh on the handle's stream.  push/pop/discardTop become a (current, trial) double buffer.
// Multi-GPU: landmarks (and their observations) are sharded across ranks; per LM iteration one all-reduce of
// [Hpp | bp | chi2], per LM trial one all-reduce of [S upper blocks | bschur part] and one of [chi2, scale].
#include <algorithm>
#include <chrono>
#include <cmath>
#include <numeric>

#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>

#include "ba_kernels.cuh"
#include "common.cuh"
#include "lm_schedule.h"
#include "pcg2.cuh"

namespace ccm {
void allreduce_f64(double* buf, size_t count, int op, cudaStream_t s);  // runtime.cu ; op: 0 sum, 2 max
}

using namespace ccm;
using namespace ccm::ba;

namespace {
template <typename T>
void upload_vec(DevBuf<T>& b, const std::vector<T>& v, cudaStream_t s) {  // never a zero-sized allocation
  b.alloc(std::max(v.size(), (size_t)1));
  if (!v.empty()) CCM_CUDA(cudaMemcpyAsync(b.p, v.data(), v.size() * sizeof(T), cudaMemcpyHostToDevice, s));
}
double now_ms() {
  return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now().time_since_epoch()).count();
}
int env_int(const char* name, int dflt) {
  const char* v = getenv(name);
  return v ? atoi(v) : dflt;
}
}  // namespace

struct ccm_ba_handle {
  cudaStream_t stream = nullptr;
  int device = 0;
  int K = 0, P = 0, E = 0, Kf = 0;
  int rank = 0, nranks = 1;
  int L0 = 0, L1 = 0, Pl = 0, El = 0;
  long long E0 = 0;
  size_t Ep = 0;
  std::vector<int> perm;            // landmark-grouped position -> input edge index; empty when the input came grouped
  std::vector<uint8_t> h_flags;     // local shard, grouped order
  std::vector<int> h_pose_slot, h_slot_pose;
  int words = 0, nub = 0;
  long long nnzb = 0, nprod = 0;
  // state
  DevBuf<double> pose0, poseA, poseB, intr, pt0, ptA, ptB;
  double *pose_cur = nullptr, *pose_trial = nullptr, *pt_cur = nullptr, *pt_trial = nullptr;
  const double *pose_eval = nullptr, *pt_eval = nullptr;  // last state errors were evaluated on
  DevBuf<int> pose_slot, slot_pose;
  // observations (landmark order, local shard)
  DevBuf<int> o_kf, o_lm, lm_ptr;
  DevBuf<float2> o_uv;
  DevBuf<float> o_w, o_w_raw;
  DevBuf<uint8_t> d_flags;
  // linear system
  DevBuf<double> Z, HllBl, gvec;          // HllBl = [Hll 6*Pl | bl 3*Pl]
  DevBuf<double> W;                       // ccm_ba_debug_build only: allocated on its first call
  DevBuf<int> units;                      // landmark-aligned CTA schedule of k_linearize / k_backsub_points
  int nunits = 0, lin_grid = 1, bs_grid = 1;
  DevBuf<double> Hbuf;                    // [Hpp Kf*36 | bp Kf*6 | chi2_cur | maxdiag-bits]
  DevBuf<double> Ubuf;                    // [U_val nub*36 | bneg Kf*6]
  DevBuf<double> s_val, Minv, bschur, dxl;
  DevBuf<int> s_rowptr, s_col, s_row, s_diag, csr_u, u_row, u_col, u_diag, word_prefix;
  DevBuf<unsigned> bitmap, u_prod_ptr;
  DevBuf<uint2> prod;
  DevBuf<int> u_sched, task_ptr, next_task;   // k_schur_mma's schedule: upper blocks by row, longest list first, cut into tasks
  int ntasks = 0, schur_grid = 1;
  DevBuf<float4> kobs;            // per free pose: (u, v, signed w, landmark) of its observations, packed
  DevBuf<unsigned> kobs_ptr;
  // pcg
  PcgDriver<6> pcg;               // k_pcg, and the x / r / p / q / partials / bar / status k_pcg2 reads as well
  int pcg_refresh = 4, pcg_age = 0, pcg_last_mode = 1;
  bool pcg_coarse_valid = false;  // Ac holds a usable inverse from an earlier trial
  DevBuf<long long> pcg_prof;  // allocated only with CCM_PCG_PROF=1
  DevBuf<int> jac_fail;
  // second-generation PCG (pcg2.cuh): TMA-streamed product, three synchronisations per iteration, rows distributed over the ranks
  struct Pcg2 {
    bool on = false;
    Pcg2Layout lay{};
    char* window = nullptr;          // own exchange window: plain cudaMalloc (exportable through cudaIpc) on several ranks, pool memory on one
    bool window_pooled = false;
    std::vector<char*> peer;         // every rank's window as mapped here; peer[rank] == window
    DevBuf<char*> d_win;
    DevBuf<int> items, cta_row, cta_item, rank_row, slab_lo;
    DevBuf<unsigned char> need;
    DevBuf<double> yc, tpart;
    int r0 = 0, r1 = 0, rank = 0, grid = 1;
    long long nitems = 0, streamed = 0;
    unsigned long long launches = 0;
    long long timeout_cycles = 0;
  } p2;
  // scalars / partials
  DevBuf<double> partials, scal;  // scal: [0] chi2_trial [1] scale_l [2] scale_p [3..5] pcg status
  double* h_scal = nullptr;       // pinned, 16 doubles
  DevBuf<double> rep_chi2;
  DevBuf<uint8_t> rep_depth;
  int64_t device_bytes = 0;
  double t_setup_ms = 0;
  // per-kernel CUDA-event accounting (ccm_ba_get_kernel_stats): events are recorded on the launching stream
  bool profile = false;
  std::vector<cudaEvent_t> ev_pool;
  size_t ev_used = 0;
  struct Span { int which; size_t e0, e1; };
  std::vector<Span> spans;
  double k_ms[CCM_BA_NKERNELS] = {0};
  long long k_count[CCM_BA_NKERNELS] = {0};

  double* Hll() { return HllBl.p; }
  double* bl() { return HllBl.p + (size_t)6 * Pl; }
  double* Hpp() { return Hbuf.p; }
  double* bp() { return Hbuf.p + (size_t)Kf * 36; }
  double* chi2_cur_dev() { return Hbuf.p + (size_t)Kf * 42; }
  double* U_val() { return Ubuf.p; }
  double* bneg() { return Ubuf.p + (size_t)nub * 36; }

  ~ccm_ba_handle() {
    for (size_t k = 0; k < p2.peer.size(); k++)
      if (p2.peer[k] && (int)k != p2.rank) cudaIpcCloseMemHandle(p2.peer[k]);
    if (p2.window) { if (p2.window_pooled) dev_free(p2.window); else cudaFree(p2.window); }
    for (cudaEvent_t e : ev_pool) cudaEventDestroy(e);
    if (h_scal) cudaFreeHost(h_scal);
    if (stream) cudaStreamDestroy(stream);
  }
};

namespace {

int grid_stride(long long n) {
  long long g = (n + TPB - 1) / TPB;
  const long long cap = (long long)sm_count() * 8;
  if (g > cap) g = cap;
  if (g < 1) g = 1;
  return (int)g;
}

// Cut k of `parts` contiguous ranges of [0, n) balanced by the non-decreasing prefix ptr[0..n]: the first index where the prefix
// reaches k * ptr[n] / parts, clamped to [0, n]
int prefix_cut(const int* ptr, int n, int k, int parts) {
  if (k <= 0) return 0;
  if (k >= parts) return n;
  const long long want = (long long)ptr[n] * k / parts;
  return std::min((int)(std::lower_bound(ptr, ptr + n + 1, (int)want) - ptr), n);
}

// the caller's index of the observation at landmark-grouped position gi
long long input_edge(const ccm_ba_handle* h, long long gi) { return h->perm.empty() ? gi : h->perm[gi]; }

size_t ev_record(ccm_ba_handle* h) {
  if (h->ev_used == h->ev_pool.size()) {
    cudaEvent_t e;
    CCM_CUDA(cudaEventCreate(&e));
    h->ev_pool.push_back(e);
  }
  CCM_CUDA(cudaEventRecord(h->ev_pool[h->ev_used], h->stream));
  return h->ev_used++;
}
struct KernelSpan {  // brackets one kernel (or kernel group) with events when profiling is on
  ccm_ba_handle* h; int which; size_t e0 = 0;
  KernelSpan(ccm_ba_handle* h_, int w) : h(h_), which(w) { if (h->profile) e0 = ev_record(h); }
  ~KernelSpan() { if (h->profile) { try { size_t e1 = ev_record(h); h->spans.push_back({which, e0, e1}); } catch (...) {} } }
};
void collect_spans(ccm_ba_handle* h) {  // call after a stream synchronize
  for (const auto& sp : h->spans) {
    float ms = 0.f;
    if (cudaEventElapsedTime(&ms, h->ev_pool[sp.e0], h->ev_pool[sp.e1]) == cudaSuccess) { h->k_ms[sp.which] += ms; h->k_count[sp.which]++; }
  }
  h->spans.clear();
  h->ev_used = 0;
}

// mode: LIN_H (Hll, bl, chi2 partials) | LIN_Z (g and Z at damping lambda); dbgW: W export of ccm_ba_debug_build
void launch_linearize(ccm_ba_handle* h, int robust, double delta, int mode, double lambda, double* dbgW = nullptr) {
  k_linearize<<<h->lin_grid, LIN_TILE, 0, h->stream>>>(h->units.p, h->nunits, h->lm_ptr.p, h->o_kf.p, h->o_lm.p, h->o_uv.p, h->o_w.p,
                                                      h->pose_cur, h->intr.p, h->pose_slot.p, h->pt_cur, h->Pl, robust, delta, lambda,
                                                      mode, h->Hll(), h->bl(), h->gvec.p, h->Z.p, h->partials.p, dbgW, h->Ep);
  CCM_LAUNCHED();
}

void launch_backsub(ccm_ba_handle* h, double lambda, double* dx_points) {
  k_backsub_points<<<h->bs_grid, LIN_TILE, 0, h->stream>>>(h->units.p, h->nunits, h->lm_ptr.p, h->o_kf.p, h->pose_slot.p, h->Z.p,
                                                           h->Hll(), h->bl(), h->pcg.x.p, h->pt_cur, h->Pl, lambda, h->pt_trial, dx_points,
                                                           h->partials.p);
  CCM_LAUNCHED();
}

void pack_pose_obs(ccm_ba_handle* h) {
  if (h->Kf == 0 || h->El == 0) return;
  k_pack_pose_obs<<<h->Kf, 128, 0, h->stream>>>(h->prod.p, h->u_prod_ptr.p, h->u_diag.p, h->kobs_ptr.p, h->o_lm.p, h->o_uv.p,
                                              h->o_w.p, h->kobs.p);
  CCM_LAUNCHED();
}

void sum_partials_to(ccm_ba_handle* h, int n, double* out) {
  k_sum_partials<<<1, 1024, 0, h->stream>>>(h->partials.p, n, out);
  CCM_LAUNCHED();
}

// ---- kernels wrapped as steps --------------------------------------------------------------------------------
// linearisation at the current estimate: Hll / bl / chi2 and the pose pass; with LIN_Z in mode also g and Z at lambda
void step_linearize(ccm_ba_handle* h, int robust, double delta, int mode, double lambda, double* dbgW = nullptr) {
  cudaStream_t s = h->stream;
  {
    KernelSpan sp(h, CCM_BA_K_LINEARIZE);
    launch_linearize(h, robust, delta, LIN_H | mode, lambda, dbgW);
  }
  sum_partials_to(h, h->lin_grid, h->chi2_cur_dev());
  if (h->Kf > 0) {
    KernelSpan sp(h, CCM_BA_K_POSE_PASS);
    k_pose_pass<<<h->Kf, 128, 0, s>>>(h->kobs.p, h->kobs_ptr.p, h->slot_pose.p, h->pose_cur, h->intr.p, h->pt_cur, robust, delta,
                                      h->Hpp(), h->bp());
    CCM_LAUNCHED();
  }
  if (h->nranks > 1) allreduce_f64(h->Hbuf.p, (size_t)h->Kf * 42 + 1, 0, s);
  h->pose_eval = h->pose_cur;
  h->pt_eval = h->pt_cur;
}

double step_max_diag(ccm_ba_handle* h) {
  cudaStream_t s = h->stream;
  double* slot = h->Hbuf.p + (size_t)h->Kf * 42 + 1;
  CCM_CUDA(cudaMemsetAsync(slot, 0, sizeof(double), s));
  k_max_diag<<<grid_stride((long long)h->Kf * 6 + (long long)h->Pl * 3), TPB, 0, s>>>(
      h->Hpp(), h->Kf, h->Hll(), h->Pl, reinterpret_cast<unsigned long long*>(slot));
  CCM_LAUNCHED();
  if (h->nranks > 1) allreduce_f64(slot, 1, 2, s);
  CCM_CUDA(cudaMemcpyAsync(h->h_scal + 8, h->chi2_cur_dev(), 2 * sizeof(double), cudaMemcpyDeviceToHost, s));
  CCM_CUDA(cudaStreamSynchronize(s));
  return h->h_scal[9];
}

double read_chi2_cur(ccm_ba_handle* h) {
  CCM_CUDA(cudaMemcpyAsync(h->h_scal + 8, h->chi2_cur_dev(), sizeof(double), cudaMemcpyDeviceToHost, h->stream));
  CCM_CUDA(cudaStreamSynchronize(h->stream));
  return h->h_scal[8];
}

// g and Z at a new lambda on the unchanged estimate (the first iteration's damping, a rejected trial): the linearisation recomputed,
// nothing but g and Z written
void step_z(ccm_ba_handle* h, int robust, double delta, double lambda) {
  KernelSpan sp(h, CCM_BA_K_LINEARIZE);
  launch_linearize(h, robust, delta, LIN_Z, lambda);
}

// K4: the Schur products, one warp per upper block, the blocks of a row on one SM (k_schur_mma)
void launch_schur(ccm_ba_handle* h, cudaStream_t s) {
  if (h->ntasks == 0) return;
  CCM_CUDA(cudaMemsetAsync(h->next_task.p, 0, sizeof(int), s));
  k_schur_mma<<<h->schur_grid, SCHUR_CTA, 0, s>>>(h->prod.p, h->u_prod_ptr.p, h->u_row.p, h->u_col.p, h->u_sched.p, h->task_ptr.p,
                                                  h->ntasks, h->next_task.p, h->Z.p, h->o_lm.p, h->gvec.p, h->U_val(), h->bneg());
}

void step_schur(ccm_ba_handle* h) {
  KernelSpan sp(h, CCM_BA_K_SCHUR);
  launch_schur(h, h->stream);
  CCM_LAUNCHED();
}

void step_finalize(ccm_ba_handle* h, double lambda) {
  cudaStream_t s = h->stream;
  if (h->nranks > 1) {
    KernelSpan sp(h, CCM_BA_K_ALLREDUCE);
    allreduce_f64(h->Ubuf.p, (size_t)h->nub * 36 + (size_t)h->Kf * 6, 0, s);
  }
  KernelSpan sp(h, CCM_BA_K_FINALIZE);
  k_finalize_S<<<div_up(h->nnzb * 36, TPB), TPB, 0, s>>>(h->s_row.p, h->s_col.p, h->csr_u.p, h->nnzb, h->U_val(), h->Hpp(),
                                                         lambda, h->s_val.p);
  CCM_LAUNCHED();
  CCM_CUDA(cudaMemsetAsync(h->jac_fail.p, 0, sizeof(int), s));
  k_block_jacobi<<<div_up(h->Kf, 128), 128, 0, s>>>(h->s_diag.p, h->s_val.p, h->bp(), h->bneg(), h->Kf, h->Minv.p,
                                                    h->bschur.p, h->jac_fail.p);
  CCM_LAUNCHED();
}

void step_pcg(ccm_ba_handle* h, double tol, int max_iter) {
  cudaStream_t s = h->stream;
  KernelSpan sp(h, CCM_BA_K_PCG);
  PcgDriver<6>& pcg = h->pcg;
  const int coarse_mode = (h->pcg_coarse_valid && h->pcg_age < h->pcg_refresh) ? 2 : 1;
  h->pcg_last_mode = coarse_mode;
  if (h->p2.on) {
    ccm_ba_handle::Pcg2& d = h->p2;
    // (re)build the coarse inverse with k_pcg's set-up phase: no iteration
    if (coarse_mode == 1 && pcg.agg > 0) pcg.launch(tol, 0, coarse_mode, h->pcg_prof.p, s);
    const int nC = pcg.nC();
    Pcg2Args b;
    b.n = h->Kf; b.val = h->s_val.p; b.items = d.items.p; b.cta_row = d.cta_row.p; b.cta_item = d.cta_item.p; b.slab_lo = d.slab_lo.p;
    b.Minv = h->Minv.p; b.b = h->bschur.p; b.x = pcg.x.p; b.r = pcg.r.p; b.q = pcg.q.p; b.p = pcg.p.p;
    b.partials = pcg.partials.p; b.bar = pcg.bar.p; b.tol = tol; b.max_iter = max_iter; b.status = pcg.status.p;
    b.agg = pcg.agg; b.nc = pcg.nc; b.prolong = pcg.prolong;
    b.Ainv = nC > 0 ? coarse_inverse(pcg.Ac.p, nC) : nullptr;
    b.yc = d.yc.p; b.tpart = d.tpart.p;
    b.rank = h->rank; b.nranks = h->nranks; b.r0 = d.r0; b.r1 = d.r1; b.win = d.d_win.p;
    b.off_z = d.lay.off_z; b.off_x = d.lay.off_x;
    b.off_flags = d.lay.off_flags; b.off_ctl = d.lay.off_ctl; b.off_lls = d.lay.off_lls; b.off_llt = d.lay.off_llt;
    b.rank_row = d.rank_row.p; b.need = d.need.p;
    b.epoch0 = (++d.launches) << 24;   // every rank issues the same sequence of solves: the epochs line up and only grow
    b.ll_epoch0 = (unsigned)((d.launches & 0x7FFFFu) << 13) | 0x1000u;   // + 2 (it + 1) + {0, 1} <= 4003 below bit 12; never 0
    b.timeout_cycles = d.timeout_cycles;
    b.prof = h->pcg_prof.p;
    CCM_CUDA(cudaMemsetAsync(pcg.bar.p, 0, 2 * sizeof(unsigned), s));
    CCM_CUDA(cudaMemsetAsync(d.tpart.p, 0, d.tpart.bytes(), s));
    CCM_CUDA(cudaMemsetAsync(d.window + d.lay.off_ctl, 0, sizeof(unsigned), s));
    void* bargs[] = {&b};
    CCM_CUDA(cudaLaunchCooperativeKernel((void*)k_pcg2, dim3(d.grid), dim3(P2_TPB), bargs, P2_SMEM_BYTES, s));
    CCM_LAUNCHED();
    return;
  }
  pcg.launch(tol, max_iter, coarse_mode, h->pcg_prof.p, s);
}

// pcg2.cuh set-up: own rows, item records, CTA cuts, exchange window (IPC-mapped on every rank when nranks > 1).
// CCM_PCG_IMPL=1 keeps the first-generation kernel (replicated solve on several ranks).
void setup_pcg2(ccm_ba_handle* h, const std::vector<int>& rowptr) {
  // The streamed / distributed kernel pays off when S is large (cfg5: 788 k blocks, 227 MB) and it is the only solve that scales
  // across ranks.  Small systems (cfg3 / cfg4, LocalBA: a few 10 k blocks) are latency-bound: there the first-generation kernel is
  // faster on one GPU and, replicated, faster than a solve that crosses NVLink twice per iteration.  CCM_PCG_IMPL = 1 / 2 forces one.
  const int impl = env_int("CCM_PCG_IMPL", 0);
  if (impl == 1 || h->Kf < 1 || h->Kf < h->nranks) return;
  if (impl != 2 && rowptr[h->Kf] < env_int("CCM_PCG2_MIN_BLOCKS", 200000)) return;
  const int nC = h->pcg.nC();
  if (nC > P2_MAX_NC) return;
  static_assert(sizeof(cudaIpcMemHandle_t) == 64, "IPC handle size");
  ccm_ba_handle::Pcg2& d = h->p2;
  cudaStream_t s = h->stream;
  const int N = h->nranks, Kf = h->Kf;
  d.rank = h->rank;
  // contiguous block rows per rank, balanced by block count
  std::vector<int> rank_row((size_t)N + 1);
  for (int k = 0; k <= N; k++) rank_row[k] = prefix_cut(rowptr.data(), Kf, k, N);
  for (int k = 1; k <= N; k++) rank_row[k] = std::max(rank_row[k], rank_row[k - 1]);
  d.r0 = rank_row[h->rank];
  d.r1 = rank_row[h->rank + 1];
  upload_vec(d.rank_row, rank_row, s);
  const int rows = d.r1 - d.r0;
  // the CTAs' rows are cut by the items of the full rows (<= 16 consecutive blocks each); pcg2_plan then builds the items streamed
  std::vector<int> row_item((size_t)rows + 1, 0);
  for (int a = 0; a < rows; a++) row_item[a + 1] = row_item[a] + (rowptr[d.r0 + a + 1] - rowptr[d.r0 + a] + P2_ITEM_BLOCKS - 1) / P2_ITEM_BLOCKS;
  d.nitems = row_item[rows];
  CCM_CUDA(cudaFuncSetAttribute((const void*)k_pcg2, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)P2_SMEM_BYTES));  // per device
  int per_sm = 0;
  CCM_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, (const void*)k_pcg2, P2_TPB, P2_SMEM_BYTES));
  CCM_REQUIRE(per_sm >= 1, "k_pcg2 does not fit on an SM");
  // one CTA per SM; small systems use fewer CTAs (>= one item per warp) so that the grid barriers stay cheap
  d.grid = (int)std::max<long long>(1, std::min<long long>(sm_count(), (d.nitems + P2_W - 1) / P2_W));
  d.grid = std::max(1, env_int("CCM_PCG2_GRID", d.grid));
  d.grid = std::min(d.grid, sm_count() * per_sm);
  std::vector<int> cta_row((size_t)d.grid + 1);
  for (int c = 0; c <= d.grid; c++) cta_row[c] = d.r0 + prefix_cut(row_item.data(), rows, c, d.grid);
  std::vector<int> col((size_t)rowptr[Kf]);
  if (!col.empty()) h->s_col.download(col.data(), col.size(), s);
  CCM_CUDA(cudaStreamSynchronize(s));
  const Pcg2Plan plan = pcg2_plan(rowptr, col, cta_row);
  d.nitems = (long long)plan.items.size() / P2_REC;
  d.streamed = plan.streamed;
  std::vector<unsigned char> need((size_t)std::max(Kf, 1), 0);
  for (long long m = 0; m < d.nitems; m++)
    for (int k = 0; k < plan.items[(size_t)m * P2_REC + 1]; k++) need[plan.items[(size_t)m * P2_REC + 4 + k]] = 1;
  upload_vec(d.cta_row, cta_row, s);
  upload_vec(d.cta_item, plan.cta_item, s);
  upload_vec(d.slab_lo, plan.slab_lo, s);
  upload_vec(d.items, plan.items, s);
  upload_vec(d.need, need, s);
  d.yc.alloc_zero(std::max<size_t>((size_t)2 * nC, 1), s);
  d.tpart.alloc_zero(std::max<size_t>((size_t)2 * nC, 1), s);
  if ((size_t)3 * d.grid > h->pcg.partials.n) h->pcg.partials.alloc((size_t)3 * d.grid);
  // exchange window
  d.lay = pcg2_layout(Kf, N, nC);
  if (N == 1) {   // no peer maps it: stream-ordered pool memory (cudaMalloc / cudaFree synchronise the device on every create / destroy)
    d.window = static_cast<char*>(dev_alloc(d.lay.bytes));
    d.window_pooled = true;
    CCM_CUDA(cudaMemsetAsync(d.window, 0, d.lay.bytes, s));
  } else {
    CCM_CUDA(cudaMalloc((void**)&d.window, d.lay.bytes));
    CCM_CUDA(cudaMemset(d.window, 0, d.lay.bytes));
  }
  d.peer.assign(N, nullptr);
  d.peer[h->rank] = d.window;
  DevBuf<double> tmp;
  if (N > 1) {
    // the 64-byte IPC handles travel through the existing all-reduce, one double per byte (exact: each slot has one writer)
    cudaIpcMemHandle_t mine;
    CCM_CUDA(cudaIpcGetMemHandle(&mine, d.window));
    std::vector<double> enc((size_t)N * 64, 0.0);
    for (int i = 0; i < 64; i++) enc[(size_t)h->rank * 64 + i] = (double)reinterpret_cast<const unsigned char*>(&mine)[i];
    tmp.alloc(enc.size());
    CCM_CUDA(cudaMemcpyAsync(tmp.p, enc.data(), enc.size() * sizeof(double), cudaMemcpyHostToDevice, s));
    allreduce_f64(tmp.p, enc.size(), 0, s);
    CCM_CUDA(cudaMemcpyAsync(enc.data(), tmp.p, enc.size() * sizeof(double), cudaMemcpyDeviceToHost, s));
    CCM_CUDA(cudaStreamSynchronize(s));
    for (int k = 0; k < N; k++) {
      if (k == h->rank) continue;
      cudaIpcMemHandle_t hk;
      for (int i = 0; i < 64; i++) reinterpret_cast<unsigned char*>(&hk)[i] = (unsigned char)enc[(size_t)k * 64 + i];
      void* ptr = nullptr;
      CCM_CUDA(cudaIpcOpenMemHandle(&ptr, hk, cudaIpcMemLazyEnablePeerAccess));
      d.peer[k] = static_cast<char*>(ptr);
    }
  }
  d.d_win.alloc(N);
  CCM_CUDA(cudaMemcpyAsync(d.d_win.p, d.peer.data(), sizeof(char*) * N, cudaMemcpyHostToDevice, s));
  int khz = 0;
  CCM_CUDA(cudaDeviceGetAttribute(&khz, cudaDevAttrClockRate, h->device));
  d.timeout_cycles = (long long)env_int("CCM_PCG_DIST_TIMEOUT_MS", 2000) * std::max(khz, 1000000);
  if (N > 1) {  // every rank must have mapped every window before anybody stores into one: a last all-reduce is the fence
    allreduce_f64(tmp.p, 1, 0, s);
  }
  CCM_CUDA(cudaStreamSynchronize(s));  // the staging vectors die at the end of this scope
  d.on = true;
}

// trial state + gain-ratio denominator + chi2 of the trial state -> scal[0..5]
void step_update_and_residual(ccm_ba_handle* h, double lambda, int robust, double delta, double* dx_points, bool stop_local = false) {
  cudaStream_t s = h->stream;
  const int g1 = grid_stride(h->K);
  size_t ev0 = h->profile ? ev_record(h) : 0;
  k_update_poses<<<g1, TPB, 0, s>>>(h->pose_cur, h->pose_slot.p, h->pcg.x.p, h->bp(), h->K, lambda, h->pose_trial, h->partials.p);
  CCM_LAUNCHED();
  sum_partials_to(h, g1, h->scal.p + 2);
  launch_backsub(h, lambda, dx_points);
  sum_partials_to(h, h->bs_grid, h->scal.p + 1);
  if (h->profile) { size_t ev1 = ev_record(h); h->spans.push_back({CCM_BA_K_BACKSUB, ev0, ev1}); ev0 = ev1; }
  const int g3 = grid_stride(h->El);
  k_residual<<<g3, TPB, 0, s>>>(h->o_kf.p, h->o_lm.p, h->o_uv.p, h->o_w.p, h->pose_trial, h->intr.p, h->pt_trial, h->El,
                                robust, delta, h->partials.p);
  CCM_LAUNCHED();
  sum_partials_to(h, g3, h->scal.p + 0);
  if (h->profile) { size_t ev1 = ev_record(h); h->spans.push_back({CCM_BA_K_RESIDUAL, ev0, ev1}); }
  if (h->nranks > 1) {
    // one all-reduce carries [chi2, scale_l, scale_p, stop]: scale_p is replicated (only rank 0 contributes it, so the sum is exact),
    // stop is this rank's view of the caller's force-stop flag -> every rank takes the same decision (a flag seen by one rank a
    // trial earlier than by its peers would otherwise desynchronise the collectives and hang the job)
    if (h->rank != 0) CCM_CUDA(cudaMemsetAsync(h->scal.p + 2, 0, sizeof(double), s));
    h->h_scal[12] = stop_local ? 1.0 : 0.0;
    CCM_CUDA(cudaMemcpyAsync(h->scal.p + 3, h->h_scal + 12, sizeof(double), cudaMemcpyHostToDevice, s));
    allreduce_f64(h->scal.p, 4, 0, s);
  }
  h->pose_eval = h->pose_trial;
  h->pt_eval = h->pt_trial;
}

// landmark range [L0, L1) of `rank`: contiguous, balanced by observation count
void shard_range(const int* lm_ptr, int P, int rank, int nranks, int* L0, int* L1) {
  *L0 = prefix_cut(lm_ptr, P, rank, nranks);
  *L1 = std::max(prefix_cut(lm_ptr, P, rank + 1, nranks), *L0);
}

void do_reset(ccm_ba_handle* h) {
  cudaStream_t s = h->stream;
  CCM_CUDA(cudaMemcpyAsync(h->pose_cur, h->pose0.p, h->pose0.bytes(), cudaMemcpyDeviceToDevice, s));
  if (h->Pl) CCM_CUDA(cudaMemcpyAsync(h->pt_cur, h->pt0.p, sizeof(double) * 3 * h->Pl, cudaMemcpyDeviceToDevice, s));
  h->pose_eval = h->pose_cur; h->pt_eval = h->pt_cur;
  CCM_CUDA(cudaStreamSynchronize(s));
}

// k_check_obs over n observations: throws `what` if an index is out of range or, with w given, a weight is negative; returns whether
// the observations come grouped by landmark
bool check_obs(ccm_ba_handle* h, const int* kf, const int* mp, const float* w, int n, int P, const char* what) {
  cudaStream_t s = h->stream;
  DevBuf<int> chk; chk.alloc_zero(2, s);
  k_check_obs<<<grid_stride(n), TPB, 0, s>>>(kf, mp, w, n, h->K, P, chk.p);
  CCM_LAUNCHED();
  int hc[2];
  chk.download(hc, 2, s);
  CCM_CUDA(cudaStreamSynchronize(s));
  CCM_REQUIRE(hc[0] == 0, what);
  return hc[1] == 0;
}

// the caller's edge flags (input order; null: none) on the local shard, in grouped order
void map_edge_flags(ccm_ba_handle* h, const uint8_t* flags) {
  h->h_flags.assign(h->El, 0);
  for (int i = 0; flags && i < h->El; i++) h->h_flags[i] = flags[input_edge(h, h->E0 + i)];
}

// the weights the LM loop reads: the raw ones with h_flags applied (none given: every flag is 0)
void apply_edge_flags(ccm_ba_handle* h, bool given) {
  cudaStream_t s = h->stream;
  const int El = h->El;
  if (!El) return;
  if (given) h->d_flags.upload(h->h_flags.data(), El, s);
  else CCM_CUDA(cudaMemsetAsync(h->d_flags.p, 0, (size_t)El, s));   // no flags: nothing to send
  k_apply_flags<<<div_up(El, TPB), TPB, 0, s>>>(h->o_w_raw.p, h->d_flags.p, El, h->o_w.p);
  CCM_LAUNCHED();
}

// ---- structure: the phases of ccm_ba_create --------------------------------------------------------------------------------------
// What the phases hand each other besides the handle, alive until the create ends: the device scratch is freed only after the
// system's storage is allocated, so that storage never lands in its blocks (the PCG vectors' placement is measured: system_storage).
// One rank: the measurements (pixel coordinates and weights, 12 of the 20 bytes per observation) travel on a second stream while the
// structure of S is built from the index lists on the first; the LM stream waits for them just before their first reader.  The
// stream and its event live as long as the process (a stream per handle goes through the driver's global lock and can stall for a
// long time when something else holds it).  Builds on several threads share stream and event: a later record only makes an earlier
// build wait for more.  The destructor drains the stream before any member goes away, the grouped host arrays it reads included.
struct Setup {
  std::vector<int> kf, mp;             // ungrouped input grouped by landmark on the host; empty when the input came grouped
  std::vector<float> uv, w;
  DevBuf<int> g_kf, g_lm, g_ptr;       // several ranks: every observation and the landmark offsets on the device
  cudaStream_t meas = nullptr; cudaEvent_t meas_done = nullptr;   // one rank: the measurements' copy stream and its event
  DevBuf<int> row_count;               // blocks of S per row
  DevBuf<unsigned> cursor;             // per upper block: list lengths (count walk), then cursors (fill walk)
  DevBuf<int> row_obs, row_obs_ptr;    // the local observations grouped by block row
  ~Setup() { if (meas) cudaStreamSynchronize(meas); }
};

struct ObsLists { const int *kf, *lm, *ptr; };   // every observation on the device, grouped by landmark, and the landmark offsets

void open_handle(ccm_ba_handle* h, const ccm_ba_problem* p) {
  ensure_device();
  h->device = current_device();
  CCM_CUDA(cudaStreamCreateWithFlags(&h->stream, cudaStreamNonBlocking));
  CCM_CUDA(cudaMallocHost((void**)&h->h_scal, 16 * sizeof(double)));
  CCM_REQUIRE(p && p->K > 0 && p->P >= 0 && p->E >= 0, "ccm_ba_create: bad sizes");
  CCM_REQUIRE(p->poses && p->intr && p->fixed && (p->P == 0 || p->points), "ccm_ba_create: null pose/point arrays");
  CCM_REQUIRE(p->E == 0 || (p->obs_kf && p->obs_mp && p->obs_uv && p->obs_w), "ccm_ba_create: null observation arrays");
  h->K = p->K; h->P = p->P; h->E = p->E;
  h->rank = comm().rank; h->nranks = comm().nranks;
}

void free_pose_slots(ccm_ba_handle* h, const ccm_ba_problem* p) {
  cudaStream_t s = h->stream;
  const int K = h->K;
  h->h_pose_slot.assign(K, -1);
  for (int k = 0; k < K; k++)
    if (!p->fixed[k]) { h->h_pose_slot[k] = (int)h->h_slot_pose.size(); h->h_slot_pose.push_back(k); }
  h->Kf = (int)h->h_slot_pose.size();
  h->pose0.upload(p->poses, (size_t)K * 7, s);
  h->poseA.alloc((size_t)K * 7); h->poseB.alloc((size_t)K * 7);
  h->intr.upload(p->intr, (size_t)K * 4, s);
  h->pose_slot.upload(h->h_pose_slot.data(), K, s);
  upload_vec(h->slot_pose, h->h_slot_pose, s);
}

// Observations must be grouped by landmark (the reference adds edges landmark by landmark).  The index lists go to the device as
// they are and are validated there; ungrouped input is grouped on the host by a stable counting sort and sent again, and from then
// on every input takes one path.  On one rank the shard is every observation: the device lists are the global and the local ones.
// On several ranks the shard is cut from the landmark offsets and sliced from the global lists on the device.
ObsLists take_observations(ccm_ba_handle* h, const ccm_ba_problem* p, Setup& st) {
  cudaStream_t s = h->stream;
  const int P = h->P, E = h->E;
  const bool multi = h->nranks > 1;
  DevBuf<int>& dk = multi ? st.g_kf : h->o_kf;
  DevBuf<int>& dl = multi ? st.g_lm : h->o_lm;
  DevBuf<int>& dp = multi ? st.g_ptr : h->lm_ptr;
  const int *kf = p->obs_kf, *mp = p->obs_mp;
  const float *uv = p->obs_uv, *w = p->obs_w;
  auto send = [&] {
    dk.upload(kf, E, s); dl.upload(mp, E, s);
    if (multi) return;   // several ranks send their shard's measurements once it is cut
    copy_stream(&st.meas, &st.meas_done);
    h->o_uv.upload(reinterpret_cast<const float2*>(uv), E, st.meas); h->o_w_raw.upload(w, E, st.meas);
    CCM_CUDA(cudaEventRecord(st.meas_done, st.meas));
  };
  if (E > 0) {
    send();
    if (!check_obs(h, dk.p, dl.p, nullptr, E, P, "ccm_ba_create: observation index out of range")) {
      std::vector<int> at((size_t)P + 1, 0);   // the indices are in range: the counting sort stays inside its arrays
      for (int e = 0; e < E; e++) at[mp[e] + 1]++;
      for (int l = 0; l < P; l++) at[l + 1] += at[l];
      h->perm.resize(E);
      for (int e = 0; e < E; e++) h->perm[at[mp[e]]++] = e;
      st.kf.resize(E); st.mp.resize(E); st.uv.resize((size_t)2 * E); st.w.resize(E);
      for (int i = 0; i < E; i++) {
        const int e = h->perm[i];
        st.kf[i] = kf[e]; st.mp[i] = mp[e]; st.uv[2 * i] = uv[2 * e]; st.uv[2 * i + 1] = uv[2 * e + 1]; st.w[i] = w[e];
      }
      kf = st.kf.data(); mp = st.mp.data(); uv = st.uv.data(); w = st.w.data();
      send();
    }
  }
  dp.alloc((size_t)P + 1);
  k_lm_ptr<<<div_up((long long)P + 1, TPB), TPB, 0, s>>>(dl.p, E, P, dp.p);
  CCM_LAUNCHED();
  const ObsLists all{dk.p, dl.p, dp.p};
  if (!multi) {
    h->L0 = 0; h->L1 = P; h->Pl = P; h->E0 = 0; h->El = E;
    return all;
  }
  // several ranks: the shard's cut needs the landmark offsets on the host (4 B per landmark), then the lists are sliced on the device
  // and only this rank's measurements are sent
  std::vector<int> hp((size_t)P + 1);
  dp.download(hp.data(), hp.size(), s);
  CCM_CUDA(cudaStreamSynchronize(s));
  shard_range(hp.data(), P, h->rank, h->nranks, &h->L0, &h->L1);
  h->Pl = h->L1 - h->L0; h->E0 = hp[h->L0]; h->El = hp[h->L1] - hp[h->L0];
  const int El = h->El, Pl = h->Pl;
  h->o_kf.alloc(std::max(El, 1)); h->o_lm.alloc(std::max(El, 1)); h->lm_ptr.alloc((size_t)Pl + 1);
  h->o_uv.alloc(std::max(El, 1)); h->o_w_raw.alloc(std::max(El, 1));
  if (El) {
    CCM_CUDA(cudaMemcpyAsync(h->o_kf.p, st.g_kf.p + h->E0, sizeof(int) * (size_t)El, cudaMemcpyDeviceToDevice, s));
    k_shift<<<div_up(El, TPB), TPB, 0, s>>>(st.g_lm.p + h->E0, El, h->L0, h->o_lm.p);
    CCM_LAUNCHED();
    CCM_CUDA(cudaMemcpyAsync(h->o_uv.p, reinterpret_cast<const float2*>(uv) + h->E0, sizeof(float2) * (size_t)El, cudaMemcpyHostToDevice, s));
    CCM_CUDA(cudaMemcpyAsync(h->o_w_raw.p, w + h->E0, sizeof(float) * (size_t)El, cudaMemcpyHostToDevice, s));
    check_obs(h, h->o_kf.p, h->o_lm.p, h->o_w_raw.p, El, std::max(Pl, 1), "ccm_ba_create: negative information weight");
  }
  k_shift<<<div_up((long long)Pl + 1, TPB), TPB, 0, s>>>(st.g_ptr.p + h->L0, (long long)Pl + 1, (int)h->E0, h->lm_ptr.p);
  CCM_LAUNCHED();
  return all;
}

// the shard's points and the buffers of its flagged weights
void shard_storage(ccm_ba_handle* h, const ccm_ba_problem* p) {
  cudaStream_t s = h->stream;
  const int Pl = h->Pl, El = h->El;
  h->Ep = ((size_t)El + 31) / 32 * 32;
  h->pt0.alloc(std::max((size_t)Pl * 3, (size_t)1));
  if (Pl) CCM_CUDA(cudaMemcpyAsync(h->pt0.p, p->points + 3 * (size_t)h->L0, sizeof(double) * 3 * Pl, cudaMemcpyHostToDevice, s));
  h->ptA.alloc(std::max((size_t)Pl * 3, (size_t)1)); h->ptB.alloc(std::max((size_t)Pl * 3, (size_t)1));
  h->o_w.alloc(std::max(El, 1)); h->d_flags.alloc(std::max(El, 1));
}

// covisibility bitmap over ALL observations (every rank needs the global pattern of S), its per-word prefix and the blocks per row
void covisibility_bitmap(ccm_ba_handle* h, const ObsLists& all, Setup& st) {
  cudaStream_t s = h->stream;
  const int Kf = h->Kf, E = h->E;
  const int words = h->words = std::max((Kf + 31) / 32, 1);
  h->bitmap.alloc_zero((size_t)std::max(Kf, 1) * words, s);
  h->word_prefix.alloc((size_t)std::max(Kf, 1) * words);
  st.row_count.alloc(std::max(Kf, 1));
  if (Kf > 0) {
    if (E > 0) {
      k_pattern_bitmap<<<div_up(E, TPB), TPB, 0, s>>>(all.kf, all.lm, all.ptr, h->pose_slot.p, E, words, h->bitmap.p);
      CCM_LAUNCHED();
    }
    k_set_diag_bits<<<div_up(Kf, TPB), TPB, 0, s>>>(Kf, words, h->bitmap.p);
    CCM_LAUNCHED();
    k_row_prefix<<<div_up(Kf, TPB), TPB, 0, s>>>(h->bitmap.p, Kf, words, h->word_prefix.p, st.row_count.p);
    CCM_LAUNCHED();
  }
}

struct Pattern { std::vector<int> rowptr, udiag; };   // block rows of S, and each row's first upper block (its diagonal)

// the block-CSR pattern of S, then the upper-block numbering, mirror map and diagonal positions: O(1) per pattern entry through the
// bitmap prefix, on the device
Pattern s_pattern(ccm_ba_handle* h, Setup& st) {
  cudaStream_t s = h->stream;
  const int Kf = h->Kf, words = h->words;
  Pattern pat{std::vector<int>((size_t)Kf + 1, 0), std::vector<int>(std::max(Kf, 1), 0)};
  std::vector<int> &h_rowptr = pat.rowptr, &h_udiag = pat.udiag;
  if (Kf > 0) {
    std::vector<int> cnt(Kf);
    st.row_count.download(cnt.data(), Kf, s);
    CCM_CUDA(cudaStreamSynchronize(s));
    long long run = 0;
    for (int a = 0; a < Kf; a++) { h_rowptr[a] = (int)run; run += cnt[a]; CCM_REQUIRE(run < (1ll << 31), "S pattern too large"); }
    h_rowptr[Kf] = (int)run;
  }
  h->nnzb = h_rowptr[Kf];
  const long long nnzb = h->nnzb;
  upload_vec(h->s_rowptr, h_rowptr, s);
  h->s_col.alloc(std::max<long long>(nnzb, 1)); h->s_row.alloc(std::max<long long>(nnzb, 1));
  if (Kf > 0) {
    k_fill_cols<<<div_up((long long)Kf * words, TPB), TPB, 0, s>>>(h->bitmap.p, h->word_prefix.p, h->s_rowptr.p, Kf, words,
                                                                  h->s_col.p, h->s_row.p);
    CCM_LAUNCHED();
  }
  h->s_diag.alloc(std::max(Kf, 1)); h->u_diag.alloc(std::max(Kf, 1)); h->csr_u.alloc(std::max<long long>(nnzb, 1));
  if (Kf > 0) {
    DevBuf<int> upper_count, u_rowstart, perr;
    upper_count.alloc(Kf); perr.alloc_zero(1, s);
    k_diag_pos<<<div_up(Kf, TPB), TPB, 0, s>>>(h->bitmap.p, h->word_prefix.p, h->s_rowptr.p, Kf, words, h->s_diag.p, upper_count.p);
    CCM_LAUNCHED();
    std::vector<int> cnt(Kf), h_ustart((size_t)Kf + 1, 0);
    upper_count.download(cnt.data(), Kf, s);
    CCM_CUDA(cudaStreamSynchronize(s));
    for (int a2 = 0; a2 < Kf; a2++) { h_ustart[a2 + 1] = h_ustart[a2] + cnt[a2]; h_udiag[a2] = h_ustart[a2]; }
    h->nub = h_ustart[Kf];
    upload_vec(u_rowstart, h_ustart, s);
    h->u_diag.upload(h_udiag.data(), Kf, s);
    h->u_row.alloc(std::max(h->nub, 1)); h->u_col.alloc(std::max(h->nub, 1));
    k_upper_index<<<div_up(nnzb, TPB), TPB, 0, s>>>(h->s_row.p, h->s_col.p, nnzb, h->bitmap.p, h->word_prefix.p, h->s_rowptr.p, words,
                                                    h->s_diag.p, u_rowstart.p, h->csr_u.p, h->u_row.p, h->u_col.p, perr.p);
    CCM_LAUNCHED();
    int e1 = 0;
    perr.download(&e1, 1, s);
    CCM_CUDA(cudaStreamSynchronize(s));  // also keeps the host vectors alive until their uploads are done
    CCM_REQUIRE(e1 == 0, "internal: asymmetric covisibility pattern");
  } else {
    h->u_row.alloc(1); h->u_col.alloc(1);
  }
  return pat;
}

// Schur product lists (local shard) and their offsets, in landmark order: the local observations grouped by block row (a stable radix
// sort keeps landmark order inside a row), then one warp per row counts, and after the scan fills, its blocks' lists (k_row_products)
std::vector<unsigned> product_lists(ccm_ba_handle* h, Setup& st) {
  cudaStream_t s = h->stream;
  const int Kf = h->Kf, El = h->El, nub = h->nub;
  std::vector<unsigned> h_pp((size_t)nub + 1, 0);
  st.cursor.alloc_zero(std::max(nub, 1), s);
  auto row_products = [&](int fill, const unsigned* u_prod_ptr, uint2* prod) {
    k_row_products<<<div_up((long long)Kf * 32, 128), 128, 0, s>>>(st.row_obs.p, st.row_obs_ptr.p, Kf, h->o_kf.p, h->o_lm.p, h->lm_ptr.p,
                                                                   h->pose_slot.p, h->bitmap.p, h->word_prefix.p, h->s_rowptr.p,
                                                                   h->s_diag.p, h->u_diag.p, nub, h->words, fill, st.cursor.p,
                                                                   u_prod_ptr, prod);
    CCM_LAUNCHED();
  };
  if (El && nub) {
    {
      DevBuf<int> key, idx, key_s;
      key.alloc(El); idx.alloc(El); key_s.alloc(El); st.row_obs.alloc(El); st.row_obs_ptr.alloc((size_t)Kf + 1);
      k_row_keys<<<div_up(El, TPB), TPB, 0, s>>>(h->o_kf.p, h->pose_slot.p, El, Kf, key.p, idx.p);
      CCM_LAUNCHED();
      int bits = 1;
      while ((1ll << bits) <= Kf) bits++;
      size_t tb = 0;
      CCM_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, tb, key.p, key_s.p, idx.p, st.row_obs.p, El, 0, bits, s));
      DevBuf<unsigned char> tmp; tmp.alloc(tb + 16);
      CCM_CUDA(cub::DeviceRadixSort::SortPairs(tmp.p, tb, key.p, key_s.p, idx.p, st.row_obs.p, El, 0, bits, s));
      k_lm_ptr<<<div_up((long long)Kf + 1, TPB), TPB, 0, s>>>(key_s.p, El, Kf, st.row_obs_ptr.p);   // first observation of each row
      CCM_LAUNCHED();
      CCM_CUDA(cudaStreamSynchronize(s));   // the temporaries die here
    }
    row_products(0, nullptr, nullptr);
    std::vector<unsigned> c(nub);
    st.cursor.download(c.data(), nub, s);
    CCM_CUDA(cudaStreamSynchronize(s));
    unsigned long long run = 0;
    for (int u = 0; u < nub; u++) { h_pp[u] = (unsigned)run; run += c[u]; }
    CCM_REQUIRE(run < (1ull << 32), "too many Schur products for 32-bit offsets");
    h_pp[nub] = (unsigned)run;
  }
  h->nprod = h_pp[nub];
  upload_vec(h->u_prod_ptr, h_pp, s);
  h->prod.alloc(std::max<long long>(h->nprod, 1));
  if (h->nprod) {
    CCM_CUDA(cudaMemsetAsync(st.cursor.p, 0, sizeof(unsigned) * nub, s));
    row_products(1, h->u_prod_ptr.p, h->prod.p);
  }
  return h_pp;
}

// k_schur_mma's schedule: per row its upper blocks by decreasing list length (ties by block number), cut into tasks of at most
// SCHUR_TASK blocks of similar size
void schur_schedule(ccm_ba_handle* h, const std::vector<int>& udiag, const std::vector<unsigned>& pp) {
  cudaStream_t s = h->stream;
  const int Kf = h->Kf, nub = h->nub;
  std::vector<int> sched((size_t)std::max(nub, 1)), tptr(1, 0);
  for (int a = 0; a < Kf; a++) {
    const int ub = udiag[a], n = (a + 1 < Kf ? udiag[a + 1] : nub) - ub;
    int* r = sched.data() + ub;
    std::iota(r, r + n, ub);
    std::sort(r, r + n, [&](int x, int y) {
      const unsigned nx = pp[x + 1] - pp[x], ny = pp[y + 1] - pp[y];
      return nx != ny ? nx > ny : x < y;
    });
    const int parts = (n + SCHUR_TASK - 1) / SCHUR_TASK;
    for (int k = 1; k <= parts; k++) tptr.push_back(ub + (int)((long long)n * k / parts));
  }
  h->ntasks = (int)tptr.size() - 1;
  upload_vec(h->u_sched, sched, s);
  upload_vec(h->task_ptr, tptr, s);
  h->next_task.alloc(1);
  int per_sm = 0;
  CCM_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, (const void*)k_schur_mma, SCHUR_CTA, 0));
  CCM_REQUIRE(per_sm >= 1, "k_schur_mma does not fit on an SM");
  h->schur_grid = std::max(1, std::min(h->ntasks, sm_count()));
  CCM_CUDA(cudaStreamSynchronize(s));   // the host vectors die at the end of this scope
}

// measurements: wait for their copy (one rank, E > 0), validate the weights there, apply the edge flags
void measurements(ccm_ba_handle* h, const ccm_ba_problem* p, const Setup& st) {
  if (st.meas) {
    CCM_CUDA(cudaStreamWaitEvent(h->stream, st.meas_done, 0));
    check_obs(h, h->o_kf.p, h->o_lm.p, h->o_w_raw.p, h->El, std::max(h->P, 1), "ccm_ba_create: negative information weight");
  }
  apply_edge_flags(h, p->edge_flags != nullptr);
}

// packed per-pose observation stream for the pose pass
void pose_obs_stream(ccm_ba_handle* h, const std::vector<int>& udiag, const std::vector<unsigned>& pp) {
  const int Kf = h->Kf;
  std::vector<unsigned> kp((size_t)Kf + 1, 0);
  for (int a = 0; a < Kf; a++) kp[a + 1] = kp[a] + (pp[udiag[a] + 1] - pp[udiag[a]]);
  upload_vec(h->kobs_ptr, kp, h->stream);
  h->kobs.alloc(std::max((size_t)kp[Kf], (size_t)1));
  pack_pose_obs(h);
}

// landmark-aligned CTA schedule: unit heads (ba_kernels.cuh), numbered by an inclusive scan, cut where a head starts; and the grids
// of k_linearize and k_backsub_points over it
void landmark_units(ccm_ba_handle* h) {
  cudaStream_t s = h->stream;
  const int Pl = h->Pl;
  h->nunits = 0;
  if (Pl > 0) {
    DevBuf<int> head, rank;
    head.alloc(Pl); rank.alloc(Pl);
    k_lin_heads<<<div_up(Pl, TPB), TPB, 0, s>>>(h->lm_ptr.p, Pl, head.p);
    CCM_LAUNCHED();
    size_t tb = 0;
    CCM_CUDA(cub::DeviceScan::InclusiveSum(nullptr, tb, head.p, rank.p, Pl, s));
    DevBuf<unsigned char> tmp; tmp.alloc(tb + 16);
    CCM_CUDA(cub::DeviceScan::InclusiveSum(tmp.p, tb, head.p, rank.p, Pl, s));
    h->units.alloc((size_t)Pl + 1);
    k_unit_ptr<<<div_up(Pl, TPB), TPB, 0, s>>>(head.p, rank.p, Pl, h->units.p);   // units[rank - 1] = head, units[nunits] = Pl
    CCM_LAUNCHED();
    CCM_CUDA(cudaMemcpyAsync(&h->nunits, rank.p + (Pl - 1), sizeof(int), cudaMemcpyDeviceToHost, s));
    CCM_CUDA(cudaStreamSynchronize(s));   // nunits sizes the grids; the temporaries die here
  } else {
    h->units.alloc_zero(1, s);
  }
  int per_sm_lin = 0, per_sm_bs = 0;
  CCM_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm_lin, (const void*)k_linearize, LIN_TILE, 0));
  CCM_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm_bs, (const void*)k_backsub_points, LIN_TILE, 0));
  h->lin_grid = std::max(1, std::min(h->nunits, sm_count() * std::max(per_sm_lin, 1)));
  h->bs_grid = std::max(1, std::min(h->nunits, sm_count() * std::max(per_sm_bs, 1)));
}

// linear-system storage and the PCG's shape, then k_pcg2's set-up
void system_storage(ccm_ba_handle* h, const std::vector<int>& rowptr) {
  cudaStream_t s = h->stream;
  const int Kf = h->Kf, Pl = h->Pl, El = h->El, nub = h->nub;
  h->Z.alloc(std::max((size_t)El * 18, (size_t)2));
  h->HllBl.alloc(std::max((size_t)Pl * 9, (size_t)1)); h->gvec.alloc(std::max((size_t)Pl * 3, (size_t)1));
  h->Hbuf.alloc_zero((size_t)Kf * 42 + 2, s);
  h->Ubuf.alloc_zero((size_t)nub * 36 + (size_t)Kf * 6 + 1, s);
  h->s_val.alloc(std::max<long long>(h->nnzb * 36, 1)); h->Minv.alloc(std::max((size_t)Kf * 36, (size_t)1));
  h->bschur.alloc(std::max((size_t)Kf * 6, (size_t)1));
  // coarse space: <= 128 aggregates for small systems, <= 384 for long trajectories where the smooth modes dominate the
  // iteration count; the inverse is refreshed every 2nd solve (measured sweeps: tools/ba_probe.py with CCM_PCG_NC/REFRESH)
  // CCM_PCG_PROLONG=1: piecewise-linear prolongation (pcg.cuh); half the coarse nodes then already beat the constant P
  const int prolong = env_int("CCM_PCG_PROLONG", 1) ? 1 : 0;  // cfg5: 1538 -> 617 PCG iterations per Global BA at 192 coarse nodes
  // PCG iterations per Global BA on cfg5: NC 192 refresh 4: 617, NC 192 refresh 2: 545, NC 256 refresh 2: 400, NC 256 refresh 1: 384,
  // NC 384 refresh 4: 357 (its 2304^2 inverse is the most expensive), NC 128 refresh 1: 1014; refresh 8 (one inverse per BA): 1950
  // From Kf >= 8192 (cfg5: Kf = 9999) 320 nodes: an iteration of k_pcg2 there costs about 110 us, so the iterations a larger coarse
  // space saves outweigh its dearer inverse; below that the iterations are cheaper and 256 nodes stay the better trade.
  h->pcg.shape(Kf, env_int("CCM_PCG_NC", Kf >= 4096 ? (prolong ? (Kf >= 8192 ? 320 : 256) : 384) : 128), prolong);
  // the PCG's vectors follow the system's directly: allocated after dxl, the same code ran cfg5 1.2 % slower (H100 80GB HBM3, 700 W)
  h->pcg.alloc({h->s_rowptr.p, h->s_col.p, h->s_val.p, h->Minv.p, h->bschur.p}, s);
  h->dxl.alloc(std::max((size_t)Pl * 3, (size_t)1));
  h->jac_fail.alloc_zero(1, s);
  if (env_int("CCM_PCG_PROF", 0)) h->pcg_prof.alloc_zero(8, s);
  // refresh 1 / 2 / 4 with NC 256: 384 / 400 / 496 iterations per cfg5 Global BA.  An iteration of k_pcg2 costs about 120 us and
  // the set-up launch that rebuilds the 1536^2 inverse 2.0 ms, so one BA takes 173 / 167 / 174 ms; cfg4 (k_pcg, nC = 690) takes
  // 27.3 / 24.5 ms at refresh 1 / 2 (H100 80GB HBM3, 700 W).  Every size rebuilds every 2nd solve.
  // cfg5, one Global BA (8 LM trials, median of 3; H100 80GB HBM3, 700 W), NC x refresh -> PCG iterations, ms:
  //   256 / 2: 400, 167.5   320 / 2: 262, 157.1   384 / 2: 212, 160.3
  //   256 / 1: 384, 172.9   320 / 1: 246, 168.7   384 / 1: 197, 179.9
  h->pcg_refresh = std::max(1, env_int("CCM_PCG_REFRESH", 2));
  setup_pcg2(h, rowptr);
  h->partials.alloc((size_t)std::max({sm_count() * 8 + 8, h->lin_grid, h->bs_grid}));
  h->scal.alloc_zero(16, s);
  h->rep_chi2.alloc(std::max(El, 1)); h->rep_depth.alloc(std::max(El, 1));
}

// the estimate the caller gave, as the current and the trial state
void initial_state(ccm_ba_handle* h) {
  cudaStream_t s = h->stream;
  h->pose_cur = h->poseA.p; h->pose_trial = h->poseB.p; h->pt_cur = h->ptA.p; h->pt_trial = h->ptB.p;
  CCM_CUDA(cudaMemcpyAsync(h->pose_trial, h->pose0.p, h->pose0.bytes(), cudaMemcpyDeviceToDevice, s));
  if (h->Pl) CCM_CUDA(cudaMemcpyAsync(h->pt_trial, h->pt0.p, sizeof(double) * 3 * h->Pl, cudaMemcpyDeviceToDevice, s));
  do_reset(h);
  h->device_bytes = (int64_t)(h->Z.bytes() + h->prod.bytes() + h->s_val.bytes() + h->Ubuf.bytes() +
                              h->bitmap.bytes() + h->word_prefix.bytes() + h->HllBl.bytes() + h->o_kf.bytes() * 2 +
                              h->o_uv.bytes() + h->o_w.bytes() * 2 + h->ptA.bytes() * 3);
}

void build(ccm_ba_handle* h, const ccm_ba_problem* p) {
  const double T0 = now_ms();
  open_handle(h, p);
  // CCM_SETUP_PROF=1: wall time of the set-up phases on stderr (each lap synchronises the stream: diagnostics only)
  const bool sprof = env_int("CCM_SETUP_PROF", 0) != 0;
  double t_lap = now_ms();
  auto lap = [&](const char* what) {
    if (!sprof) return;
    cudaStreamSynchronize(h->stream);
    const double t = now_ms();
    fprintf(stderr, "[ccm_ba_create r%d] %-28s %8.2f ms\n", h->rank, what, t - t_lap);
    t_lap = t;
  };
  Setup st;
  free_pose_slots(h, p);
  const ObsLists all = take_observations(h, p, st);
  map_edge_flags(h, p->edge_flags);   // host work while the measurements are still on their way (one rank)
  lap("observations + shard");
  shard_storage(h, p);
  covisibility_bitmap(h, all, st);
  lap("points, flags, bitmap, prefix");
  const Pattern pat = s_pattern(h, st);
  lap("pattern, upper index");
  const std::vector<unsigned> pp = product_lists(h, st);
  schur_schedule(h, pat.udiag, pp);
  lap("product lists");
  measurements(h, p, st);
  pose_obs_stream(h, pat.udiag, pp);
  lap("pose observation stream");
  landmark_units(h);
  system_storage(h, pat.rowptr);
  initial_state(h);
  lap("storage + initial state");
  h->t_setup_ms = now_ms() - T0;
}

void download_state(ccm_ba_handle* h, ccm_ba_result* r) {
  cudaStream_t s = h->stream;
  if (r->poses) CCM_CUDA(cudaMemcpyAsync(r->poses, h->pose_cur, sizeof(double) * 7 * h->K, cudaMemcpyDeviceToHost, s));
  if (r->points && h->P) {
    if (h->nranks == 1) {
      CCM_CUDA(cudaMemcpyAsync(r->points, h->pt_cur, sizeof(double) * 3 * h->Pl, cudaMemcpyDeviceToHost, s));
    } else {  // every rank returns the full point set: scatter own shard into a zeroed P*3 buffer and all-reduce
      DevBuf<double> full; full.alloc_zero((size_t)h->P * 3, s);
      if (h->Pl) CCM_CUDA(cudaMemcpyAsync(full.p + 3 * (size_t)h->L0, h->pt_cur, sizeof(double) * 3 * h->Pl, cudaMemcpyDeviceToDevice, s));
      allreduce_f64(full.p, (size_t)h->P * 3, 0, s);
      full.download(r->points, (size_t)h->P * 3, s);
      CCM_CUDA(cudaStreamSynchronize(s));
    }
  }
  if ((r->chi2 || r->depth_pos) && h->El) {
    k_edge_report<<<div_up(h->El, TPB), TPB, 0, s>>>(h->o_kf.p, h->o_lm.p, h->o_uv.p, h->o_w_raw.p, h->pose_eval, h->pt_eval,
                                                     h->pose_cur, h->pt_cur, h->intr.p, h->El, h->rep_chi2.p, h->rep_depth.p);
    CCM_LAUNCHED();
    std::vector<double> c(h->El);
    std::vector<uint8_t> d(h->El);
    h->rep_chi2.download(c.data(), h->El, s); h->rep_depth.download(d.data(), h->El, s);
    CCM_CUDA(cudaStreamSynchronize(s));
    for (int i = 0; i < h->El; i++) {
      const long long e = input_edge(h, h->E0 + i);
      if (r->chi2 && !(h->h_flags[i] & 1)) r->chi2[e] = c[i];
      if (r->depth_pos) r->depth_pos[e] = d[i];
    }
  }
  CCM_CUDA(cudaStreamSynchronize(s));
}

void optimize(ccm_ba_handle* h, const ccm_ba_options* o, ccm_ba_result* r) {
  CCM_CUDA(cudaSetDevice(h->device));
  const double T0 = now_ms();
  cudaStream_t s = h->stream;
  struct EventPair {  // device-side bracket of the whole LM loop; destroyed on every exit path
    cudaEvent_t a = nullptr, b = nullptr;
    ~EventPair() { if (a) cudaEventDestroy(a); if (b) cudaEventDestroy(b); }
  } ev;
  CCM_CUDA(cudaEventCreate(&ev.a)); CCM_CUDA(cudaEventCreate(&ev.b));
  cudaEvent_t evA = ev.a, evB = ev.b;
  CCM_CUDA(cudaEventRecord(evA, s));
  const int robust = o->robust ? 1 : 0;
  const double delta = o->huber_delta;
  const int max_trials = o->max_trials > 0 ? o->max_trials : 10;
  const int pcg_max = o->pcg_max_iter > 0 ? o->pcg_max_iter : 2000;
  // 1e-8: measured against the exact-factorisation oracle the estimates then differ by ~2e-10 relative (cfg4) and by 1e-10
  // from a 1e-13 solve on cfg5 (tools/tol_probe.py) -- far below the f32 the reference writes results back in
  const double pcg_tol = o->pcg_tol > 0 ? o->pcg_tol : 1e-8;
  h->pcg_coarse_valid = false;  // every optimize() starts with a fresh coarse inverse
  r->trace_len = 0; r->iters_done = 0; r->trials_total = 0; r->pcg_iters_total = 0; r->pcg_not_converged = 0;
  r->chi2_initial = r->chi2_final = 0; r->lambda_final = 0;
  // force-stop flag (g2o terminate()): read locally on one rank; on several ranks the decision is collective (it rides in the
  // per-trial all-reduce, plus one all-reduce before the first iteration)
  auto stop_local = [&]() { return o->stop && *o->stop; };
  bool stop_all = false;
  if (h->nranks > 1) {
    h->h_scal[12] = stop_local() ? 1.0 : 0.0;
    CCM_CUDA(cudaMemcpyAsync(h->scal.p + 3, h->h_scal + 12, sizeof(double), cudaMemcpyHostToDevice, s));
    allreduce_f64(h->scal.p + 3, 1, 2, s);
    CCM_CUDA(cudaMemcpyAsync(h->h_scal + 13, h->scal.p + 3, sizeof(double), cudaMemcpyDeviceToHost, s));
    CCM_CUDA(cudaStreamSynchronize(s));
    stop_all = h->h_scal[13] > 0.0;
  }
  auto terminate = [&]() { return h->nranks > 1 ? stop_all : stop_local(); };
  int ret_iters = 0;
  if (h->Kf == 0 || h->E == 0) {
    // g2o: landmarks-only graphs are still optimised, but every cslam call site has free poses; keep it simple
    ret_iters = h->E == 0 ? -1 : 0;
  }
  LmSchedule lm{max_trials};
  for (int it = 0; h->Kf > 0 && h->E > 0 && it < o->iterations && !terminate(); it++) {
    // from the second iteration on lambda is known before the linearisation, which then forms Z as well; the first iteration takes
    // lambda from the diagonal it has just built and forms Z in a second, Z-only pass
    step_linearize(h, robust, delta, it == 0 ? 0 : LIN_Z, lm.lambda);
    if (it == 0) {
      const double maxdiag = step_max_diag(h);
      if (!(maxdiag > 0.0)) {  // every edge is inactive (weight 0): nothing to optimise, the estimate is left alone
        ret_iters = -1;
        break;
      }
      lm.start(o->lambda_init, maxdiag);
      lm.begin_iteration(h->h_scal[8]);
      r->chi2_initial = lm.currentChi;
      step_z(h, robust, delta, lm.lambda);
    } else {
      lm.begin_iteration(read_chi2_cur(h));
    }
    do {
      if (lm.qmax > 0) step_z(h, robust, delta, lm.lambda);   // the trial before was rejected: same estimate, larger lambda
      step_schur(h);
      step_finalize(h, lm.lambda);
      step_pcg(h, pcg_tol, pcg_max);
      step_update_and_residual(h, lm.lambda, robust, delta, nullptr, stop_local());
      CCM_CUDA(cudaMemcpyAsync(h->h_scal, h->scal.p, 3 * sizeof(double), cudaMemcpyDeviceToHost, s));
      if (h->nranks > 1) CCM_CUDA(cudaMemcpyAsync(h->h_scal + 13, h->scal.p + 3, sizeof(double), cudaMemcpyDeviceToHost, s));
      CCM_CUDA(cudaMemcpyAsync(h->h_scal + 3, h->pcg.status.p, 4 * sizeof(double), cudaMemcpyDeviceToHost, s));
      CCM_CUDA(cudaMemcpyAsync(h->h_scal + 7, h->jac_fail.p, sizeof(int), cudaMemcpyDeviceToHost, s));
      CCM_CUDA(cudaStreamSynchronize(s));
      if (h->profile) collect_spans(h);
      if (h->nranks > 1) stop_all = h->h_scal[13] > 0.0;
      const int pcg_it = (int)h->h_scal[3];
      const int pcg_flag = (int)h->h_scal[5];
      int jfail;
      memcpy(&jfail, h->h_scal + 7, sizeof(int));
      if (h->pcg_last_mode == 1) { h->pcg_coarse_valid = h->h_scal[6] > 0; h->pcg_age = 1; } else h->pcg_age++;
      r->pcg_iters_total += pcg_it;
      if (pcg_flag == 1) r->pcg_not_converged++;
      if (pcg_flag == 3) throw Error(CCM_ERR_NCCL, "distributed PCG: a peer's packet did not arrive within CCM_PCG_DIST_TIMEOUT_MS");
      const bool solved = !(pcg_flag == 2 || jfail);  // linear solve failed (not SPD): the trial is rejected
      if (lm.trial(h->h_scal[0], h->h_scal[1] + h->h_scal[2], solved, pcg_it, h->h_scal[4])) {  // rejected: pop, the estimate stays
        std::swap(h->pose_cur, h->pose_trial);  // discardTop: the trial state becomes the estimate
        std::swap(h->pt_cur, h->pt_trial);
      }
      r->trials_total++;
    } while (lm.retry() && !terminate());
    ret_iters++;
    if (lm.end_iteration(r, it)) break;
  }
  r->iters_done = ret_iters;
  CCM_CUDA(cudaEventRecord(evB, s));
  CCM_CUDA(cudaStreamSynchronize(s));
  if (h->profile) collect_spans(h);
  r->t_optimize_ms = now_ms() - T0;
  {
    float ms = 0.f;
    cudaEventElapsedTime(&ms, evA, evB);
    r->t_optimize_event_ms = ms;
  }
  const double T1 = now_ms();
  download_state(h, r);
  r->t_download_ms = now_ms() - T1;
  r->t_setup_ms = h->t_setup_ms;
}

}  // namespace

// ---- C ABI ------------------------------------------------------------------------------------------------------
extern "C" int ccm_ba_create(const ccm_ba_problem* p, ccm_ba_handle** out) {
  return guarded([&] {
    CCM_REQUIRE(out, "ccm_ba_create: out is NULL");
    *out = nullptr;
    ccm_ba_handle* h = new ccm_ba_handle();
    try {
      build(h, p);
    } catch (...) {
      cudaDeviceSynchronize();  // in-flight kernels must not outlive the buffers that go back to the pool
      delete h;
      throw;
    }
    *out = h;
  });
}

extern "C" void ccm_ba_destroy(ccm_ba_handle* h) {
  if (!h) return;
  cudaSetDevice(h->device);
  if (h->stream) cudaStreamSynchronize(h->stream);  // nothing may still use the buffers that go back to the pool
  delete h;
}

extern "C" int ccm_ba_reset(ccm_ba_handle* h) {
  return guarded([&] { CCM_REQUIRE(h, "null handle"); CCM_CUDA(cudaSetDevice(h->device)); do_reset(h); });
}

extern "C" int ccm_ba_set_estimate(ccm_ba_handle* h, const double* poses, const double* points) {
  return guarded([&] {
    CCM_REQUIRE(h, "null handle");
    CCM_CUDA(cudaSetDevice(h->device));
    cudaStream_t s = h->stream;
    if (poses) CCM_CUDA(cudaMemcpyAsync(h->pose0.p, poses, sizeof(double) * 7 * (size_t)h->K, cudaMemcpyHostToDevice, s));
    if (points && h->Pl) CCM_CUDA(cudaMemcpyAsync(h->pt0.p, points + 3 * (size_t)h->L0, sizeof(double) * 3 * (size_t)h->Pl, cudaMemcpyHostToDevice, s));
    do_reset(h);   // the new values become the current estimate (synchronises the stream: the caller's buffers are free again)
  });
}

extern "C" int ccm_ba_set_edge_flags(ccm_ba_handle* h, const uint8_t* edge_flags) {
  return guarded([&] {
    CCM_REQUIRE(h, "null handle");
    CCM_CUDA(cudaSetDevice(h->device));
    map_edge_flags(h, edge_flags);
    apply_edge_flags(h, edge_flags != nullptr);
    pack_pose_obs(h);
    CCM_CUDA(cudaStreamSynchronize(h->stream));
  });
}

extern "C" int ccm_ba_optimize(ccm_ba_handle* h, const ccm_ba_options* o, ccm_ba_result* r) {
  return guarded([&] { CCM_REQUIRE(h && o && r, "null argument"); optimize(h, o, r); });
}

extern "C" int ccm_ba_solve(const ccm_ba_problem* p, const ccm_ba_options* o, ccm_ba_result* r) {
  const bool sprof = env_int("CCM_SETUP_PROF", 0) != 0;
  const double t0 = now_ms();
  ccm_ba_handle* h = nullptr;
  int rc = ccm_ba_create(p, &h);
  if (rc != CCM_OK) return rc;
  const double t1 = now_ms();
  rc = ccm_ba_optimize(h, o, r);
  const double t2 = now_ms();
  ccm_ba_destroy(h);
  if (sprof) fprintf(stderr, "[ccm_ba_solve] create %.2f ms, optimize %.2f ms, destroy %.2f ms\n", t1 - t0, t2 - t1, now_ms() - t2);
  return rc;
}

extern "C" int ccm_ba_set_profile(ccm_ba_handle* h, int on) {
  return guarded([&] {
    CCM_REQUIRE(h, "null handle");
    h->profile = on != 0;
    for (int i = 0; i < CCM_BA_NKERNELS; i++) { h->k_ms[i] = 0; h->k_count[i] = 0; }
    h->spans.clear(); h->ev_used = 0;
  });
}

extern "C" int ccm_ba_get_kernel_stats(const ccm_ba_handle* h, double* total_ms, int64_t* launches) {
  return guarded([&] {
    CCM_REQUIRE(h && total_ms && launches, "null argument");
    for (int i = 0; i < CCM_BA_NKERNELS; i++) { total_ms[i] = h->k_ms[i]; launches[i] = h->k_count[i]; }
  });
}

extern "C" int ccm_ba_shard_range(const int32_t* obs_mp, int32_t E, int32_t P, int32_t rank, int32_t nranks, int32_t* L0,
                                   int32_t* L1, int64_t* E0, int64_t* E1) {
  return guarded([&] {  // host only: usable without a device
    CCM_REQUIRE(P >= 0 && E >= 0 && nranks >= 1 && rank >= 0 && rank < nranks && L0 && L1, "ccm_ba_shard_range: bad argument");
    std::vector<int> ptr((size_t)P + 1, 0);
    for (int e = 0; e < E; e++) { CCM_REQUIRE(obs_mp[e] >= 0 && obs_mp[e] < P, "obs_mp out of range"); ptr[obs_mp[e] + 1]++; }
    for (int l = 0; l < P; l++) ptr[l + 1] += ptr[l];
    shard_range(ptr.data(), P, rank, nranks, L0, L1);
    if (E0) *E0 = ptr[*L0];
    if (E1) *E1 = ptr[*L1];
  });
}

extern "C" int ccm_ba_debug_pcg_cycles(ccm_ba_handle* h, int64_t* cycles8) {
  return guarded([&] {
    CCM_REQUIRE(h && cycles8, "null argument");
    for (int i = 0; i < 8; i++) cycles8[i] = 0;
    if (h->pcg_prof.p) { CCM_CUDA(cudaMemcpy(cycles8, h->pcg_prof.p, 8 * sizeof(long long), cudaMemcpyDeviceToHost)); }
  });
}

extern "C" int ccm_ba_get_info(const ccm_ba_handle* h, ccm_ba_info* info) {
  return guarded([&] {
    CCM_REQUIRE(h && info, "null argument");
    info->K = h->K; info->K_free = h->Kf; info->P_local = h->Pl; info->E_local = h->El; info->rank = h->rank;
    info->nranks = h->nranks; info->s_blocks_upper = h->nub; info->s_blocks_full = h->nnzb;
    info->schur_products = h->nprod; info->device_bytes = h->device_bytes;
  });
}

extern "C" int ccm_ba_debug_build(ccm_ba_handle* h, int robust, double huber_delta, double* Hpp, double* bp, double* Hll,
                                  double* bl, double* W, double* chi2_robust_sum) {
  return guarded([&] {
    CCM_REQUIRE(h, "null handle");
    CCM_REQUIRE(h->nranks == 1, "debug entry points are single-rank");
    CCM_CUDA(cudaSetDevice(h->device));
    cudaStream_t s = h->stream;
    if (h->W.n < h->Ep * 18) h->W.alloc(std::max(h->Ep * 18, (size_t)1));   // W exists for this export only
    step_linearize(h, robust, huber_delta, 0, 0.0, h->W.p);
    const int K = h->K, Kf = h->Kf, Pl = h->Pl, El = h->El;
    std::vector<double> hH((size_t)Kf * 42 + 1), hL((size_t)Pl * 9), hW(h->Ep * 18);
    h->Hbuf.download(hH.data(), hH.size(), s); h->HllBl.download(hL.data(), hL.size(), s); h->W.download(hW.data(), hW.size(), s);
    CCM_CUDA(cudaStreamSynchronize(s));
    if (Hpp) memset(Hpp, 0, sizeof(double) * 36 * K);
    if (bp) memset(bp, 0, sizeof(double) * 6 * K);
    for (int a = 0; a < Kf; a++) {
      if (Hpp) memcpy(Hpp + 36 * (size_t)h->h_slot_pose[a], hH.data() + (size_t)a * 36, 36 * sizeof(double));
      if (bp) memcpy(bp + 6 * (size_t)h->h_slot_pose[a], hH.data() + (size_t)Kf * 36 + (size_t)a * 6, 6 * sizeof(double));
    }
    static const int ut[9] = {0, 1, 2, 1, 3, 4, 2, 4, 5};
    for (int l = 0; l < Pl; l++) {
      if (Hll) for (int i = 0; i < 9; i++) Hll[9 * (size_t)l + i] = hL[(size_t)ut[i] * Pl + l];
      if (bl) for (int i = 0; i < 3; i++) bl[3 * (size_t)l + i] = hL[(size_t)(6 + i) * Pl + l];
    }
    if (W)
      for (int i = 0; i < El; i++) {
        const long long e = input_edge(h, i);
        for (int c = 0; c < 18; c++) W[18 * (size_t)e + c] = hW[(size_t)c * h->Ep + i];
      }
    if (chi2_robust_sum) *chi2_robust_sum = hH[(size_t)Kf * 42];
  });
}

extern "C" int ccm_ba_debug_schur(ccm_ba_handle* h, int robust, double huber_delta, double lambda, double* S_dense,
                                  double* bschur, double* dx_pose, double* dx_point, int32_t* pcg_iters, double* pcg_relres) {
  return guarded([&] {
    CCM_REQUIRE(h, "null handle");
    CCM_REQUIRE(h->nranks == 1, "debug entry points are single-rank");
    CCM_CUDA(cudaSetDevice(h->device));
    cudaStream_t s = h->stream;
    step_linearize(h, robust, huber_delta, LIN_Z, lambda);
    step_schur(h);
    step_finalize(h, lambda);
    step_pcg(h, 1e-13, 5000);
    step_update_and_residual(h, lambda, robust, huber_delta, h->dxl.p);
    const int K = h->K, Kf = h->Kf, Pl = h->Pl;
    std::vector<double> hx((size_t)Kf * 6), hdl((size_t)Pl * 3), hb((size_t)Kf * 6), st(3);
    h->pcg.x.download(hx.data(), hx.size(), s); h->dxl.download(hdl.data(), hdl.size(), s);
    h->bschur.download(hb.data(), hb.size(), s); h->pcg.status.download(st.data(), 3, s);
    CCM_CUDA(cudaStreamSynchronize(s));
    if (pcg_iters) *pcg_iters = (int)st[0];
    if (pcg_relres) *pcg_relres = st[1];
    if (dx_pose) {
      memset(dx_pose, 0, sizeof(double) * 6 * K);
      for (int a = 0; a < Kf; a++) memcpy(dx_pose + 6 * (size_t)h->h_slot_pose[a], hx.data() + (size_t)a * 6, 6 * sizeof(double));
    }
    if (dx_point) memcpy(dx_point, hdl.data(), sizeof(double) * 3 * Pl);
    if (bschur) {
      memset(bschur, 0, sizeof(double) * 6 * K);
      for (int a = 0; a < Kf; a++) memcpy(bschur + 6 * (size_t)h->h_slot_pose[a], hb.data() + (size_t)a * 6, 6 * sizeof(double));
    }
    if (S_dense) {
      const size_t n = 6 * (size_t)K;
      memset(S_dense, 0, sizeof(double) * n * n);
      std::vector<int> rp((size_t)Kf + 1), cl(h->nnzb);
      std::vector<double> v((size_t)h->nnzb * 36);
      h->s_rowptr.download(rp.data(), rp.size(), s); h->s_col.download(cl.data(), cl.size(), s); h->s_val.download(v.data(), v.size(), s);
      CCM_CUDA(cudaStreamSynchronize(s));
      for (int a = 0; a < Kf; a++)
        for (int q = rp[a]; q < rp[a + 1]; q++) {
          const size_t gi = 6 * (size_t)h->h_slot_pose[a], gj = 6 * (size_t)h->h_slot_pose[cl[q]];
          for (int rr = 0; rr < 6; rr++)
            for (int cc = 0; cc < 6; cc++) S_dense[(gi + rr) * n + gj + cc] = v[(size_t)q * 36 + rr * 6 + cc];
        }
    }
  });
}

extern "C" int ccm_ba_debug_step(ccm_ba_handle* h, int robust, double huber_delta, double lambda, const double* dx_pose,
                                 double* pose_trial, double* pt_trial, double* dx_point, double* chi2_trial, double* scale_pose,
                                 double* scale_point) {
  return guarded([&] {
    CCM_REQUIRE(h && dx_pose, "null argument");
    CCM_REQUIRE(h->nranks == 1, "debug entry points are single-rank");
    CCM_CUDA(cudaSetDevice(h->device));
    cudaStream_t s = h->stream;
    const int K = h->K, Kf = h->Kf, Pl = h->Pl;
    std::vector<double> hx((size_t)std::max(Kf, 1) * 6, 0.0);
    for (int a = 0; a < Kf; a++) memcpy(hx.data() + (size_t)a * 6, dx_pose + 6 * (size_t)h->h_slot_pose[a], 6 * sizeof(double));
    step_linearize(h, robust, huber_delta, LIN_Z, lambda);
    if (Kf > 0) h->pcg.x.upload(hx.data(), (size_t)Kf * 6, s);
    step_update_and_residual(h, lambda, robust, huber_delta, h->dxl.p);
    std::vector<double> hp((size_t)K * 7), hq((size_t)Pl * 3), hd((size_t)Pl * 3), sc(3);
    if (K > 0) CCM_CUDA(cudaMemcpyAsync(hp.data(), h->pose_trial, hp.size() * sizeof(double), cudaMemcpyDeviceToHost, s));
    if (Pl > 0) {
      CCM_CUDA(cudaMemcpyAsync(hq.data(), h->pt_trial, hq.size() * sizeof(double), cudaMemcpyDeviceToHost, s));
      h->dxl.download(hd.data(), hd.size(), s);
    }
    h->scal.download(sc.data(), 3, s);
    CCM_CUDA(cudaStreamSynchronize(s));
    if (pose_trial) memcpy(pose_trial, hp.data(), hp.size() * sizeof(double));
    if (pt_trial) memcpy(pt_trial, hq.data(), hq.size() * sizeof(double));
    if (dx_point) memcpy(dx_point, hd.data(), hd.size() * sizeof(double));
    if (chi2_trial) *chi2_trial = sc[0];
    if (scale_point) *scale_point = sc[1];
    if (scale_pose) *scale_pose = sc[2];
  });
}

extern "C" int ccm_ba_debug_schur_blocks(ccm_ba_handle* h, int32_t* rowptr, int32_t* col, double* val, double* bschur) {
  return guarded([&] {
    CCM_REQUIRE(h, "null handle");
    CCM_REQUIRE(h->nranks == 1, "debug entry points are single-rank");
    CCM_CUDA(cudaSetDevice(h->device));
    cudaStream_t s = h->stream;
    const int K = h->K, Kf = h->Kf;
    const long long nnzb = h->nnzb;
    std::vector<int> rp((size_t)Kf + 1, 0), cl((size_t)std::max<long long>(nnzb, 1));
    std::vector<double> v((size_t)std::max<long long>(nnzb * 36, 1)), hb((size_t)std::max(Kf * 6, 1));
    if (Kf > 0) {
      h->s_rowptr.download(rp.data(), rp.size(), s);
      if (nnzb) { h->s_col.download(cl.data(), nnzb, s); h->s_val.download(v.data(), (size_t)nnzb * 36, s); }
      h->bschur.download(hb.data(), (size_t)Kf * 6, s);
    }
    CCM_CUDA(cudaStreamSynchronize(s));
    // slots are numbered in increasing pose order, so the slot-ordered rows and columns stay sorted in pose indices
    long long q = 0;
    for (int k = 0; k < K; k++) {
      if (rowptr) rowptr[k] = (int32_t)q;
      const int a = h->h_pose_slot[k];
      if (a < 0) continue;
      for (int t = rp[a]; t < rp[a + 1]; t++, q++) {
        if (col) col[q] = h->h_slot_pose[cl[t]];
        if (val) memcpy(val + (size_t)q * 36, v.data() + (size_t)t * 36, 36 * sizeof(double));
      }
    }
    if (rowptr) rowptr[K] = (int32_t)q;
    if (bschur) {
      memset(bschur, 0, sizeof(double) * 6 * (size_t)K);
      for (int a = 0; a < Kf; a++) memcpy(bschur + 6 * (size_t)h->h_slot_pose[a], hb.data() + (size_t)a * 6, 6 * sizeof(double));
    }
  });
}

extern "C" int ccm_ba_debug_coarse(ccm_ba_handle* h, double* Ac, double* Ainv) {
  return guarded([&] {
    CCM_REQUIRE(h && Ac && Ainv, "null argument");
    const int nC = h->pcg.nC();
    CCM_REQUIRE(nC > 0, "the handle has no coarse space");
    cudaStream_t s = h->stream;
    const size_t bytes = (size_t)nC * nC * sizeof(double);
    for (int mode : {3, 1}) {  // the assembled matrix, then the set-up launch step_pcg makes before k_pcg2
      h->pcg.launch(0.0, 0, mode, h->pcg_prof.p, s);
      CCM_CUDA(cudaMemcpyAsync(mode == 3 ? Ac : Ainv, mode == 3 ? h->pcg.Ac.p : coarse_inverse(h->pcg.Ac.p, nC), bytes,
                               cudaMemcpyDeviceToHost, s));
    }
    CCM_CUDA(cudaStreamSynchronize(s));
    double st[4];
    CCM_CUDA(cudaMemcpy(st, h->pcg.status.p, sizeof(st), cudaMemcpyDeviceToHost));
    CCM_REQUIRE(st[3] > 0.0, "the coarse matrix has a non-positive pivot");
  });
}

extern "C" int ccm_ba_debug_products(ccm_ba_handle* h, int32_t* blk, uint32_t* ptr, int32_t* pairs) {
  return guarded([&] {
    CCM_REQUIRE(h, "null handle");
    CCM_REQUIRE(h->nranks == 1, "debug entry points are single-rank");
    CCM_CUDA(cudaSetDevice(h->device));
    cudaStream_t s = h->stream;
    const int nub = h->nub;
    std::vector<int> ur((size_t)std::max(nub, 1)), uc((size_t)std::max(nub, 1));
    std::vector<unsigned> pp((size_t)nub + 1, 0);
    std::vector<uint2> pr((size_t)std::max<long long>(h->nprod, 1));
    if (nub) {
      h->u_row.download(ur.data(), nub, s); h->u_col.download(uc.data(), nub, s); h->u_prod_ptr.download(pp.data(), (size_t)nub + 1, s);
    }
    if (h->nprod) h->prod.download(pr.data(), (size_t)h->nprod, s);
    CCM_CUDA(cudaStreamSynchronize(s));
    for (int u = 0; u < nub; u++) {
      if (blk) { blk[2 * (size_t)u] = h->h_slot_pose[ur[u]]; blk[2 * (size_t)u + 1] = h->h_slot_pose[uc[u]]; }
      if (ptr) ptr[u] = pp[u];
    }
    if (ptr) ptr[nub] = pp[nub];
    if (pairs)
      for (long long q = 0; q < h->nprod; q++) {
        pairs[2 * q] = (int32_t)(h->E0 + pr[q].x);
        pairs[2 * q + 1] = (int32_t)(h->E0 + pr[q].y);
      }
  });
}

extern "C" int ccm_ba_debug_schedule(ccm_ba_handle* h, int32_t* counts, int32_t* task_ptr, int32_t* sched) {
  return guarded([&] {
    CCM_REQUIRE(h, "null handle");
    CCM_CUDA(cudaSetDevice(h->device));
    cudaStream_t s = h->stream;
    if (counts) { counts[0] = h->ntasks; counts[1] = h->schur_grid; }
    if (task_ptr) h->task_ptr.download(task_ptr, (size_t)h->ntasks + 1, s);
    if (sched && h->nub) h->u_sched.download(sched, (size_t)h->nub, s);
    CCM_CUDA(cudaStreamSynchronize(s));
  });
}

extern "C" int ccm_ba_debug_pcg2(ccm_ba_handle* h, int64_t* counts, int32_t* items, int32_t* cta_row, int32_t* cta_item, int32_t* slab_lo) {
  return guarded([&] {
    CCM_REQUIRE(h, "null handle");
    CCM_REQUIRE(h->p2.on, "the handle does not run k_pcg2");
    CCM_CUDA(cudaSetDevice(h->device));
    cudaStream_t s = h->stream;
    const ccm_ba_handle::Pcg2& d = h->p2;
    if (counts) { counts[0] = d.nitems; counts[1] = d.grid; counts[2] = d.streamed; }
    if (items && d.nitems) d.items.download(items, (size_t)d.nitems * P2_REC, s);
    if (cta_row) d.cta_row.download(cta_row, (size_t)d.grid + 1, s);
    if (cta_item) d.cta_item.download(cta_item, (size_t)d.grid + 1, s);
    if (slab_lo) d.slab_lo.download(slab_lo, (size_t)d.grid * P2_W, s);
    CCM_CUDA(cudaStreamSynchronize(s));
  });
}

extern "C" int ccm_ba_debug_paths(ccm_ba_handle* h, int32_t* out) {
  return guarded([&] {
    CCM_REQUIRE(h && out, "null argument");
    out[0] = h->p2.on ? 2 : 1;
    out[1] = h->pcg.block;
    out[2] = h->pcg.agg;
    out[3] = h->pcg.nc;
  });
}

extern "C" int ccm_ba_time_kernel(ccm_ba_handle* h, int which, int reps, double huber_delta, double lambda, double* ms_per_launch) {
  return guarded([&] {
    CCM_REQUIRE(h && ms_per_launch && reps > 0, "bad argument");
    CCM_CUDA(cudaSetDevice(h->device));
    cudaStream_t s = h->stream;
    // make sure every input of the timed kernel exists
    step_linearize(h, 1, huber_delta, LIN_Z, lambda);
    step_schur(h);
    step_finalize(h, lambda);
    step_pcg(h, 1e-10, 2000);
    cudaEvent_t e0, e1;
    CCM_CUDA(cudaEventCreate(&e0)); CCM_CUDA(cudaEventCreate(&e1));
    float total = 0.f;
    for (int i = 0; i < reps; i++) {
      CCM_CUDA(cudaEventRecord(e0, s));
      switch (which) {
        case 0:
          launch_linearize(h, 1, huber_delta, LIN_H | LIN_Z, lambda);
          break;
        case 1:
          k_pose_pass<<<h->Kf, 128, 0, s>>>(h->kobs.p, h->kobs_ptr.p, h->slot_pose.p, h->pose_cur, h->intr.p, h->pt_cur, 1, huber_delta,
                                            h->Hpp(), h->bp());
          break;
        case 2:
          k_residual<<<grid_stride(h->El), TPB, 0, s>>>(h->o_kf.p, h->o_lm.p, h->o_uv.p, h->o_w.p, h->pose_cur, h->intr.p,
                                                        h->pt_cur, h->El, 1, huber_delta, h->partials.p);
          break;
        case 3:
          launch_linearize(h, 1, huber_delta, LIN_Z, lambda);
          break;
        case 4:
          launch_schur(h, s);
          break;
        case 5:
          launch_backsub(h, lambda, nullptr);
          break;
        case 6: {
          step_pcg(h, 1e-10, 2000);
          break;
        }
        default:
          throw Error(CCM_ERR_INVALID, "ccm_ba_time_kernel: unknown kernel id");
      }
      if (which == 1 || which == 2 || which == 4) CCM_LAUNCHED();
      CCM_CUDA(cudaEventRecord(e1, s));
      CCM_CUDA(cudaEventSynchronize(e1));
      float ms = 0.f;
      CCM_CUDA(cudaEventElapsedTime(&ms, e0, e1));
      total += ms;
    }
    cudaEventDestroy(e0); cudaEventDestroy(e1);
    *ms_per_launch = total / reps;
  });
}

// Converter::toSE3Quat: f32 4x4 -> (q, t) in f64 through SE3Quat(R, t)  (S/Converter.cc:40-51, G/types/se3quat.h:58-60)
extern "C" void ccm_pose_from_Tcw_f32(const float* T, int32_t n, double* qt) {
  for (int i = 0; i < n; i++) {
    const float* t = T + 16 * (size_t)i;
    const double R[9] = {t[0], t[1], t[2], t[4], t[5], t[6], t[8], t[9], t[10]};
    double x, y, z, w;
    R_to_quat(R, x, y, z, w);
    quat_normalize_pos_w(x, y, z, w);
    double* o = qt + 7 * (size_t)i;
    o[0] = x; o[1] = y; o[2] = z; o[3] = w; o[4] = t[3]; o[5] = t[7]; o[6] = t[11];
  }
}

// Converter::toCvMat(SE3Quat): homogeneous matrix rounded to f32  (S/Converter.cc:53-72)
extern "C" void ccm_pose_to_Tcw_f32(const double* qt, int32_t n, float* T) {
  for (int i = 0; i < n; i++) {
    const double* q = qt + 7 * (size_t)i;
    double R[9];
    quat_to_R(q[0], q[1], q[2], q[3], R);
    float* o = T + 16 * (size_t)i;
    for (int r = 0; r < 3; r++) {
      for (int c = 0; c < 3; c++) o[r * 4 + c] = (float)R[r * 3 + c];
      o[r * 4 + 3] = (float)q[4 + r];
    }
    o[12] = o[13] = o[14] = 0.f; o[15] = 1.f;
  }
}

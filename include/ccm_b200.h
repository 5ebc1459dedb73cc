/*
 * ccm_b200.h — C ABI of libccm_b200.so: the H100-native (sm_90a) replacement for the
 * bundle-adjustment + ORB hot path of VIS4ROB-lab/ccm_slam.
 *
 * The reference has no FFI for this path: the boundary is plain C++ linkage of
 *   cslam::Optimizer  (cslam/include/cslam/Optimizer.h:84-112)  -> vendored g2o
 *   cslam::ORBextractor (cslam/include/cslam/ORBextractor.h:103-138)
 *   cslam::ORBmatcher   (cslam/include/cslam/ORBmatcher.h:97-145)
 * A drop-in keeps those headers byte-identical and replaces the three .cpp files by shim TUs (shim/)
 * that flatten the pointer graph into the structs below, call these entry points, and write back.
 * INTEGRATION.md shows the binding.  Every entry point cites the reference code it replaces.
 *
 * Conventions: plain pointers + sizes, host buffers, no torch / CUDA types.  All functions return
 * CCM_OK (0) or a negative error code; ccm_last_error() gives the message (thread-local).  The library
 * never falls back to a CPU path: without a CUDA device every compute entry point returns
 * CCM_ERR_NO_DEVICE.  Thread-safe per handle; each handle owns its CUDA stream.
 */
#ifndef CCM_B200_H
#define CCM_B200_H
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define CCM_OK 0
#define CCM_ERR_INVALID (-1)
#define CCM_ERR_NO_DEVICE (-2)
#define CCM_ERR_CUDA (-3)
#define CCM_ERR_NCCL (-4)
#define CCM_ERR_OOM (-5)

int ccm_version(void);
const char* ccm_last_error(void);
/* number of CUDA devices visible (0 when none / driver missing); never fails */
int ccm_device_count(void);
/* bind the calling thread's subsequent handles to `device` */
int ccm_init(int device);
int ccm_shutdown(void);
/* cumulative number of kernels this library launched in this process (bench.py's gpu_launches) */
uint64_t ccm_kernel_launches(void);

/* write a buffer larger than L2 (256 MiB) and synchronise: benchmarks call it between timed iterations */
int ccm_l2_flush(void);
/* page-lock / unlock caller memory so that the uploads inside ccm_*_create/solve run from pinned memory */
int ccm_host_register(void* ptr, uint64_t bytes);
int ccm_host_unregister(void* ptr);

/* ---- multi-GPU: one process per GPU, landmarks sharded across ranks (SURVEY.md §8(e)) --------------------
 * Rank 0 calls ccm_comm_unique_id and ships the 128 bytes to the other ranks (e.g. torch.distributed
 * broadcast); every rank then calls ccm_comm_init.  NCCL is dlopen'ed lazily (libnccl.so.2). */
int ccm_comm_unique_id(uint8_t id[128]);
int ccm_comm_init(int rank, int nranks, const uint8_t id[128]);
int ccm_comm_destroy(void);
int ccm_comm_rank(void);
int ccm_comm_size(void);

/* ---- bundle adjustment ---------------------------------------------------------------------------------
 * Replaces g2o::SparseOptimizer::{initializeOptimization, optimize} as driven by
 *   Optimizer::MapFusionGBA                (cslam/src/Optimizer.cpp:646-859, optimize at :797)
 *   Optimizer::LocalBundleAdjustmentClient (cslam/src/Optimizer.cpp:349-644, optimize at :537 and :567)
 *   Optimizer::BundleAdjustmentClient      (cslam/src/Optimizer.cpp:40-212,  optimize at :166)
 * i.e. BlockSolver_6_3 + OptimizationAlgorithmLevenberg + EdgeSE3ProjectXYZ + RobustKernelHuber
 * (cslam/thirdparty/g2o/g2o/core/optimization_algorithm_levenberg.cpp:61-164, core/block_solver.hpp:354-604,
 *  types/types_six_dof_expmap.{h:80-109,cpp:103-147}).  The direct LDL^T on the reduced camera system
 * (solvers/linear_solver_eigen.h:106-133) is replaced by block-Jacobi PCG run to `pcg_tol`.               */
typedef struct ccm_ba_problem {
  int32_t K, P, E;
  const double* poses;       /* K*7 : qx qy qz qw tx ty tz of Tcw  (g2o::SE3Quat; Converter::toSE3Quat, Converter.cc:40-51) */
  const double* intr;        /* K*4 : fx fy cx cy (KeyFrame::fx.. widened, Optimizer.cpp:777-780) */
  const uint8_t* fixed;      /* K   : vSE3->setFixed(...)  (Optimizer.cpp:705, :435, :455) */
  const double* points;      /* P*3 : Converter::toVector3d(pMP->GetWorldPos()) */
  const int32_t* obs_kf;     /* E   : pose index of the observing keyframe */
  const int32_t* obs_mp;     /* E   : point index */
  const float* obs_uv;       /* E*2 : kpUn.pt.{x,y}  (Optimizer.cpp:758-762) */
  const float* obs_w;        /* E   : pKF->mvInvLevelSigma2[kpUn.octave]  (Optimizer.cpp:768-769) */
  const uint8_t* edge_flags; /* E or NULL : bit0 = e->setLevel(1) (inactive), bit1 = e->setRobustKernel(0)  (Optimizer.cpp:556-561) */
} ccm_ba_problem;

typedef struct ccm_ba_options {
  int32_t iterations;        /* optimizer.optimize(n) */
  int32_t robust;            /* bRobust: Huber kernel on every edge that does not carry bit1 */
  double huber_delta;        /* (double)(float)sqrt(5.99) for GBA, sqrt(5.991) for LocalBA */
  double lambda_init;        /* <= 0 : g2o default tau*max|H_jj|, tau = 1e-5 */
  int32_t max_trials;        /* <= 0 : 10 (maxTrialsAfterFailure) */
  int32_t pcg_max_iter;      /* <= 0 : 2000 */
  double pcg_tol;            /* <= 0 : 1e-8 ; stop when |r|_2 <= pcg_tol*|b|_2 */
  const volatile uint8_t* stop; /* optimizer.setForceStopFlag(pbStopFlag): polled between LM iterations and trials; may be NULL */
} ccm_ba_options;

#define CCM_TRACE_COLS 8 /* iter, lambda_used, chi2_after, rho, trials, lambda_after, pcg_iters(last trial), pcg_relres */

typedef struct ccm_ba_result {
  double* poses;             /* K*7 out (may be NULL) */
  double* points;            /* P*3 out (may be NULL) */
  double* chi2;              /* E out or NULL: e'We per ACTIVE edge at the last evaluated state; inactive entries untouched
                                (reference keeps the round-1 value there, Optimizer.cpp:582) */
  uint8_t* depth_pos;        /* E out or NULL: EdgeSE3ProjectXYZ::isDepthPositive on the final estimate, all edges */
  double* trace;             /* trace_cap*CCM_TRACE_COLS or NULL */
  int32_t trace_cap;
  int32_t trace_len;
  int32_t iters_done;        /* return value of SparseOptimizer::optimize (-1: nothing to optimise) */
  int32_t trials_total;
  int32_t pcg_iters_total;
  int32_t pcg_not_converged; /* number of trials whose PCG hit pcg_max_iter */
  double chi2_initial, chi2_final, lambda_final;
  double t_setup_ms;         /* upload + structure (buildStructure equivalent) */
  double t_optimize_ms;      /* LM loop (device time + host control) */
  double t_download_ms;
  double t_optimize_event_ms; /* the LM loop bracketed by CUDA events on the handle's stream */
} ccm_ba_result;

typedef struct ccm_ba_handle ccm_ba_handle;

/* one-shot: upload, build structure, optimise, download (the call the shim makes). */
int ccm_ba_solve(const ccm_ba_problem* p, const ccm_ba_options* o, ccm_ba_result* r);

/* handle API (device-resident state between calls; used by LocalBA's two rounds and by bench.py) */
int ccm_ba_create(const ccm_ba_problem* p, ccm_ba_handle** out);
/* restore the estimate uploaded at create time (edge flags unchanged) */
int ccm_ba_reset(ccm_ba_handle* h);
/* replace the estimate (K*7 poses, P*3 points; either may be NULL = keep): the structure, the observations and everything built from
 * them stay on the device.  A server whose map changed in value only since the last global BA (the persistent mirror says so) keeps
 * its handle and uploads K*56 + P*24 bytes instead of the whole problem (cfg5: 24.6 MB instead of 425 MB, no structure build). */
int ccm_ba_set_estimate(ccm_ba_handle* h, const double* poses, const double* points);
/* replace edge flags (E bytes, same order as at create) — LocalBA round 2 */
int ccm_ba_set_edge_flags(ccm_ba_handle* h, const uint8_t* edge_flags);
int ccm_ba_optimize(ccm_ba_handle* h, const ccm_ba_options* o, ccm_ba_result* r);
void ccm_ba_destroy(ccm_ba_handle* h);

/* host-only: the landmark range [L0, L1) and observation range [E0, E1) rank `rank` of `nranks` owns (the same cut
 * ccm_ba_create applies to its communicator rank); observations need not be sorted */
int ccm_ba_shard_range(const int32_t* obs_mp, int32_t E, int32_t P, int32_t rank, int32_t nranks, int32_t* L0, int32_t* L1,
                       int64_t* E0, int64_t* E1);

/* developer hook: SM-clock cycles CTA 0 of the PCG kernel spent per phase (needs CCM_PCG_PROF=1 at create time) */
int ccm_ba_debug_pcg_cycles(ccm_ba_handle* h, int64_t* cycles8);

/* problem-shape facts of a handle (for roofline accounting) */
typedef struct ccm_ba_info {
  int32_t K, K_free, P_local, E_local, rank, nranks;
  int64_t s_blocks_upper, s_blocks_full, schur_products;
  int64_t device_bytes;
} ccm_ba_info;
int ccm_ba_get_info(const ccm_ba_handle* h, ccm_ba_info* info);

/* per-kernel CUDA-event accounting over everything ccm_ba_optimize launches while profiling is on (events are
 * recorded on the handle's stream around each kernel / kernel group; two records per span). */
#define CCM_BA_K_LINEARIZE 0   /* k_linearize: residual + Jacobian + Hll/bl + Z = W U^-1         (per LM iteration; Z-only
                                  launches in the first iteration and after a rejected trial) */
#define CCM_BA_K_POSE_PASS 1   /* k_pose_pass: Hpp/bp                                            (per LM iteration) */
#define CCM_BA_K_SCALE 2       /* no kernel: Z is formed by k_linearize (slot kept, records no launches) */
#define CCM_BA_K_SCHUR 3       /* k_schur_mma: Schur products                                    (per LM trial) */
#define CCM_BA_K_ALLREDUCE 4   /* NCCL all-reduce of [S upper | bschur part]                     (per LM trial, N>1) */
#define CCM_BA_K_FINALIZE 5    /* k_finalize_S + k_block_jacobi                                  (per LM trial) */
#define CCM_BA_K_PCG 6         /* k_pcg (persistent)                                             (per LM trial) */
#define CCM_BA_K_BACKSUB 7     /* k_update_poses + k_backsub_points (+ their partial sums)       (per LM trial) */
#define CCM_BA_K_RESIDUAL 8    /* k_residual on the trial state (+ partial sum)                  (per LM trial) */
#define CCM_BA_NKERNELS 9
int ccm_ba_set_profile(ccm_ba_handle* h, int on);   /* also zeroes the counters */
int ccm_ba_get_kernel_stats(const ccm_ba_handle* h, double* total_ms /*CCM_BA_NKERNELS*/, int64_t* launches /*CCM_BA_NKERNELS*/);

/* kernel-level entry points for parity tests and ncu: run ONE pass on the handle's current estimate.
 * Outputs are host buffers in the caller's index space (same layout as the oracle's orc_ba_build). */
int ccm_ba_debug_build(ccm_ba_handle* h, int robust, double huber_delta,
                       double* Hpp /*K*36*/, double* bp /*K*6*/, double* Hll /*P*9*/, double* bl /*P*3*/,
                       double* W /*E*18*/, double* chi2_robust_sum);
int ccm_ba_debug_schur(ccm_ba_handle* h, int robust, double huber_delta, double lambda,
                       double* S_dense /*(6K)^2 or NULL*/, double* bschur /*6K or NULL*/,
                       double* dx_pose /*K*6*/, double* dx_point /*P*3*/, int32_t* pcg_iters, double* pcg_relres);
/* one LM trial from a caller-given pose step, without the Schur and PCG passes: linearise at the current estimate with damping
 * lambda, then the pose update exp(x) * T, the landmark back-substitution from x, and the robust chi2 of the trial state.
 * dx_pose (K*6, caller's pose indices; rows of fixed poses are ignored) is x.  Outputs: the trial state, the landmark step, the trial
 * chi2 and the two halves of the gain-ratio denominator, sum x (lambda x + bp) and sum xl (lambda xl + bl).  Any output may be NULL. */
int ccm_ba_debug_step(ccm_ba_handle* h, int robust, double huber_delta, double lambda, const double* dx_pose /*K*6*/,
                      double* pose_trial /*K*7*/, double* pt_trial /*P*3*/, double* dx_point /*P*3*/, double* chi2_trial,
                      double* scale_pose, double* scale_point);
/* S (lambda included) and b_schur as the last ccm_ba_debug_schur left them, as block CSR in the caller's pose indices: every stored
 * 6x6 block of the full symmetric pattern, row-major, columns ascending; fixed poses have empty rows and zero b_schur.
 * nnzb = ccm_ba_info.s_blocks_full.  Any output may be NULL. */
int ccm_ba_debug_schur_blocks(ccm_ba_handle* h, int32_t* rowptr /*K+1*/, int32_t* col /*nnzb*/, double* val /*nnzb*36*/,
                              double* bschur /*6K*/);
/* the Schur product lists of the handle: upper block u = (blk[2u], blk[2u+1]) in the caller's pose indices (row <= column, row-major,
 * columns ascending), its products pairs[2p], pairs[2p+1] for p in [ptr[u], ptr[u+1]): observation pairs (e, o) with e seen by the
 * row's pose and o by the column's, as positions in the landmark-sorted observation order (the caller's order when obs_mp is
 * sorted; a stable sort by obs_mp otherwise).  nub = ccm_ba_info.s_blocks_upper, nprod = ccm_ba_info.schur_products.  Any output
 * may be NULL. */
int ccm_ba_debug_products(ccm_ba_handle* h, int32_t* blk /*2*nub*/, uint32_t* ptr /*nub+1*/, int32_t* pairs /*2*nprod*/);
/* the Schur kernel's schedule: counts[0] tasks, counts[1] CTAs of its launch; task t covers sched[task_ptr[t] .. task_ptr[t+1]),
 * upper block numbers as in ccm_ba_debug_products.  Call with task_ptr and sched NULL to learn the number of tasks first.  Any
 * output may be NULL. */
int ccm_ba_debug_schedule(ccm_ba_handle* h, int32_t* counts /*2*/, int32_t* task_ptr /*ntasks+1*/, int32_t* sched /*nub*/);
/* the PCG path the handle runs: out[0] implementation (1 k_pcg, 2 k_pcg2), out[1] k_pcg CTA size, out[2] coarse aggregate size,
 * out[3] coarse nodes (0: no coarse space) */
int ccm_ba_debug_paths(ccm_ba_handle* h, int32_t* out /*4*/);
/* k_pcg2's streamed items (handles that run k_pcg2 only): counts[0] items, counts[1] CTAs, counts[2] blocks streamed per product;
 * items[20 * m] = first block, #blocks, row, flags (1 first of row, 2 last of row, 1 << (4 + k): block k also applied transposed),
 * 16 columns; cta_row / cta_item (CTAs + 1) the CTAs' first rows and items; slab_lo (16 per CTA) every warp's first slab row.  Call
 * with the arrays NULL to learn the counts first.  Any output may be NULL. */
int ccm_ba_debug_pcg2(ccm_ba_handle* h, int64_t* counts /*3*/, int32_t* items, int32_t* cta_row, int32_t* cta_item, int32_t* slab_lo);
/* the coarse level of the PCG preconditioner on the S the last ccm_ba_debug_schur left: the assembled Galerkin matrix P^T S P and
 * its inverse as the PCG set-up computes it (nC = 6 * coarse nodes, row-major nC x nC each).  Fails when the handle has no
 * coarse space or the set-up meets a non-positive pivot. */
int ccm_ba_debug_coarse(ccm_ba_handle* h, double* Ac /*nC*nC*/, double* Ainv /*nC*nC*/);
/* time `reps` launches of one kernel with CUDA events on the handle's stream; returns mean ms per launch.
 * which: 0 linearize (landmark pass, Hll/bl and Z), 1 pose pass, 2 residual/chi2, 3 Z-only linearize (g and Z at lambda),
 * 4 schur products, 5 back-substitution */
int ccm_ba_time_kernel(ccm_ba_handle* h, int which, int reps, double huber_delta, double lambda, double* ms_per_launch);

/* Converter::toSE3Quat / toCvMat restated (cslam/src/Converter.cc:40-72) — host-side helpers for the shim */
void ccm_pose_from_Tcw_f32(const float* T /*n*16 row-major*/, int32_t n, double* qt /*n*7*/);
void ccm_pose_to_Tcw_f32(const double* qt /*n*7*/, int32_t n, float* T /*n*16*/);

/* ---- Sim3 essential-graph optimisation -----------------------------------------------------------------
 * Replaces optimizer.optimize(20) in Optimizer::OptimizeEssentialGraph{LoopClosure,MapFusion}
 * (cslam/src/Optimizer.cpp:1277, :1513): VertexSim3Expmap / EdgeSim3 with identity information
 * (types/types_seven_dof_expmap.h:48-126), BlockSolver_7_3 without Schur, Levenberg, lambda0 = 1e-16. */
typedef struct ccm_pgo_problem {
  int32_t K, E;
  const double* sim3;        /* K*8 : qx qy qz qw tx ty tz s */
  const uint8_t* fixed;      /* K */
  const int32_t* edge_i;     /* E : vertex 0 */
  const int32_t* edge_j;     /* E : vertex 1 */
  const double* meas;        /* E*8 : Sji */
  int32_t fix_scale;         /* VSim3->_fix_scale */
} ccm_pgo_problem;

typedef struct ccm_pgo_options {
  int32_t iterations;        /* 20 */
  double lambda_init;        /* 1e-16 (solver->setUserLambdaInit) ; <=0: tau*max diag */
  int32_t pcg_max_iter;
  double pcg_tol;
  const volatile uint8_t* stop;
} ccm_pgo_options;

typedef struct ccm_pgo_result {
  double* sim3;              /* K*8 out */
  double* trace; int32_t trace_cap; int32_t trace_len;
  int32_t iters_done;
  double chi2_initial, chi2_final, lambda_final;
  double t_total_ms;
} ccm_pgo_result;

int ccm_pgo_solve(const ccm_pgo_problem* p, const ccm_pgo_options* o, ccm_pgo_result* r);

/* test-only entry points: the device code of ccm_pgo_solve on caller-chosen inputs (host buffers in and out).
 * ccm_sim3_debug_ops: one thread per row runs s3_exp(u), s3_log(a), s3_mul(a, b), s3_inv(a) and s3_oplus(a, u, fix_scale)
 * (Sim3 rows as in ccm_pgo_problem.sim3, updates u as 7-vectors omega, upsilon, sigma). */
int ccm_sim3_debug_ops(int32_t n, const double* u /*n*7*/, const double* a /*n*8*/, const double* b /*n*8*/, int32_t fix_scale,
                       double* exp_u /*n*8*/, double* log_a /*n*7*/, double* mul_ab /*n*8*/, double* inv_a /*n*8*/,
                       double* oplus_u_a /*n*8*/);
/* the per-edge linearisation of ccm_pgo_solve: error log(meas * si * sj^-1) and its central-difference Jacobians (row-major 7x7,
 * J[r*7+d] = de_r/du_d); free_ij[2e], free_ij[2e+1] == 0 marks the side as fixed (its Jacobian is zero) */
int ccm_pgo_debug_edges(int32_t n, const double* meas /*n*8*/, const double* si /*n*8*/, const double* sj /*n*8*/,
                        const int32_t* free_ij /*n*2*/, int32_t fix_scale, double* err /*n*7*/, double* Ji /*n*49*/, double* Jj /*n*49*/);
/* one linearisation at p->sim3 and one PCG solve of (H + lambda I) x = b, with the set-up, kernels and options of ccm_pgo_solve.
 * Always writes n_free (free vertices with an edge) and nnzb (stored 7x7 blocks of H); vidx (K: free index or -1), rowptr (n+1),
 * col (nnzb; full symmetric pattern, columns ascending, free-index space) and paths when given.  With H == NULL nothing runs on
 * the device.  Otherwise H (nnzb*49, without lambda), b (n*7), Minv (n*49: inverses of the damped diagonal blocks), x (n*7),
 * chi2 and pcg (4: iterations, relative residual, flag 0 converged / 1 max_iter / 2 breakdown, coarse size 7*nc or 0) are written.
 * paths (4): PCG CTA size, coarse aggregate size, coarse nodes, coarse inverse used (1/0). */
int ccm_pgo_debug_system(const ccm_pgo_problem* p, const ccm_pgo_options* o, double lambda, int32_t* n_free, int64_t* nnzb,
                         int32_t* vidx, int32_t* rowptr, int32_t* col, double* H, double* b, double* Minv, double* x, double* chi2,
                         double* pcg, int32_t* paths);

/* ---- single-vertex optimisations ------------------------------------------------------------------------
 * ccm_pose_optimize replaces the g2o part of Optimizer::PoseOptimizationClient (cslam/src/Optimizer.cpp:215-347): one SE3
 * vertex, n unary EdgeSE3ProjectXYZOnlyPose, Huber sqrt(5.991), 4 x {estimate := Tcw, optimize(10), chi2 > 5.991 -> outlier},
 * robust kernel dropped after the third round.  The shim fills the arrays from Frame (mvpMapPoints[i] != NULL only), then
 * writes `outlier` back into Frame.mvbOutlier, `Tcw` into Frame.SetPose and returns n_inliers
 * (= nInitialCorrespondences - nBad; 0 and Tcw unchanged when n < 3).
 * `batch` independent problems (frames of several agents) run in one launch, one CTA each. */
typedef struct ccm_pose_opt_problem {
  int32_t n;                 /* correspondences */
  const double* Tcw;         /* 7: qx qy qz qw tx ty tz = ccm_pose_from_Tcw_f32(Frame.mTcw) */
  const float* Xw;           /* n*3: MapPoint::GetWorldPos */
  const float* uv;           /* n*2: Frame.mvKeysUn[i].pt */
  const float* inv_sigma2;   /* n: Frame.mvInvLevelSigma2[octave] */
  float fx, fy, cx, cy;
} ccm_pose_opt_problem;
typedef struct ccm_pose_opt_result {
  double Tcw[7];
  int32_t n_inliers;
  uint8_t* outlier;          /* n, caller-allocated */
} ccm_pose_opt_result;
int ccm_pose_optimize(const ccm_pose_opt_problem* probs, int32_t batch, ccm_pose_opt_result* res);

/* ccm_sim3_optimize replaces the g2o part of Optimizer::OptimizeSim3 (cslam/src/Optimizer.cpp:861-1056): one Sim3 vertex
 * (g2oS12), per matched pair an EdgeSim3ProjectXYZ (x1 = K1 * S12 * X2c) and an EdgeInverseSim3ProjectXYZ
 * (x2 = K2 * S12^-1 * X1c) against fixed points, numeric Jacobians, Huber sqrt(th2), optimize(5), pairs with chi2 > th2 removed,
 * optimize(5 or 10).  The shim keeps the reference's pair filter (:917-931) and camera-frame points (:925,:932, f32), clears
 * vpMatches1 where `inlier` is 0, and returns n_inliers (0 with S12 unchanged when fewer than 10 pairs survive the first pass).
 * `batch`: the loop / merge candidates of one place-recognition query. */
typedef struct ccm_sim3_opt_problem {
  int32_t n;                 /* pairs */
  const double* S12;         /* 8: qx qy qz qw tx ty tz s */
  const float* P1c;          /* n*3: R1w*P1w + t1w */
  const float* P2c;          /* n*3: R2w*P2w + t2w */
  const float* uv1;          /* n*2: pKF1->mvKeysUn[i].pt */
  const float* uv2;          /* n*2: pKF2->mvKeysUn[i2].pt */
  const float* inv_sigma2_1; /* n */
  const float* inv_sigma2_2; /* n */
  float K1[4], K2[4];        /* fx fy cx cy */
  float th2;
  int32_t fix_scale;
} ccm_sim3_opt_problem;
typedef struct ccm_sim3_opt_result {
  double S12[8];
  int32_t n_inliers;
  uint8_t* inlier;           /* n, caller-allocated */
} ccm_sim3_opt_result;
int ccm_sim3_optimize(const ccm_sim3_opt_problem* probs, int32_t batch, ccm_sim3_opt_result* res);

/* test-only entry points: the device code of ccm_pose_optimize / ccm_sim3_optimize on caller-chosen inputs.
 * ccm_{pose,sim3}_optimize_traced: the same protocol as the product entry points (same results), recording g2o's Levenberg
 * protocol in `trace`: per problem CCM_SINGLE_TRACE_{POSE,SIM3}_CALLS optimize() calls of CCM_SINGLE_TRACE_HEAD +
 * CCM_SINGLE_TRACE_ITERS * CCM_SINGLE_TRACE_COLS doubles each.  Header: end (0 iteration limit, 1 ten rejected trials,
 * 2 rho == 0, 3 three iterations without gain, -1 no active edge), iterations, iteration limit of the call, chi2 of the cached
 * edge errors the classification after the call reads, chi2 of fresh errors at the estimate over the same edges, number of those
 * edges whose cached error is not bit-identical to the fresh one, edges (pose) / pairs (Sim3) the classification rejects.  Row per LM iteration: iniChi, lambda at its
 * start, trials, rho of the last trial, currentChi at its end, accepted (1/0), failed Cholesky factorisations.  NaN where a call
 * or an iteration did not happen. */
#define CCM_SINGLE_TRACE_ITERS 10
#define CCM_SINGLE_TRACE_COLS 7
#define CCM_SINGLE_TRACE_HEAD 7
#define CCM_SINGLE_TRACE_POSE_CALLS 4
#define CCM_SINGLE_TRACE_SIM3_CALLS 2
int ccm_pose_optimize_traced(const ccm_pose_opt_problem* probs, int32_t batch, ccm_pose_opt_result* res, double* trace);
int ccm_sim3_optimize_traced(const ccm_sim3_opt_problem* probs, int32_t batch, ccm_sim3_opt_result* res, double* trace);
/* ccm_{pose,sim3}_debug_system: per problem, at the state probs[b].Tcw / .S12, with the edge masks active / robust (edges of all
 * problems back to back: n per pose problem, 2n per Sim3 problem, edge 2i the forward and 2i+1 the inverse edge of pair i) and
 * delta_lambda[2b] = Huber delta, [2b+1] = lambda: one system build and one damped solve with the optimiser's device functions.
 * err (2 per edge) and J (2 x D row-major per edge, D = 6 / 7) for every edge; sys per problem = H (D*D, without lambda), b (D),
 * robust chi2 of the active edges, x (D) of (H + lambda I) x = b; solved[b] = 1, or 0 with x = 0 when a pivot is not positive.
 * th2 of a Sim3 problem is not read. */
int ccm_pose_debug_system(const ccm_pose_opt_problem* probs, int32_t batch, const uint8_t* active, const uint8_t* robust,
                          const double* delta_lambda, double* err, double* J, double* sys, int32_t* solved);
int ccm_sim3_debug_system(const ccm_sim3_opt_problem* probs, int32_t batch, const uint8_t* active, const uint8_t* robust,
                          const double* delta_lambda, double* err, double* J, double* sys, int32_t* solved);

/* ---- ORB front end ------------------------------------------------------------------------------------
 * ccm_orb_* replace ORBextractor::operator() (cslam/src/ORBextractor.cpp:1216-1278) and its helpers
 * (ComputePyramid :1280-1304, ComputeKeyPointsOctTree :933-1024, IC_Angle :68-95, computeOrbDescriptor :100-316);
 * OpenCV primitives follow the 4.x integer semantics pinned in SURVEY.md §8(c'). */
typedef struct ccm_orb_config {
  int32_t nfeatures;         /* 1000 */
  float scale_factor;        /* 1.2 */
  int32_t nlevels;           /* 8 */
  int32_t ini_th_fast;       /* 20 */
  int32_t min_th_fast;       /* 7 */
  int32_t blur_2413;         /* 0: OpenCV 4.x GaussianBlur taps [18,34,48,56,48,34,18]; 1: 2.4.13 taps [18,34,49,55,49,34,18] */
} ccm_orb_config;

typedef struct ccm_keypoint {  /* cv::KeyPoint fields the reference reads */
  float x, y, size, angle, response;
  int32_t octave;
} ccm_keypoint;

typedef struct ccm_orb_handle ccm_orb_handle;
int ccm_orb_create(const ccm_orb_config* cfg, int32_t width, int32_t height, ccm_orb_handle** out);
/* the most keypoints one extract call on this handle can return: sum over the levels of max(4 * nIni, quota + 3), where nIni
 * is the number of root nodes of the level's quadtree; size kps (and desc, 32 bytes each) with it */
int ccm_orb_max_keypoints(const ccm_orb_handle* h, int32_t* n);
/* extract: kps capacity max_kp; returns count in *n; desc = n*32 bytes.  When the count exceeds max_kp the call fails with
 * CCM_ERR_INVALID, *n holds the count and kps / desc are not written. */
int ccm_orb_extract(ccm_orb_handle* h, const uint8_t* img, int32_t stride, ccm_keypoint* kps, int32_t max_kp,
                    int32_t* n, uint8_t* desc);
/* pyramid level readback (mvImagePyramid[level], public member of the reference class) */
int ccm_orb_get_level(ccm_orb_handle* h, int32_t level, uint8_t* out, int32_t* w, int32_t* hgt);
/* test hook: FAST candidates of the last extract call before the quadtree (3 floats each: x, y relative to the 16 px border, score);
 * *n = the full count, the first min(*n, max_out) are written */
int ccm_orb_debug_candidates(ccm_orb_handle* h, float* xys, int32_t* level, int32_t max_out, int32_t* n);
/* test hook: blurred pyramid level of the last extract call (GaussianBlur 7x7 that the descriptors sample), width x height bytes
 * as ccm_orb_get_level reports them */
int ccm_orb_debug_blurred(ccm_orb_handle* h, int32_t level, uint8_t* out);
void ccm_orb_destroy(ccm_orb_handle* h);

/* ---- Hamming matching ----------------------------------------------------------------------------------
 * ccm_hamming_matrix replaces the ORBmatcher::DescriptorDistance inner loops (cslam/src/ORBmatcher.cpp:1653-1669)
 * of SearchByBoW (:178-306, :565-698) and SearchForTriangulation (:700-852): D[i*nB+j] = popcount(A_i xor B_j).
 * The order-dependent greedy selection stays on the host (ccm_match_* below) and reads D. */
int ccm_hamming_matrix(const uint8_t* A, int32_t nA, const uint8_t* B, int32_t nB, uint16_t* D);

typedef struct ccm_feature_vector { /* DBoW2::FeatureVector flattened: nodes ascending, features per node */
  int32_t n_nodes;
  const uint32_t* node_id;   /* n_nodes */
  const int32_t* node_ptr;   /* n_nodes+1 into feat */
  const uint32_t* feat;      /* feature indices */
} ccm_feature_vector;

/* SearchByBoW(kfptr, Frame&, vpMapPointMatches)  (cslam/src/ORBmatcher.cpp:178-306)
 * kf_has_mp[i]: KF feature i has a good MapPoint; out match_f_of_kf[i] = frame feature matched to KF feature i or -1 -> the
 * shim turns it into vpMapPointMatches[frame idx] = KF's MapPoint.  Returns nmatches via *nmatches. */
int ccm_match_bow_kf_frame(const uint8_t* desc_kf, int32_t n_kf, const uint8_t* kf_has_mp, const float* angle_kf,
                           const ccm_feature_vector* fv_kf,
                           const uint8_t* desc_f, int32_t n_f, const float* angle_f, const ccm_feature_vector* fv_f,
                           float nnratio, int32_t check_orientation, int32_t* match_kf_of_f /*n_f, -1 = none*/,
                           int32_t* nmatches);
/* the host half alone: D = n_kf x n_f Hamming distances (ccm_hamming_matrix) -> the same selection (no device work) */
int ccm_select_bow_kf_frame(const uint16_t* D, int32_t n_kf, const uint8_t* kf_has_mp, const float* angle_kf,
                            const ccm_feature_vector* fv_kf, int32_t n_f, const float* angle_f, const ccm_feature_vector* fv_f,
                            float nnratio, int32_t check_orientation, int32_t* match_kf_of_f, int32_t* nmatches);
/* SearchByBoW(kfptr, kfptr, vpMatches12)  (cslam/src/ORBmatcher.cpp:565-698) */
int ccm_match_bow_kf_kf(const uint8_t* desc1, int32_t n1, const uint8_t* has_mp1, const float* angle1,
                        const ccm_feature_vector* fv1,
                        const uint8_t* desc2, int32_t n2, const uint8_t* has_mp2, const float* angle2,
                        const ccm_feature_vector* fv2,
                        float nnratio, int32_t check_orientation, int32_t* match12 /*n1, -1 = none*/, int32_t* nmatches);
int ccm_select_bow_kf_kf(const uint16_t* D /*n1 x n2*/, int32_t n1, const uint8_t* has_mp1, const float* angle1, const ccm_feature_vector* fv1,
                         int32_t n2, const uint8_t* has_mp2, const float* angle2, const ccm_feature_vector* fv2,
                         float nnratio, int32_t check_orientation, int32_t* match12, int32_t* nmatches);

typedef struct ccm_tri_view {  /* the per-keyframe read set of SearchForTriangulation */
  const uint8_t* desc; int32_t n;
  const uint8_t* has_mp;     /* n : pKF->GetMapPoint(idx) != NULL */
  const float* kp_xy;        /* n*2 : mvKeysUn[idx].pt */
  const int32_t* octave;     /* n */
  const float* angle;        /* n */
  const ccm_feature_vector* fv;
  float fx, fy, cx, cy;
} ccm_tri_view;
/* SearchForTriangulation(pKF1, pKF2, F12, vMatchedPairs)  (cslam/src/ORBmatcher.cpp:700-852)
 * epipole = C1 projected into view 2 (ex, ey) is computed by the shim from the poses (:704-712); F12 row-major 3x3 f32;
 * level_sigma2 : pKF2->mvLevelSigma2 (nlevels); scale_factors : pKF2->mvScaleFactors. */
int ccm_match_triangulation(const ccm_tri_view* v1, const ccm_tri_view* v2, const float F12[9], float ex, float ey,
                            const float* level_sigma2, const float* scale_factors, int32_t nlevels,
                            int32_t check_orientation, int32_t* pairs /*2*min(n1,n2)*/, int32_t* npairs);
int ccm_select_triangulation(const uint16_t* D /*v1->n x v2->n*/, const ccm_tri_view* v1, const ccm_tri_view* v2, const float F12[9], float ex,
                             float ey, const float* level_sigma2, const float* scale_factors, int32_t nlevels,
                             int32_t check_orientation, int32_t* pairs, int32_t* npairs);

/* ---- projection-guided matching (SURVEY.md §8(f) rank 3) -------------------------------------------------
 * The seven matchers that look a projected map point up in the image grid share one shape:
 *   [caller's prelude]  isBad / projection / IsInImage / distance + viewing-angle gates / PredictScale — f32 cv::Mat
 *                       arithmetic, O(#points), stays verbatim in the shim (shim/ORBmatcher_shim.cpp);
 *   [this library]      GetFeaturesInArea (cslam/src/Frame.cpp:200-253, KeyFrame.cpp:1162-1201) over the lookup grid of
 *                       AssignFeaturesToGrid (Frame.cpp:103-119, KeyFrame.cpp:206-226), the level filter, the descriptor
 *                       distances of every (query, feature) pair on the GPU (k_hamming), and the order-dependent
 *                       selection in the reference's visiting order (cell column, cell row, feature index);
 *   [caller's epilogue] map surgery on the returned indices (AddObservation / Replace / RemapMapPointMatch ...).
 * A query is one map point after the prelude.  ccm_search_* = device distances + selection; ccm_select_* = the selection
 * alone over a caller-supplied distance matrix D[m x n] (u16, row = query; e.g. from ccm_hamming_matrix when several
 * matchers share one matrix) — host code, runs without a device.                                                        */
typedef struct ccm_feature_grid {   /* the image side: a Frame or a KeyFrame */
  int32_t n;
  const uint8_t* desc;       /* n*32 : mDescriptors */
  const float* kp_xy;        /* n*2  : mvKeysUn[i].pt */
  const int32_t* octave;     /* n    : mvKeysUn[i].octave */
  const float* angle;        /* n    : mvKeysUn[i].angle (only read when check_orientation) */
  float min_x, min_y, max_x, max_y;   /* mnMinX, mnMinY, mnMaxX, mnMaxY */
  float grid_w_inv, grid_h_inv;       /* mfGridElementWidthInv, mfGridElementHeightInv (Frame.cpp:86-87) */
  int32_t grid_cols, grid_rows;       /* FRAME_GRID_COLS x FRAME_GRID_ROWS = 75 x 48 (Frame.h:51-52) / mnGridCols x mnGridRows */
} ccm_feature_grid;

typedef struct ccm_proj_queries {
  int32_t m;
  const uint8_t* valid;      /* m    : the prelude let this point through */
  const float* uv;           /* m*2  : projected pixel */
  const float* radius;       /* m    : r handed to GetFeaturesInArea */
  const int32_t* level;      /* m    : nPredictedLevel / mnTrackScaleLevel / nLastOctave */
  const uint8_t* desc;       /* m*32 : pMP->GetDescriptor() */
  const float* angle;        /* m    : keypoint angle on the query side (only read when check_orientation) */
} ccm_proj_queries;

/* GetFeaturesInArea alone (host; min_level/max_level as Frame's overload, -1/-1 = KeyFrame's): count in *n, at most cap indices */
int ccm_features_in_area(const ccm_feature_grid* g, float x, float y, float r, int32_t min_level, int32_t max_level,
                         int32_t* out, int32_t cap, int32_t* n);

/* SearchByProjection(Frame&, const vector<mpptr>&, th)  (cslam/src/ORBmatcher.cpp:71-148): levels [L-1, L], best and
 * second best, TH_HIGH, ratio test when both sit on one level.  query_has_obs[i] = pMP->Observations()>0 and feat_blocked[j] =
 * (F.mvpMapPoints[j] && Observations()>0) drive the skip of :107-109.  match_of_feat[j] = query last written to
 * F.mvpMapPoints[j], -1 = untouched. */
int ccm_search_by_projection_track(const ccm_feature_grid* g, const ccm_proj_queries* q, const uint8_t* query_has_obs,
                                   const uint8_t* feat_blocked, float nnratio, int32_t* match_of_feat /*n*/, int32_t* nmatches);
int ccm_select_by_projection_track(const ccm_feature_grid* g, const ccm_proj_queries* q, const uint16_t* D, const uint8_t* query_has_obs,
                                   const uint8_t* feat_blocked, float nnratio, int32_t* match_of_feat, int32_t* nmatches);

/* reloc = 0: SearchByProjection(Frame&, const Frame& LastFrame, th)  (ORBmatcher.cpp:1350-1476), threshold TH_HIGH, a feature
 *            is skipped when it holds a map point with observations;
 * reloc = 1: SearchByProjection(Frame&, kfptr, sAlreadyFound, th, ORBdist)  (ORBmatcher.cpp:1478-1605), threshold orb_dist,
 *            a feature is skipped when it holds any map point (feat_blocked) and every assignment shields.
 * Levels [L-1, L+1].  match_of_feat[j]: >= 0 query, -1 untouched, -2 assigned then cleared by the rotation histogram. */
int ccm_search_by_projection_frame(const ccm_feature_grid* g, const ccm_proj_queries* q, const uint8_t* query_has_obs,
                                   const uint8_t* feat_blocked, int32_t reloc, int32_t orb_dist, int32_t check_orientation,
                                   int32_t* match_of_feat /*n*/, int32_t* nmatches);
int ccm_select_by_projection_frame(const ccm_feature_grid* g, const ccm_proj_queries* q, const uint16_t* D, const uint8_t* query_has_obs,
                                   const uint8_t* feat_blocked, int32_t reloc, int32_t orb_dist, int32_t check_orientation,
                                   int32_t* match_of_feat, int32_t* nmatches);

/* SearchByProjection(kfptr, Scw, vpPoints, vpMatched, th)  (ORBmatcher.cpp:308-446): levels [L-1, L], TH_LOW.
 * feat_matched[j] = vpMatched[j] != nullptr on entry; existing_idx[i] = pMP->GetIndexInKeyFrame(pKF).  best_idx[i] = the
 * keypoint found for query i (-1 none): the shim calls RemapMapPointMatch for queries with existing_idx != -1 (:418-432) and
 * sets vpMatched[best_idx] otherwise (= match_of_feat, counted in *nmatches). */
int ccm_search_by_projection_sim3(const ccm_feature_grid* g, const ccm_proj_queries* q, const uint8_t* feat_matched,
                                  const int32_t* existing_idx, int32_t* best_idx /*m*/, int32_t* match_of_feat /*n*/, int32_t* nmatches);
int ccm_select_by_projection_sim3(const ccm_feature_grid* g, const ccm_proj_queries* q, const uint16_t* D, const uint8_t* feat_matched,
                                  const int32_t* existing_idx, int32_t* best_idx, int32_t* match_of_feat, int32_t* nmatches);

/* the search half of Fuse(kfptr, const vector<mpptr>&, th) (ORBmatcher.cpp:854-993; pass inv_level_sigma2 = pKF->mvInvLevelSigma2
 * for its chi-square gate :941-947) and of Fuse(kfptr, Scw, vpPoints, th, vpReplacePoint) (:995-1122; inv_level_sigma2 = NULL):
 * best_idx[i] = keypoint to fuse query i with (-1 none).  The epilogue (:955-990 / :1103-1118) runs in query order in the shim. */
int ccm_fuse_search(const ccm_feature_grid* g, const ccm_proj_queries* q, const float* inv_level_sigma2, int32_t nlevels,
                    int32_t* best_idx /*m*/, int32_t* nfound);
int ccm_fuse_select(const ccm_feature_grid* g, const ccm_proj_queries* q, const uint16_t* D, const float* inv_level_sigma2, int32_t nlevels,
                    int32_t* best_idx, int32_t* nfound);

/* SearchBySim3(pKF1, pKF2, vpMatches12, s12, R12, t12, th)  (ORBmatcher.cpp:1124-1348): q12 = one query per KF1 feature
 * projected into KF2 (searched in g2), q21 the converse; TH_HIGH each way, kept when both directions agree (:1327-1343).
 * match12[i1] = idx2 or -1. */
int ccm_search_by_sim3(const ccm_feature_grid* g1, const ccm_feature_grid* g2, const ccm_proj_queries* q12, const ccm_proj_queries* q21,
                       int32_t* match12 /*q12->m*/, int32_t* nfound);
int ccm_select_by_sim3(const ccm_feature_grid* g1, const ccm_feature_grid* g2, const ccm_proj_queries* q12, const ccm_proj_queries* q21,
                       const uint16_t* D12 /*q12->m x g2->n*/, const uint16_t* D21 /*q21->m x g1->n*/, int32_t* match12, int32_t* nfound);

/* SearchForInitialization(F1, F2, vbPrevMatched, vnMatches12, windowSize)  (ORBmatcher.cpp:448-563): one query per keypoint of F1
 * (level = its octave: only octave 0 is searched, uv = vbPrevMatched[i1], radius = windowSize), looked up in F2's grid; a keypoint of
 * F2 stays with the closest F1 keypoint (vMatchedDistance), ratio test, rotation histogram.  match12[i1] = i2 or -1; the shim
 * refreshes vbPrevMatched from it (:557-560). */
int ccm_search_for_initialization(const ccm_feature_grid* g2, const ccm_proj_queries* q, float nnratio, int32_t check_orientation,
                                  int32_t* match12 /*q->m*/, int32_t* nmatches);
int ccm_select_for_initialization(const ccm_feature_grid* g2, const ccm_proj_queries* q, const uint16_t* D, float nnratio,
                                  int32_t check_orientation, int32_t* match12, int32_t* nmatches);

/* ---- DBoW2 transform (SURVEY.md §8(f) rank 2) ------------------------------------------------------------
 * Replaces ORBVocabulary::transform(features, BowVector&, FeatureVector&, levelsup) as called by Frame::ComputeBoW
 * (cslam/src/Frame.cpp:268-275) and KeyFrame::ComputeBoW (KeyFrame.cpp:277-286): the tree descent of every descriptor
 * (thirdparty/DBoW2/DBoW2/TemplatedVocabulary.h:1219-1260, FORB::distance FORB.cpp:77-100) runs on the GPU over a
 * device-resident vocabulary; the two std::map containers (TemplatedVocabulary.h:1127-1192, BowVector.cpp:34-88,
 * FeatureVector.cpp:28-43) are assembled on the host in feature order so the f64 sums round as the reference's.
 * The vocabulary arrives as the rows of its text file (loadFromTextFile, TemplatedVocabulary.h:1338-1422): row 0 = root,
 * row i = node id i: parent id, leaf flag, 32 descriptor bytes, weight; word ids are dealt in order of the leaf flags. */
typedef struct ccm_voc_handle ccm_voc_handle;
int ccm_voc_create(int32_t k, int32_t L, int32_t scoring /*DBoW2::ScoringType*/, int32_t weighting /*DBoW2::WeightingType*/,
                   int32_t n_nodes, const int32_t* parent, const uint8_t* is_leaf, const uint8_t* desc /*n_nodes*32*/,
                   const double* weight, ccm_voc_handle** out);
int ccm_voc_words(const ccm_voc_handle* h);
/* outputs sized n (fv_node_ptr n+1); any of word/node/weight_of_feat may be NULL */
int ccm_voc_transform(ccm_voc_handle* h, const uint8_t* desc, int32_t n, int32_t levelsup,
                      uint32_t* word_of_feat, uint32_t* node_of_feat, double* weight_of_feat,
                      uint32_t* bow_id, double* bow_val, int32_t* bow_n,
                      uint32_t* fv_node_id, int32_t* fv_node_ptr, uint32_t* fv_feat, int32_t* fv_n_nodes);
/* the container half alone (host): per-feature (word, weight, node) -> BowVector + FeatureVector */
int ccm_bow_assemble(int32_t scoring, int32_t weighting, int32_t n, const uint32_t* word_of_feat, const double* weight_of_feat,
                     const uint32_t* node_of_feat, uint32_t* bow_id, double* bow_val, int32_t* bow_n,
                     uint32_t* fv_node_id, int32_t* fv_node_ptr, uint32_t* fv_feat, int32_t* fv_n_nodes);
void ccm_voc_destroy(ccm_voc_handle* h);

/* ---- map update after a global BA (SURVEY.md §8(f) rank 1) ------------------------------------------------
 * Replaces the loop both Map::RunGBA (cslam/src/Map.cpp:1441-1570) and MapMerger::RunGBA (cslam/src/MapMerger.cpp:637-753) run
 * once MapFusionGBA has returned: the spanning-tree propagation of mTcwGBA to keyframes the BA did not hold, and the correction
 * of every map point (mPosGBA, or through its reference keyframe).  Flat view of the map:
 *   kf_parent[k]     index of the keyframe whose GetChilds() holds k; -1 = k is in mvpKeyFrameOrigins; -2 = not in the tree
 *   kf_optimized[k]  mBAGlobalForKF == nLoopKF (kf_TcwGBA[k] holds the BA's result); origins must be optimised
 *   kf_Tcw           GetPose() before the update (4x4 row-major f32) = what mTcwBefGBA receives
 *   kf_TcwGBA        in/out: filled for propagated keyframes; the caller SetPose()s it on every keyframe with kf_visited[k] = 1
 *   mp_state[i]      0 skip (isBad), 1 mBAGlobalForKF == nLoopKF (take mp_pos_gba), 2 follow reference keyframe mp_ref[i] (-1 none)
 *   mp_pos_out       the position to SetWorldPos() where mp_corrected[i] = 1 (elsewhere a copy of mp_pos)
 * Keyframe pass on the host (tree order), point pass on the GPU (one thread per point). */
int ccm_gba_map_update(int32_t n_kf, const int32_t* kf_parent, const uint8_t* kf_optimized, const float* kf_Tcw, float* kf_TcwGBA,
                       uint8_t* kf_visited, int32_t n_mp, const uint8_t* mp_state, const int32_t* mp_ref, const float* mp_pos,
                       const float* mp_pos_gba, float* mp_pos_out, uint8_t* mp_corrected);

/* ---- persistent flat mirror of the map for the global BA (SURVEY.md §8(f) rank 1) -----------------------------
 * Replaces the per-call flattening at the head of Optimizer::MapFusionGBA (cslam/src/Optimizer.cpp:658-787): the map tells the
 * mirror about changes where they happen (KeyFrame::SetPose, MapPoint::SetWorldPos, AddObservation / EraseObservation, SetBadFlag;
 * INTEGRATION.md) and ccm_mirror_ba_problem hands out a ccm_ba_problem over arrays the mirror owns, valid until the next ccm_mirror_*
 * call on it.  Value changes patch that problem in place; structural changes cost one pass over flat arrays at the next request,
 * applying the reference's selection rules (keyframes: not bad, uid <= max_kf_uid; edges: both ends selected; points: not bad, at
 * least min_edges observations in all and min_edges selected edges — 2, MapFusionGBA's rule (cslam/src/Optimizer.cpp:722-740), unless
 * ccm_mirror_set_min_edges(m, 1) asks for BundleAdjustmentClient's (:117-160)).  Rows keep first-insertion order; observations come
 * grouped by point row (insertion order inside a group), the layout ccm_ba_create takes without sorting.  uid = mUniqueId.  Host code;
 * one mirror is not thread-safe (the reference holds LockMapUpdate around a GBA). */
typedef struct ccm_map_mirror ccm_map_mirror;
int ccm_mirror_create(ccm_map_mirror** out);
void ccm_mirror_destroy(ccm_map_mirror* m);
int ccm_mirror_set_keyframe(ccm_map_mirror* m, uint64_t uid, const float* Tcw /*16*/, const float* intr4 /*fx fy cx cy; may be NULL on update*/, int32_t bad);
int ccm_mirror_erase_keyframe(ccm_map_mirror* m, uint64_t uid);
int ccm_mirror_set_point(ccm_map_mirror* m, uint64_t uid, const float* pos3, int32_t bad);
int ccm_mirror_erase_point(ccm_map_mirror* m, uint64_t uid);
int ccm_mirror_set_observation(ccm_map_mirror* m, uint64_t kf_uid, uint64_t mp_uid, float u, float v, float inv_sigma2);
int ccm_mirror_erase_observation(ccm_map_mirror* m, uint64_t kf_uid, uint64_t mp_uid);
int ccm_mirror_ba_problem(ccm_map_mirror* m, uint64_t max_kf_uid, const uint64_t* fixed_uid, int32_t n_fixed, ccm_ba_problem* out,
                          const uint64_t** kf_uid_of_row, const uint64_t** mp_uid_of_row);
long long ccm_mirror_rebuilds(const ccm_map_mirror* m);   /* how many flat passes have run (tests, tuning) */
int ccm_mirror_set_min_edges(ccm_map_mirror* m, int32_t min_edges);   /* 2 (default, MapFusionGBA) or 1 (BundleAdjustmentClient) */

/* ---- device-resident keyframe features (SURVEY.md §8(f) rank 4) ------------------------------------------------
 * The server receives every keyframe as a ccmslam_msgs::KF (cslam_msgs/msg/KF.msg) in Communicator::ProcessKfInServer
 * (cslam/src/Communicator.cpp:815-1140); KeyFrame::WriteMembersFromMessage (cslam/src/KeyFrame.cpp:1662-1726) copies mvKeysUn and
 * mDescriptors out of it, runs the vocabulary transform, and every later place-recognition / map-fusion matcher call reads the
 * descriptors from host memory again.  The store takes them ONCE, at ingest, straight from the message's storage — keypoints in the
 * ROS wire layout of ccmslam_msgs/CvKeyPoint (15 packed bytes: f32 x, f32 y, u8 size, f32 angle, u8 response, i8 octave; decoded
 * as Converter::fromCvKeyPointMsg does, cslam/src/Converter.cc:180-192), descriptors as the n contiguous 32-byte records of
 * ccmslam_msgs/Descriptor[] — keeps the descriptors in HBM, and the server-side matchers name their operands by mUniqueId.
 * Thread-safe; a keyframe is never moved once placed. */
typedef struct ccm_kf_store ccm_kf_store;
int ccm_kfstore_create(ccm_kf_store** out);
void ccm_kfstore_destroy(ccm_kf_store* s);
int ccm_kfstore_put_wire(ccm_kf_store* s, uint64_t uid, int32_t n, const uint8_t* keypoints_wire /*n*15*/, const uint8_t* descriptors /*n*32*/,
                         ccm_keypoint* kp_out /*n decoded keypoints for the caller's mvKeysUn, or NULL*/);
int ccm_kfstore_put(ccm_kf_store* s, uint64_t uid, int32_t n, const ccm_keypoint* kps, const uint8_t* descriptors);
int ccm_kfstore_erase(ccm_kf_store* s, uint64_t uid);
int32_t ccm_kfstore_features(ccm_kf_store* s, uint64_t uid);            /* N of the keyframe, -1 if unknown */
int64_t ccm_kfstore_keyframes(ccm_kf_store* s);
int64_t ccm_kfstore_h2d_bytes(ccm_kf_store* s);                         /* descriptor bytes uploaded so far (ingest only) */
int ccm_kfstore_get(ccm_kf_store* s, uint64_t uid, ccm_keypoint* kps /*or NULL*/, uint8_t* descriptors /*or NULL*/);
int ccm_kfstore_hamming(ccm_kf_store* s, uint64_t uid1, uint64_t uid2, uint16_t* D /*n1*n2*/);
int ccm_kfstore_hamming_query(ccm_kf_store* s, const uint8_t* Q, int32_t nQ, uint64_t uid, uint16_t* D /*nQ*n*/);
/* ORBmatcher::SearchByBoW(kfptr, kfptr, vpMatches12) (cslam/src/ORBmatcher.cpp:565-698) on two resident keyframes */
int ccm_kfstore_match_bow_kf_kf(ccm_kf_store* s, uint64_t uid1, const uint8_t* has_mp1, const ccm_feature_vector* fv1, uint64_t uid2,
                                const uint8_t* has_mp2, const ccm_feature_vector* fv2, float nnratio, int32_t check_orientation,
                                int32_t* match12 /*n1*/, int32_t* nmatches);
/* mpORBvocabulary->transform(vCurrentDesc, mBowVec, mFeatVec, 4) of WriteMembersFromMessage over the resident descriptors; outputs as ccm_voc_transform */
int ccm_kfstore_transform(ccm_kf_store* s, uint64_t uid, ccm_voc_handle* voc, int32_t levelsup, uint32_t* word_of_feat, uint32_t* node_of_feat,
                          double* weight_of_feat, uint32_t* bow_id, double* bow_val, int32_t* bow_n, uint32_t* fv_node_id,
                          int32_t* fv_node_ptr, uint32_t* fv_feat, int32_t* fv_n_nodes);
/* host only (usable without a device): n wire keypoints -> ccm_keypoint, the arithmetic of Converter::fromCvKeyPointMsg */
int ccm_wire_keypoints_decode(const uint8_t* keypoints_wire, int32_t n, ccm_keypoint* out);

/* ---- device-resident keyframe database (place recognition) --------------------------------------------------------
 * Replaces cslam::KeyFrameDatabase (cslam/src/Database.cpp): add :37-43, erase :45-64, clear :66-70 and the candidate
 * queries DetectLoopCandidates :72-202, DetectMapMatchCandidates :204-327, DetectRelocalizationCandidates :329-439 with the
 * DBoW2 scores they call (thirdparty/DBoW2/DBoW2/ScoringObject.cpp:23-311).  One database serves every agent and map of the
 * server (cslam/src/server/ServerSystem.cpp:185).  uid = mUniqueId, client = mId.second; a BowVector is (n, word[], value[]) in
 * std::map order.  The inverted file and the BowVectors live on the device; within a word the postings keep the reference's
 * list order (insertion order minus erased entries).
 * A query counts shared words per visible keyframe, keeps those with more than minCommonWords = (int)(max * 0.8f) and scores
 * them against the query: the output is the reference's scored list (lScoreAndMatch before the minScore filter) in the order
 * of lKFsSharingWords.  A keyframe is visible when its client's bit is set in client_mask and its uid is not in exclude_uid:
 *   DetectLoopCandidates      mask = the clients of the query's map; exclude = the query keyframe, GetConnectedKeyFrames(), and
 *                             every database keyframe of those clients that is not in GetMapptr()->GetMmpKeyFrames()
 *   DetectMapMatchCandidates  mask = every client not in pMap->msuAssClients; exclude = none
 *   DetectRelocalizationCandidates  mask = all ones; exclude = none
 * ccm_kfdb_select then runs the covisibility accumulation and the 0.75 * bestAccScore retain on the host.
 * Thread-safe per handle; every call returns after its device work has finished. */
typedef struct ccm_kfdb ccm_kfdb;
typedef struct ccm_kfdb_request {
  int32_t n;                 /* the query's BowVector */
  const uint32_t* word;      /* n, strictly ascending */
  const double* value;       /* n */
  uint64_t client_mask;      /* bit c: keyframes of client c are visible (client ids < 64) */
  int32_t n_exclude;
  const uint64_t* exclude_uid; /* n_exclude uids that are invisible (uids not in the database are ignored) */
} ccm_kfdb_request;
typedef struct ccm_kfdb_candidate {
  uint64_t uid;
  int32_t n_words;           /* shared words (mnLoopWords / mnRelocWords) */
  float score;               /* (float) of the score: what mLoopScore / mRelocScore receive */
  double score_f64;          /* mpVoc->score(query, keyframe) */
} ccm_kfdb_candidate;
typedef struct ccm_kfdb_result {
  ccm_kfdb_candidate* cand;  /* caller-allocated, cap entries (ccm_kfdb_size is always enough) */
  int32_t cap;
  int32_t n;                 /* scored candidates, in the reference's order */
  int32_t n_sharing;         /* visible keyframes sharing at least one word (lKFsSharingWords.size()) */
  int32_t max_common, min_common;
} ccm_kfdb_result;
int ccm_kfdb_create(int32_t n_words /*vocabulary size*/, int32_t scoring /*DBoW2::ScoringType*/, ccm_kfdb** out);
void ccm_kfdb_destroy(ccm_kfdb* h);
/* a keyframe already in the database is refused (erase it first); erasing an unknown uid is a no-op */
int ccm_kfdb_add(ccm_kfdb* h, uint64_t uid, uint32_t client, int32_t n, const uint32_t* word, const double* value);
int ccm_kfdb_erase(ccm_kfdb* h, uint64_t uid);
int ccm_kfdb_clear(ccm_kfdb* h);
int64_t ccm_kfdb_size(ccm_kfdb* h);       /* keyframes in the database, -1 for a null handle */
int ccm_kfdb_query(ccm_kfdb* h, const ccm_kfdb_request* q, ccm_kfdb_result* r);
/* nq queries against the same database state in one launch sequence; identical to nq calls of ccm_kfdb_query */
int ccm_kfdb_query_batch(ccm_kfdb* h, const ccm_kfdb_request* q, int32_t nq, ccm_kfdb_result* r);
/* score[i] = mpVoc->score(query, keyframe uid[i]) (the minScore loop over the covisible keyframes, LoopFinder.cpp:125-139) */
int ccm_kfdb_score_many(ccm_kfdb* h, int32_t n, const uint32_t* word, const double* value, int32_t n_uid, const uint64_t* uid,
                        double* score);
/* CUDA-event time of the counting kernels and of the threshold / order / score kernels, summed over queries while on */
int ccm_kfdb_set_timing(ccm_kfdb* h, int32_t on);   /* also zeroes the sums */
int ccm_kfdb_get_timing(ccm_kfdb* h, double* count_ms, double* score_ms, int64_t* queries);
/* host only (usable without a device): candidate r->cand[i]'s GetBestCovisibilityKeyFrames(10) is covis_uid[covis_ptr[i] ..
 * covis_ptr[i+1]), in its order.  reloc = 0: loop / map-match (minScore filter, bestAccScore starts at min_score); reloc = 1:
 * relocalisation (no filter, bestAccScore starts at 0).  out_uid (r->n entries) receives the returned vector<kfptr>.
 * Equivalence with the reference: the queries are stateless, Database.cpp reads marker members left by earlier queries.  They agree
 * whenever each (kind, query id) is queried once (LoopFinder, MapMatcher, Tracking) and, for relocalisation, whenever the mRelocScore
 * of every covisible keyframe that shares a word with the frame but is not scored in this query is 0: the reference adds that value
 * (Database.cpp:403-406 checks mRelocQuery only), left by an earlier relocalisation query or uninitialised; this selection adds
 * nothing for such a keyframe, and the ABI has no input that would reproduce the stale value (DESIGN.md §5). */
int ccm_kfdb_select(const ccm_kfdb_result* r, const int32_t* covis_ptr, const uint64_t* covis_uid, int32_t reloc, float min_score,
                    uint64_t* out_uid, int32_t* n_out);

/* ---- map-point normals and depth limits ------------------------------------------------------------------------------
 * MapPoint::UpdateNormalAndDepth (cslam/src/MapPoint.cpp:779-823) for a batch of points, bit for bit (f32 as OpenCV evaluates each
 * cv::Mat expression; see ccm_slam_b200/csrc/normal_depth_math.cuh).
 *   kf_centre [n_kf][3]   GetCameraCenter() of each keyframe row;  kf_bad [n_kf]: isBad() (a bad observer is skipped and not counted)
 *   mp_pos [n_mp][3]      mWorldPos
 *   obs_ptr [n_mp+1], obs_kf [obs_ptr[n_mp]]   the observers of point i, obs_kf[obs_ptr[i] .. obs_ptr[i+1]), in mObservations order
 *                         (the normal is an f32 sum over them: the order is kept as given)
 *   mp_ref [n_mp]         row of mpRefKF (used even when bad); -1: none
 *   mp_scale_ref          pRefKF->mvScaleFactors[octave of mvKeysUn[observations[pRefKF]]] (index 0 when pRefKF does not observe it:
 *                         the reference's operator[] inserts 0)
 *   mp_scale_last         pRefKF->mvScaleFactors[mnScaleLevels - 1]
 * Out: normal [n_mp][3] (mNormalVector), max_dist (mfMaxDistance), min_dist (mfMinDistance), status [n_mp]: 1 written, 0 untouched
 * (no observers, or mp_ref = -1; a bad point is passed with no observers).  Untouched points read 0 in every output.  Every observer
 * bad gives NaN in the normal, a point on an observer's centre too: both are the reference's values.
 * ccm_normal_depth runs on the GPU (host buffers in and out, its own stream); ccm_normal_depth_host is the same contract on the host,
 * usable without a device, for the single points tracking and mapping update one at a time. */
int ccm_normal_depth(int32_t n_kf, const float* kf_centre, const uint8_t* kf_bad, int32_t n_mp, const float* mp_pos, const int64_t* obs_ptr,
                     const int32_t* obs_kf, const int32_t* mp_ref, const float* mp_scale_ref, const float* mp_scale_last, float* normal,
                     float* max_dist, float* min_dist, uint8_t* status);
int ccm_normal_depth_host(int32_t n_kf, const float* kf_centre, const uint8_t* kf_bad, int32_t n_mp, const float* mp_pos, const int64_t* obs_ptr,
                          const int32_t* obs_kf, const int32_t* mp_ref, const float* mp_scale_ref, const float* mp_scale_last, float* normal,
                          float* max_dist, float* min_dist, uint8_t* status);

/* ---- map-point descriptors ------------------------------------------------------------------------------------------
 * MapPoint::ComputeDistinctiveDescriptors (cslam/src/MapPoint.cpp:929-994) for a batch of points, exactly (integer work): among the
 * observers that are not bad, the row whose median Hamming distance to all of them (itself included, the ((N-1)/2)-th smallest: the
 * lower middle for even N) is the first strictly smallest.  Any N; the reference's stack array limits it to about 1400.
 *   kf_bad [n_kf]         isBad() of each keyframe row (a bad observer is skipped: neither a candidate nor counted in N)
 *   obs_ptr [n_mp+1], obs_kf [obs_ptr[n_mp]]   the observers of point i, obs_kf[obs_ptr[i] .. obs_ptr[i+1]), in mObservations order
 *   obs_desc [E][32]      pKF->mDescriptors.row(idx) of each observation (read only for observers that are not bad)
 * Out: best [n_mp]        position of the chosen observer IN THE CALLER'S LIST obs_ptr[i] .. obs_ptr[i+1), bad observers counted, so
 *                         that it maps straight back to (pKF, idx); -1: untouched (no observers, or every observer bad; a bad point
 *                         is passed with no observers)
 *      best_median [n_mp] the chosen row's median (or NULL); desc_out [n_mp][32] its bytes (or NULL).  Untouched points read 0.
 * ccm_distinctive_descriptors runs on the GPU (host buffers in and out, its own stream); ccm_distinctive_descriptors_host is the same
 * contract on the host, usable without a device, for the single points that mapping and map merging update one at a time.
 * ccm_kfstore_distinctive_descriptors reads the rows from the keyframe store instead: kf_uid [n_kf] names each row's keyframe
 * (mUniqueId), obs_feat [E] the feature index (idx), so 8 bytes per observation cross the bus and ccm_kfstore_h2d_bytes does not
 * move.  An unknown uid or a feature index outside [0, N of the keyframe) of an observer that is not bad, or any keyframe row out of
 * range, fails the call with CCM_ERR_INVALID and a message naming the point; no output is written then. */
int ccm_distinctive_descriptors(int32_t n_kf, const uint8_t* kf_bad, int32_t n_mp, const int64_t* obs_ptr, const int32_t* obs_kf,
                                const uint8_t* obs_desc, int32_t* best, int32_t* best_median, uint8_t* desc_out);
int ccm_distinctive_descriptors_host(int32_t n_kf, const uint8_t* kf_bad, int32_t n_mp, const int64_t* obs_ptr, const int32_t* obs_kf,
                                     const uint8_t* obs_desc, int32_t* best, int32_t* best_median, uint8_t* desc_out);
int ccm_kfstore_distinctive_descriptors(ccm_kf_store* store, int32_t n_kf, const uint64_t* kf_uid, const uint8_t* kf_bad, int32_t n_mp,
                                        const int64_t* obs_ptr, const int32_t* obs_kf, const int32_t* obs_feat, int32_t* best,
                                        int32_t* best_median, uint8_t* desc_out);

/* ---- covisibility weights --------------------------------------------------------------------------------------------
 * The counting and the two orders of KeyFrame::UpdateConnections (cslam/src/KeyFrame.cpp:629-711) for a batch of keyframes, exactly
 * (integer work).  For batch keyframe b (row batch[b]): every entry of its mvpMapPoints that is not null and whose point is not bad
 * (a point at two indices counts twice) adds 1 to the weight of each of the point's observers whose kf_id differs from its own (the
 * idpair, not the row: another row with the same mId is skipped too; bad observers are counted).
 *   kf_id [n_kf]          mId of each keyframe row, packed (any injective packing of the idpair)
 *   kf_rank [n_kf]        each row's place in std::map<kfptr,int>'s order (the address rank); a permutation of 0 .. n_kf-1
 *   batch [n_b]           the keyframe row of each batch entry
 *   kf_mp_ptr [n_b+1], kf_mp [kf_mp_ptr[n_b]]   entry b's mvpMapPoints in index order as point rows, -1 = null
 *   mp_bad [n_mp]         isBad() of each point
 *   obs_ptr [n_mp+1], obs_kf [obs_ptr[n_mp]]    the observers of each point (its GetObservations() keys); observers may lie
 *                         outside the batch
 *   th                    the threshold (15 in the reference)
 * Out, for entry b at conn_ptr[b] .. conn_ptr[b+1) of arrays of `capacity` elements:
 *   conn_kf / conn_w      KFcounter (mConnectedKeyFrameWeights): (row, weight), ascending rank
 *   sel_kf / sel_w        the first n_sel[b] slots: the ordered connections (mvpOrderedConnectedKeyFrames / mvOrderedWeights as
 *                         UpdateConnections writes them): every entry with weight >= th by weight descending, ties by rank
 *                         descending; when none reaches th, the single entry (nmax, pKFmax), the LOWEST-rank entry among the tied
 *                         maxima.  The slots after n_sel[b] read -1 / 0.
 *   status [n_b]          0: the counter is empty (the reference returns with nothing changed), 1 otherwise
 *   total                 conn_ptr[n_b], always written.  When capacity is below it the call fails with CCM_ERR_INVALID and no
 *                         other output is written.
 * A row out of range (batch, point or observer) fails with CCM_ERR_INVALID and a message naming the batch keyframe; nothing is written.
 * ccm_covisibility runs on the GPU (host buffers in and out, its own stream); ccm_covisibility_host is the same contract on the host,
 * usable without a device, for the keyframes that ingest connects one at a time. */
int ccm_covisibility(int32_t n_kf, const uint64_t* kf_id, const uint32_t* kf_rank, int32_t n_b, const int32_t* batch, const int64_t* kf_mp_ptr,
                     const int32_t* kf_mp, int32_t n_mp, const uint8_t* mp_bad, const int64_t* obs_ptr, const int32_t* obs_kf, int32_t th,
                     int64_t capacity, int64_t* conn_ptr, int32_t* conn_kf, int32_t* conn_w, int32_t* n_sel, int32_t* sel_kf, int32_t* sel_w,
                     uint8_t* status, int64_t* total);
int ccm_covisibility_host(int32_t n_kf, const uint64_t* kf_id, const uint32_t* kf_rank, int32_t n_b, const int32_t* batch,
                          const int64_t* kf_mp_ptr, const int32_t* kf_mp, int32_t n_mp, const uint8_t* mp_bad, const int64_t* obs_ptr,
                          const int32_t* obs_kf, int32_t th, int64_t capacity, int64_t* conn_ptr, int32_t* conn_kf, int32_t* conn_w,
                          int32_t* n_sel, int32_t* sel_kf, int32_t* sel_w, uint8_t* status, int64_t* total);

/* ---- new map points ----------------------------------------------------------------------------------------------------
 * LocalMapping::CreateNewMapPoints (cslam/src/Mapping.cpp:284-469) for the current keyframe and all its neighbours in one call: for
 * each neighbour, SearchForTriangulation as the member constructs its matcher (ORBmatcher(0.6,false): no rotation histogram), then the
 * triangulation of every match and its gates (:362-448).  The neighbour list, the short-baseline skip (:320-328), ComputeF12 and the
 * epipole are f32 cv::Mat prelude and stay with the caller, as for ccm_match_triangulation; a skipped neighbour is not passed.
 *
 * The only coupling between neighbours in the reference is that a feature of the current keyframe triangulated with neighbour i
 * carries a map point when neighbour i+1 is searched.  So the lowest neighbour index whose pair is accepted claims the feature; a
 * rejected pair claims nothing.  Points leave in the reference's creation order: neighbour ascending, idx1 ascending within one.  Two
 * idx1 may choose the same idx2 of one neighbour; both points are reported.
 *
 * Arithmetic: ccm_slam_b200/csrc/new_points_math.cuh, one source for the device and the host entry point, which agree bit for bit.
 * cv::SVD::compute has no single bit pattern in the reference (its own Jacobi iteration or LAPACK's sgesdd, by OpenCV build); the
 * library states one: a one-sided Jacobi iteration in f32 (DESIGN.md §5).
 *
 * Every feature index may appear at most once in the current keyframe's FeatureVector (DBoW2 lists each feature under one node).
 * Out: *n_out points in out[]; when capacity is below the count the call fails with CCM_ERR_INVALID, *n_out holds the count needed
 * and nothing else is written.  best2 / verdict (each n_nb * cur->v.n, or NULL), for neighbour b and feature i at [b * n + i]:
 * the neighbour feature SearchForTriangulation pairs with i or -1, and what became of the pair.  A feature claimed by an earlier
 * neighbour reads -1 / CCM_NEWPTS_CLAIMED.  Invalid input fails with CCM_ERR_INVALID and a message naming the neighbour.
 * ccm_new_map_points: one upload, three launches whatever n_nb, one download.  ccm_new_map_points_host: the same contract, no device. */
typedef enum ccm_newpts_verdict {
  CCM_NEWPTS_NONE = 0,       /* no pair: the feature carries a map point, or no neighbour feature passes the matcher's gates */
  CCM_NEWPTS_ACCEPTED = 1,
  CCM_NEWPTS_PARALLAX = 2,   /* cosParallaxRays outside (0, 0.9998) */
  CCM_NEWPTS_W_ZERO = 3,     /* x3D(3) == 0 */
  CCM_NEWPTS_DEPTH1 = 4,     /* z1 <= 0 */
  CCM_NEWPTS_DEPTH2 = 5,     /* z2 <= 0 */
  CCM_NEWPTS_REPROJ1 = 6,    /* reprojection error in the current keyframe above 5.991 * sigma2 */
  CCM_NEWPTS_REPROJ2 = 7,    /* ... in the neighbour */
  CCM_NEWPTS_DIST_ZERO = 8,  /* dist1 == 0 || dist2 == 0 */
  CCM_NEWPTS_SCALE = 9,      /* scale consistency */
  CCM_NEWPTS_CLAIMED = 10    /* an earlier neighbour's accepted pair gave the feature its map point */
} ccm_newpts_verdict;

typedef struct ccm_newpts_view {      /* one keyframe as CreateNewMapPoints reads it */
  ccm_tri_view v;                     /* descriptors, has_mp, mvKeysUn xy / octave / angle (angle is not read), FeatureVector, fx fy cx cy */
  float Tcw[12];                      /* [Rcw | tcw], 3x4 row-major f32 */
  float Ow[3];                        /* GetCameraCenter() */
  const float* level_sigma2;          /* mvLevelSigma2, nlevels */
  const float* scale_factors;         /* mvScaleFactors, nlevels */
  int32_t nlevels;
  float scale_factor;                 /* mfScaleFactor (read of the current keyframe only) */
} ccm_newpts_view;
typedef struct ccm_newpts_neighbour {
  ccm_newpts_view view;
  float F12[9];                       /* ComputeF12(current, neighbour), row-major */
  float ex, ey;                       /* the current keyframe's centre projected into the neighbour (cslam/src/ORBmatcher.cpp:707-714) */
} ccm_newpts_neighbour;
typedef struct ccm_new_point { int32_t nb, idx1, idx2; float x3D[3]; } ccm_new_point;

int ccm_new_map_points(const ccm_newpts_view* cur, const ccm_newpts_neighbour* nb, int32_t n_nb, ccm_new_point* out, int32_t capacity,
                       int32_t* n_out, int32_t* best2, uint8_t* verdict);
int ccm_new_map_points_host(const ccm_newpts_view* cur, const ccm_newpts_neighbour* nb, int32_t n_nb, ccm_new_point* out, int32_t capacity,
                            int32_t* n_out, int32_t* best2, uint8_t* verdict);

/* ---- neighbour fusion ---------------------------------------------------------------------------------------------------
 * The searches of LocalMapping::SearchInNeighbors (cslam/src/Mapping.cpp:471-547) in one call.  The member runs
 * ORBmatcher::Fuse(pKFi, vpMapPointMatches) (cslam/src/ORBmatcher.cpp:854-993, th = 3) for every fuse target in list order (forward),
 * then Fuse(mpCurrentKeyFrame, vpFuseCandidates) once (backward).  The target list (first neighbours, their second neighbours, the
 * mFuseTargetForKF marks), the candidate list (mFuseCandidateForKF) and all map surgery stay with the caller.
 *
 * Why one pass is enough: every backward candidate is a target's point when the member starts, and the search part of Fuse reads
 * no map state that the surgery changes except isBad(), IsInKeyFrame() and, through MapPoint::Replace, the surviving point's
 * descriptor.  So every pair is searched here over the state at the start of the member; the caller walks the reference's order,
 * checks isBad() / IsInKeyFrame() live, and searches again on the host (ccm_fuse_select) only a pair whose point's descriptor no
 * longer equals the bytes passed in.
 *
 * Each (keyframe, point) pair runs Fuse's prelude (projection, IsInImage, the distance-invariance range, the 60-degree cone,
 * PredictScale; ccm_slam_b200/csrc/fuse_neighbours_math.cuh) and its window search: levels [L-1, L], the chi-square gate on
 * mvInvLevelSigma2, the first minimum of the Hamming distance, kept when <= TH_LOW.  PredictScale's log(float) is glibc's logf, which
 * the device does not reproduce; a pair whose level depends on the last bit of that logarithm is settled on the host with the host's
 * logf before the call returns (DESIGN.md §5).  *n_settled (may be NULL) counts those pairs.
 *
 * In:  cur              the current keyframe; targets[0..n_targets) the DISTINCT fuse targets (a target listed twice is passed once);
 *      pts              the point table; a point with skip set (mbDoNotReplace, or isBad() on entry) is never searched;
 *      cur_point[i]     the point row of the current keyframe's slot i (vpMapPointMatches[i]), -1 for an empty slot, cur->grid.n entries;
 *      cand[0..n_cand)  the point rows of vpFuseCandidates, in order.
 * Out: fwd_best[t * cur->grid.n + i]   keypoint of target t that slot i's point fuses with, or -1;
 *      bwd_best[c]                     keypoint of the current keyframe that candidate c fuses with, or -1.
 * A row out of range, a null array or a grid with more keypoints than the 20-bit visiting position of the window key holds fails
 * with CCM_ERR_INVALID and a message naming the target, slot or candidate; nothing is written.
 * ccm_fuse_neighbours: one upload, one launch whatever the number of targets, one download; no atomics, identical bytes every call.
 * ccm_fuse_neighbours_host: the same contract without a device; the two agree bit for bit. */
typedef struct ccm_fuse_kf {          /* one keyframe as Fuse reads it */
  ccm_feature_grid grid;              /* mvKeysUn, mDescriptors and the lookup grid; min_x .. max_y are also IsInImage's bounds */
  float Tcw[12];                      /* [Rcw | tcw], 3x4 row-major f32 */
  float Ow[3];                        /* GetCameraCenter() */
  float fx, fy, cx, cy;
  const float* scale_factors;         /* mvScaleFactors, nlevels */
  const float* inv_level_sigma2;      /* mvInvLevelSigma2, nlevels */
  int32_t nlevels;                    /* mnScaleLevels */
  float log_scale_factor;             /* mfLogScaleFactor */
} ccm_fuse_kf;
typedef struct ccm_fuse_points {      /* the map points the call may search, one row each */
  int32_t n;
  const float* pos;                   /* n*3 GetWorldPos() */
  const float* normal;                /* n*3 GetNormal() */
  const float* max_distance;          /* n   mfMaxDistance (the member's gate uses 1.2f times it, PredictScale the value itself) */
  const float* min_distance;          /* n   mfMinDistance */
  const uint8_t* desc;                /* n*32 GetDescriptor() */
  const uint8_t* skip;                /* n   ccm_fuse_neighbours: mbDoNotReplace || isBad();  ccm_search_and_fuse: isBad() only */
} ccm_fuse_points;

int ccm_fuse_neighbours(const ccm_fuse_kf* cur, const ccm_fuse_kf* targets, int32_t n_targets, const ccm_fuse_points* pts,
                        const int32_t* cur_point, const int32_t* cand, int32_t n_cand, int32_t* fwd_best, int32_t* bwd_best,
                        int32_t* n_settled);
int ccm_fuse_neighbours_host(const ccm_fuse_kf* cur, const ccm_fuse_kf* targets, int32_t n_targets, const ccm_fuse_points* pts,
                             const int32_t* cur_point, const int32_t* cand, int32_t n_cand, int32_t* fwd_best, int32_t* bwd_best,
                             int32_t* n_settled);

/* ---- loop and merge fusion -----------------------------------------------------------------------------------------------
 * The searches of LoopFinder::SearchAndFuse (cslam/src/LoopFinder.cpp:709-734) and MapMerger::SearchAndFuse
 * (cslam/src/MapMerger.cpp:574-598) in one call.  Both members run ORBmatcher::Fuse(pKF, Scw, vpLoopMapPoints, 4, vpReplacePoints)
 * (cslam/src/ORBmatcher.cpp:995-1122) for each corrected keyframe in map order, then Replace / ReplaceAndLock each point the search
 * found an occupant for.  The walk, the skip of points in pKF->GetMapPoints() and all map surgery stay with the caller.
 *
 * Why one pass is enough: a pair's search reads the point's position, normal, distance limits and descriptor, and the keyframe's
 * keypoints, grid and Scw.  Of these only the descriptor changes during the member (Replace and ReplaceAndLock end with
 * ComputeDistinctiveDescriptors on the survivor; nothing calls UpdateNormalAndDepth).  isBad() and GetMapPoints() change too, and
 * the caller checks them live.  So every pair is searched here over the state at the start of the member, and the caller searches
 * again (ccm_search_and_fuse_host, one keyframe) only points whose descriptor no longer equals the bytes passed in.
 *
 * Each (keyframe, point) pair runs Fuse(Scw)'s prelude (projection, IsInImage, the distance-invariance range, the 60-degree cone,
 * PredictScale; ccm_slam_b200/csrc/fuse_neighbours_math.cuh) with th = 4 and its window search: levels [L-1, L], no chi-square
 * gate, the first minimum of the Hamming distance, kept when <= TH_LOW.  mbDoNotReplace is not read (the reference comments it out).
 * A pair whose PredictScale level depends on the last bit of logf is settled on the host with logf before the call returns
 * (DESIGN.md §5); *n_settled (may be NULL) counts those pairs.
 *
 * In:  kfs[0..n_kf)   the corrected keyframes.  Tcw / Ow are the caller's split of the corrected Scw (Fuse's :1004-1008: scw = the
 *                     norm of row 0 of sR, Rcw = sR/scw, tcw = t/scw, Ow = -Rcw^T tcw), not the keyframe's pose.  inv_level_sigma2
 *                     is not read;
 *      pts            the loop points vpLoopMapPoints, one row each; skip = isBad() on entry.
 * Out: best[k * pts->n + i]   keypoint of keyframe k that loop point i lands on, or -1.
 * A null array, a grid with more keypoints than the 20-bit visiting position of the window key holds, or more than 2^30 pairs
 * (each keyframe's points padded to a multiple of 32) fails with CCM_ERR_INVALID and a message naming the keyframe; nothing is
 * written.  No pairs: no launch.
 * ccm_search_and_fuse: one upload, one launch whatever n_kf, one download; no atomics, identical bytes every call.
 * ccm_search_and_fuse_host: the same contract without a device; the two agree bit for bit. */
int ccm_search_and_fuse(const ccm_fuse_kf* kfs, int32_t n_kf, const ccm_fuse_points* pts, int32_t* best, int32_t* n_settled);
int ccm_search_and_fuse_host(const ccm_fuse_kf* kfs, int32_t n_kf, const ccm_fuse_points* pts, int32_t* best, int32_t* n_settled);

/* ---- Sim3 correction of a loop closure or a map merge ---------------------------------------------------------------------
 * The pass over CorrectedSim3 of LoopFinder::CorrectLoop (cslam/src/LoopFinder.cpp:568-613) and over CorrectedSim3All of
 * MapMerger::MergeMaps (cslam/src/MapMerger.cpp:349-395), bit for bit (f64 Sim3 arithmetic in Eigen's order, f32 where the reference
 * stores; see ccm_slam_b200/csrc/sim3_correction_math.cuh).  Entry e is the e-th element of the std::map in its iteration order.
 *   kf_centre [n_kf][3]   GetCameraCenter() of each keyframe row before the pass;  kf_bad [n_kf]: isBad()
 *   entry_kf [n_e]        the keyframe row of each entry (each row at most once)
 *   entry_Siw_new [n_e][8], entry_Siw_old [n_e][8]   the entry's corrected Sim3 and NonCorrectedSim3[pKFi], qx qy qz qw tx ty tz s
 *   slot_ptr [n_e+1], slot_mp [slot_ptr[n_e]]        entry e's GetMapPointMatches() in index order as point rows, -1 = null
 *   mp_pos [n_mp][3]      GetWorldPos();  mp_skip [n_mp]: isBad(), or mCorrectedByKF_LC / _MM already equal to the current mId
 *   obs_ptr, obs_kf, mp_ref, mp_scale_ref, mp_scale_last   the observers, mpRefKF and scale factors exactly as ccm_normal_depth takes them
 * Out, per entry: entry_Tcw [n_e][16] (row-major f32, the pose SetPose receives), entry_centre [n_e][3] (the Ow it leaves).
 * Out, per point: mp_entry [n_mp]: the entry that moves the point (the first in map order that lists it, when it is not skipped), -1
 * none; mp_pos_out [n_mp][3]: the corrected position (mp_pos for a point no entry moves); normal, max_dist, min_dist, status: what
 * UpdateNormalAndDepth leaves right after the move, with ccm_normal_depth's semantics (0 everywhere and status 0 for a point no entry
 * moves).  The normal reads the corrected centre of each keyframe that is an entry BEFORE mp_entry and the pre-loop centre of every
 * other keyframe, mp_entry's own included: the reference's SetPose for an entry follows its points.
 * A row out of range, a keyframe listed as two entries or a null array fails with CCM_ERR_INVALID and a message naming the entry, slot
 * or point; nothing is written then.
 * ccm_sim3_correction runs on the GPU (host buffers in and out, its own stream, three launches); ccm_sim3_correction_host is the same
 * contract on the host, usable without a device. */
int ccm_sim3_correction(int32_t n_kf, const float* kf_centre, const uint8_t* kf_bad, int32_t n_e, const int32_t* entry_kf,
                        const double* entry_Siw_new, const double* entry_Siw_old, const int64_t* slot_ptr, const int32_t* slot_mp, int32_t n_mp,
                        const float* mp_pos, const uint8_t* mp_skip, const int64_t* obs_ptr, const int32_t* obs_kf, const int32_t* mp_ref,
                        const float* mp_scale_ref, const float* mp_scale_last, float* entry_Tcw, float* entry_centre, int32_t* mp_entry,
                        float* mp_pos_out, float* normal, float* max_dist, float* min_dist, uint8_t* status);
int ccm_sim3_correction_host(int32_t n_kf, const float* kf_centre, const uint8_t* kf_bad, int32_t n_e, const int32_t* entry_kf,
                             const double* entry_Siw_new, const double* entry_Siw_old, const int64_t* slot_ptr, const int32_t* slot_mp,
                             int32_t n_mp, const float* mp_pos, const uint8_t* mp_skip, const int64_t* obs_ptr, const int32_t* obs_kf,
                             const int32_t* mp_ref, const float* mp_scale_ref, const float* mp_scale_last, float* entry_Tcw,
                             float* entry_centre, int32_t* mp_entry, float* mp_pos_out, float* normal, float* max_dist, float* min_dist,
                             uint8_t* status);

/* ---- keyframe culling --------------------------------------------------------------------------------------------------------
 * The redundancy test of LocalMapping::KeyFrameCullingV3 (cslam/src/Mapping.cpp:771-863) for every covisible keyframe of the picked
 * keyframe in one call, exactly (integer counts, one f64 comparison).  The random pick, the skips of mId.first 0 / 1 and of
 * mlpRecentAddedKFs, and the SetBadFlag calls stay with the caller; the candidates arrive already filtered, in
 * GetVectorCovisibleKeyFrames() order.
 *
 * For candidate c (row cand_kf[c]): nMPs counts the slots whose point is not null and not bad (a point at two slots counts twice);
 * nRedundant counts those whose point has nObs > th_obs and at least th_obs observers other than the candidate that are not bad and
 * whose keypoint octave is <= the slot's octave + 1.  cull[c] = nRedundant > red_thres * nMPs, in f64, strictly.
 *
 * Why one pass plus a host settle is exact: a cull that takes effect (the candidate is not bad and cand_not_erase is 0) changes
 * what later candidates read — the culled keyframe turns bad, and MapPoint::EraseObservation on each of its slots' points decrements
 * nObs, moves mpRefKF off it and can turn the point bad (nObs <= 2 after the erase, no observer left that is not bad, or mpRefKF
 * already null).  Those are the only changes, and they reach only points in the culled keyframe's slots or points that list it as an
 * observer.  So every candidate is counted over the state at the start of the member; the host then walks the candidates in order,
 * applies each effective cull and counts again a later candidate with a slot whose point an earlier cull touched.  *n_settled (may
 * be NULL) counts those candidates.  Both steps share ccm_slam_b200/csrc/keyframe_culling_math.cuh.
 *
 *   kf_bad [n_kf]          isBad() of each keyframe row at the start of the member
 *   cand_kf [n_c]          the candidate rows (each row at most once);  cand_not_erase [n_c]: mbNotErase (SetBadFlag only sets
 *                          mbToBeErased then: the verdict is reported and has no effect)
 *   slot_ptr [n_c+1], slot_mp, slot_octave [slot_ptr[n_c]]   candidate c's GetMapPointMatches() in index order as point rows (-1 null)
 *                          and pKF->mvKeysUn[i].octave of each slot
 *   mp_bad, mp_nobs, mp_ref [n_mp]   isBad(), the nObs counter as given (Observations()), the row of mpRefKF (-1 null)
 *   obs_ptr [n_mp+1], obs_kf, obs_octave [obs_ptr[n_mp]]     each point's observers in mObservations order (each keyframe at most once)
 *                          and pKFi->mvKeysUn[idx].octave of each observation
 *   th_obs                 thObs (3 in the reference);  red_thres: mfRedundancyThres (Mapping.RedThres)
 * Out: cull [n_c] (1: the member calls SetBadFlag and counts a cull), n_mps / n_red [n_c] (the two counts the decision compared, after
 * earlier culls).  A row out of range, a candidate listed twice or a null array fails with CCM_ERR_INVALID and a message naming the
 * candidate or point; nothing is written then.  No candidates: no launch.
 * ccm_keyframe_culling: one pinned upload, one launch (one CTA per candidate), one download; integer reductions only, identical bytes
 * every call.  ccm_keyframe_culling_host: the same contract without a device; the two agree bit for bit. */
int ccm_keyframe_culling(int32_t n_kf, const uint8_t* kf_bad, int32_t n_c, const int32_t* cand_kf, const uint8_t* cand_not_erase,
                         const int64_t* slot_ptr, const int32_t* slot_mp, const int32_t* slot_octave, int32_t n_mp, const uint8_t* mp_bad,
                         const int32_t* mp_nobs, const int32_t* mp_ref, const int64_t* obs_ptr, const int32_t* obs_kf,
                         const int32_t* obs_octave, int32_t th_obs, double red_thres, uint8_t* cull, int32_t* n_mps, int32_t* n_red,
                         int32_t* n_settled);
int ccm_keyframe_culling_host(int32_t n_kf, const uint8_t* kf_bad, int32_t n_c, const int32_t* cand_kf, const uint8_t* cand_not_erase,
                              const int64_t* slot_ptr, const int32_t* slot_mp, const int32_t* slot_octave, int32_t n_mp,
                              const uint8_t* mp_bad, const int32_t* mp_nobs, const int32_t* mp_ref, const int64_t* obs_ptr,
                              const int32_t* obs_kf, const int32_t* obs_octave, int32_t th_obs, double red_thres, uint8_t* cull,
                              int32_t* n_mps, int32_t* n_red, int32_t* n_settled);

#ifdef __cplusplus
}
#endif
#endif

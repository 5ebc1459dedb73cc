/*
 * oracle.h — C API of the CPU oracle (TEST INFRASTRUCTURE, NOT PRODUCT).
 *
 * The oracle is a dependency-free, single-threaded C++ restatement of the
 * reference's CPU algorithm for the BA + ORB hot path of VIS4ROB-lab/ccm_slam
 * (vendored g2o + cslam Optimizer/ORBextractor/ORBmatcher).  Only tests/,
 * __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may
 * load it.  The product library (libccm_b200.so) never links or calls it.
 *
 * PARITY PINNING: the reference ships no tests or golden vectors for this path and
 * cannot be compiled in this environment (no Eigen / OpenCV C++ / Boost / ROS), so
 * the oracle is pinned by independent witnesses instead: scipy (sparse solve,
 * finite differences, Rotation) for the BA/PGO part and Python cv2 4.13 for the
 * ORB primitives (tests/test_oracle_*.py, fixtures under tests/golden/).
 * no reference tests exist to check against — see DESIGN.md §3.  Six pieces do build from the reference's own sources, in
 * place, against the stand-in headers of oracle/ref_stub/ (oracle/Makefile `ref` -> oracle/_ref/): cslam/src/ORBextractor.cpp (on the
 * oracle's OpenCV-primitive restatements), cslam/src/ORBmatcher.cpp (on stand-in Frame / KeyFrame / MapPoint), the vendored DBoW2, and
 * g2o's Levenberg-Marquardt driver (optimization_algorithm*.cpp over stand-in SparseOptimizer / Solver classes backed by ba_oracle.cpp), and
 * g2o's vertex / edge types, Lie groups, base-edge templates and Huber kernel (over a stand-in for Eigen's small fixed-size arithmetic).
 * orb_oracle.cpp, match_oracle.cpp, proj_oracle.cpp and bow_oracle.cpp are held to that code exactly
 * (tests/test_oracle_vs_reference_{orb,matchers,dbow2,lm,g2o,single,pgo}.py); composed, the last two run every optimisation of the path
 * as reference code except the linear solve (ref_{ba,single,pgo}_full_wrap.cpp; for BA also g2o's own BlockSolver_6_3, ref_ba_block_wrap.cpp:
 * only the sparse factorisation is then the oracle's), and the oracle equals those runs bit for bit.  cslam/src/Optimizer.cpp itself builds
 * too (with the whole g2o core; liboptimizer_ref.so) and is what shim/Optimizer_shim.cpp is compared with (tests/test_shim_optimizer.py).
 *
 * Citations: G/ = cslam/thirdparty/g2o/g2o/, S/ = cslam/src/ under /root/reference.
 */
#ifndef CCM_ORACLE_H
#define CCM_ORACLE_H
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* ---- flat BA problem (same field meaning as include/ccm_b200.h) ---- */
typedef struct {
  int32_t K, P, E;
  const double* poses;       /* K*7: qx qy qz qw tx ty tz  (g2o::SE3Quat, Tcw) */
  const double* intr;        /* K*4: fx fy cx cy */
  const uint8_t* fixed;      /* K: 1 = vertex fixed */
  const double* points;      /* P*3 world xyz */
  const int32_t* obs_kf;     /* E: pose index */
  const int32_t* obs_mp;     /* E: point index */
  const float* obs_uv;       /* E*2: undistorted pixel */
  const float* obs_w;        /* E: invSigma2 of the keypoint octave */
  const uint8_t* edge_flags; /* E or NULL: bit0 = level 1 (inactive), bit1 = no robust kernel */
} orc_ba_problem;

typedef struct {
  int32_t iterations;        /* optimize(n) */
  int32_t robust;            /* 1 = Huber on every edge without bit1 */
  double huber_delta;        /* sqrt(5.99) GBA, sqrt(5.991) LocalBA */
  double lambda_init;        /* <=0: tau * max diag(H), tau = 1e-5 */
  int32_t max_trials;        /* 10 */
  const volatile uint8_t* stop; /* force-stop flag, may be NULL */
} orc_ba_options;

#define ORC_TRACE_COLS 6 /* iter, lambda_used_last_trial, chi2_after, rho, trials, lambda_after */

typedef struct {
  double* poses;             /* K*7 out */
  double* points;            /* P*3 out */
  double* chi2;              /* E out: plain e'We at the last evaluated state; inactive edges untouched */
  uint8_t* depth_pos;        /* E out: z>0 at the final estimate (all edges) */
  double* trace;             /* trace_cap*ORC_TRACE_COLS or NULL */
  int32_t trace_cap;
  int32_t trace_len;
  int32_t iters_done;        /* return value of SparseOptimizer::optimize */
  int32_t trials_total;
  double chi2_initial, chi2_final, lambda_final;
  double t_build_s, t_schur_s, t_solve_s, t_resid_s, t_total_s, t_structure_s;
} orc_ba_result;

int orc_ba_solve(const orc_ba_problem* p, const orc_ba_options* o, orc_ba_result* r);

/* pieces, for kernel-level parity tests */
/* per-edge: err[2E], Jpose[12E] (2x6 row-major), Jpoint[6E] (2x3 row-major), rho1[E], chi2[E]; returns robust chi2 sum */
double orc_ba_linearize(const orc_ba_problem* p, int robust, double huber_delta,
                        double* err, double* Jpose, double* Jpoint, double* rho1, double* chi2);
/* dense block outputs in pose/point index space (fixed poses get zero blocks):
 * Hpp[K*36] row-major 6x6, bp[K*6], Hll[P*9], bl[P*3], W[E*18] (6x3 row-major, pose-rows x point-cols) */
void orc_ba_build(const orc_ba_problem* p, int robust, double huber_delta,
                  double* Hpp, double* bp, double* Hll, double* bl, double* W);
/* one damped Schur solve at the current linearisation: dx_pose[K*6] (zero for fixed), dx_point[P*3];
 * also returns dense reduced system if S_dense (6K x 6K row-major) / bschur (6K) non-NULL. returns 0 on success */
int orc_ba_schur_solve(const orc_ba_problem* p, int robust, double huber_delta, double lambda,
                       double* dx_pose, double* dx_point, double* S_dense, double* bschur);

void orc_se3_exp(const double upd[6], double out_qt[7]);                /* G/types/se3quat.h:223-257 */
void orc_se3_mul(const double a[7], const double b[7], double out[7]);  /* G/types/se3quat.h:105-118 */
void orc_se3_map(const double qt[7], const double x[3], double out[3]); /* G/types/se3quat.h:217-220 */
void orc_pose_from_Tcw_f32(const float T[16], double out_qt[7]);        /* S/Converter.cc:40-51 */
void orc_pose_to_Tcw_f32(const double qt[7], float T[16]);              /* S/Converter.cc:53-72 */
void orc_huber(double e, double delta, double rho[3]);                  /* G/core/robust_kernel_impl.cpp:77-91 */

/* ---- Sim3 pose graph (essential graph) ---- */
typedef struct {
  int32_t K, E;
  const double* sim3;        /* K*8: qx qy qz qw tx ty tz s */
  const uint8_t* fixed;      /* K */
  const int32_t* edge_i;     /* E: vertex 0 */
  const int32_t* edge_j;     /* E: vertex 1 */
  const double* meas;        /* E*8: Sji measurement */
  int32_t fix_scale;
} orc_pgo_problem;

typedef struct {
  double* sim3;              /* K*8 out */
  double* trace; int32_t trace_cap; int32_t trace_len;
  int32_t iters_done;
  double chi2_initial, chi2_final, lambda_final;
  double t_total_s;
} orc_pgo_result;

/* analytic_jac: 0 = numeric central differences delta=1e-9 as the reference (G/core/base_binary_edge.hpp:131-205) */
int orc_pgo_solve(const orc_pgo_problem* p, int32_t iterations, double lambda_init, int32_t analytic_jac,
                  const volatile uint8_t* stop, orc_pgo_result* r);
void orc_sim3_exp(const double upd[7], double out[8]);                 /* G/types/sim3.h:70-142 */
void orc_sim3_log(const double s[8], double out[7]);                   /* G/types/sim3.h:148-230 */
void orc_sim3_mul(const double a[8], const double b[8], double out[8]);/* G/types/sim3.h:266-272 */
void orc_sim3_inv(const double a[8], double out[8]);                   /* G/types/sim3.h:233-236 */
void orc_pgo_edge_error(const double meas[8], const double si[8], const double sj[8], double err[7]);
void orc_pgo_edge_jacobian(const double meas[8], const double si[8], const double sj[8], int fix_scale, double Ji[49], double Jj[49]);
void orc_sim3_map(const double s[8], const double x[3], double out[3]);  /* G/types/sim3.h:144-146 */

/* ---- single-vertex optimisations (single_oracle.cpp) ---- */
typedef struct {
  int32_t n;                 /* correspondences = frame features with a map point */
  const double* Tcw;         /* 7: qx qy qz qw tx ty tz, Converter::toSE3Quat(Frame.mTcw) */
  const float* Xw;           /* n*3: MapPoint::GetWorldPos (f32) */
  const float* uv;           /* n*2: mvKeysUn[i].pt */
  const float* inv_sigma2;   /* n: mvInvLevelSigma2[octave] */
  float fx, fy, cx, cy;
} orc_pose_opt_problem;
/* Optimizer::PoseOptimizationClient (S/Optimizer.cpp:215-347); returns nInitialCorrespondences - nBad (0 when n < 3) */
int orc_pose_optimize(const orc_pose_opt_problem* p, double* Tcw_out /*7*/, uint8_t* outlier /*n: Frame.mvbOutlier*/);

typedef struct {
  int32_t n;                 /* matched pairs that passed the reference's validity checks */
  const double* S12;         /* 8: qx qy qz qw tx ty tz s */
  const float* P1c;          /* n*3: R1w*P1w + t1w (camera-1 frame, f32 as the reference computes it) */
  const float* P2c;          /* n*3: R2w*P2w + t2w */
  const float* uv1;          /* n*2: pKF1->mvKeysUn[i].pt */
  const float* uv2;          /* n*2: pKF2->mvKeysUn[i2].pt */
  const float* inv_sigma2_1; /* n */
  const float* inv_sigma2_2; /* n */
  float K1[4], K2[4];        /* fx fy cx cy of the two keyframes */
  float th2;
  int32_t fix_scale;
} orc_sim3_opt_problem;
/* Optimizer::OptimizeSim3 (S/Optimizer.cpp:861-1056); returns nIn (0 and S12 untouched when fewer than 10 pairs survive) */
int orc_sim3_optimize(const orc_sim3_opt_problem* p, double* S12_out /*8*/, uint8_t* inlier /*n: vpMatches1[i] kept*/);
/* the same two protocols, recording every optimize() call in `trace` (4 / 2 calls of 7 + 10 * 7 doubles, the layout of
 * ccm_pose_optimize_traced in include/ccm_b200.h); the results are those of orc_pose_optimize / orc_sim3_optimize */
int orc_pose_opt_trace(const orc_pose_opt_problem* p, double* Tcw_out, uint8_t* outlier, double* trace /*4*77*/);
int orc_sim3_opt_trace(const orc_sim3_opt_problem* p, double* S12_out, uint8_t* inlier, double* trace /*2*77*/);
/* pieces: the quadratic form all edges build at a given estimate — H (DxD row-major), b (D), err (2 per edge; Sim3: edge 2i / 2i+1) */
void orc_pose_opt_build(const orc_pose_opt_problem* p, const double* Tcw, int robust, double delta, double* H, double* b, double* err);
void orc_sim3_opt_build(const orc_sim3_opt_problem* p, const double* S12, int robust, double delta, double* H, double* b, double* err);

/* the two factorisations as services, for the stand-ins of g2o's Eigen-based linear solvers (oracle/ref_stub_g2o) */
int orc_chol_solve(int n, const double* A /*n x n row-major*/, const double* b, double* x);
void* orc_ldlt_new(void);
void orc_ldlt_free(void* h);
void orc_ldlt_reset(void* h);
int orc_ldlt_solve(void* h, int nb, int bs, const int* rowptr, const int* col, const double* val, const double* b, double* x);

/* the map update after a global BA (cslam/src/Map.cpp:1441-1570 = MapMerger.cpp:637-753); arguments as ccm_gba_map_update's
 * (include/ccm_b200.h).  Returns 0, or 1 when an origin has no BA result.  cv::gemm's f32 rounding pinned against cv2 4.13
 * (tests/golden/map_update_cv2.npz). */
int orc_gba_map_update(int32_t n_kf, const int32_t* kf_parent, const uint8_t* kf_optimized, const float* kf_Tcw, float* kf_TcwGBA,
                       uint8_t* kf_visited, int32_t n_mp, const uint8_t* mp_state, const int32_t* mp_ref, const float* mp_pos,
                       const float* mp_pos_gba, float* mp_pos_out, uint8_t* mp_corrected);

#ifdef __cplusplus
}
#endif
#endif

// ba_kernels.cuh — sm_90a kernels of the Levenberg-Marquardt bundle-adjustment hot path.
//
// Data layout in HBM (one landmark shard per GPU; poses replicated):
//   pose      [K][7]  f64  AoS  (gathered per observation, K is small -> L1/L2 resident)
//   pt        [Pl][3] f64  AoS  (observations are sorted by landmark -> consecutive threads share lines)
//   o_kf,o_lm [El]    i32       observation -> keyframe index / local landmark index (landmark order)
//   o_uv      [El]    float2    undistorted pixel
//   o_w       [El]    f32       invSigma2; sign bit = "no robust kernel"; 0 = inactive edge (level 1)
//   Z         [El][18] f64 AoS  W * U^-1 with (Hll + lambda I) = U^T U; gathered 144 B rows by the Schur products
//             (W = Hpl block per observation, 6x3, lives in shared memory only; ccm_ba_debug_build exports it as [18][Ep] SoA)
//   Hll       [6][Pl]  f64 SoA  upper triangle (00 01 02 11 12 22);  bl [3][Pl]
//   Hpp       [Kf][36], bp [Kf][6] ; U_val [nub][36] upper Schur blocks ; s_val [nnzb][36] full block-CSR for PCG
//   units     [nunits+1] i32    landmark-aligned CTA schedule of k_linearize / k_backsub_points (runs of whole landmarks)
//
// Kernels (reference loop each one replaces: SURVEY.md §2.2 K1..K7):
//   k_linearize   K1..K4 residual + Huber + Jacobians + chi2, Hll/bl summed per landmark in the CTA (no atomics), and with lambda
//                        Z = W U^-1, g = U^-T bl (lambda folded in, no setLambda/restoreDiagonal passes); a Z-only launch after a
//                        rejected trial
//   k_pose_pass   K2     Hpp/bp per free pose (CTA per pose, register accumulation, no atomics)
//   k_residual    K1     robust chi2 of a trial state
//   k_schur_mma   K4     S_ab = sum_l Z_al Z_bl^T over precomputed product lists (register accumulation, no atomics)
//   k_finalize_S  K4     S = [a==b](Hpp + lambda I) - products, mirrored to full block-CSR
//   k_block_jacobi K5    6x6 inverses of the diagonal blocks + bschur
//   k_pcg         K5     persistent cooperative PCG on the reduced camera system
//   k_update_poses / k_backsub_points  K6+K7  back-substitution (landmark-aligned, Z rows coalesced), oplus into the trial state,
//                                             gain-ratio denominator
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "ba_math.cuh"
#include "pcg.cuh"

namespace ccm {
namespace ba {

using ccm::TPB;
using ccm::warp_sum;
using ccm::block_sum;

__device__ __forceinline__ Pose load_pose(const double* __restrict__ pose, int k) {
  const double* p = pose + 7 * (size_t)k;
  Pose T;
  T.qx = __ldg(p); T.qy = __ldg(p + 1); T.qz = __ldg(p + 2); T.qw = __ldg(p + 3);
  T.tx = __ldg(p + 4); T.ty = __ldg(p + 5); T.tz = __ldg(p + 6);
  return T;
}

// ------------------------------------------------------------------------------------------------------------
// Landmark-aligned CTA schedule (k_linearize, k_backsub_points): a unit is a run [units[c], units[c+1]) of whole landmarks, cut
// once per handle by k_lin_heads + a scan.  A unit of landmarks with <= LIN_SMALL observations each holds <= LIN_TILE observations
// (its landmarks all start inside one bucket of LIN_BUCKET observations, the last one ends < LIN_SMALL past it); a larger landmark
// is a unit of its own, walked in chunks of LIN_TILE.  A unit holds <= LIN_TILE landmarks (runs of empty ones are cut too).
constexpr int LIN_TILE = 128;    // threads of a CTA = observations per chunk
constexpr int LIN_SMALL = 32;
constexpr int LIN_BUCKET = LIN_TILE - LIN_SMALL + 1;
static_assert(LIN_TILE % 32 == 0 && LIN_SMALL < LIN_TILE, "schedule constants");

__global__ void __launch_bounds__(TPB) k_lin_heads(const int* __restrict__ lm_ptr, int Pl, int* __restrict__ head) {
  const int l = blockIdx.x * TPB + threadIdx.x;
  if (l >= Pl) return;
  const int b = lm_ptr[l], n = lm_ptr[l + 1] - b;
  int h = l % LIN_TILE == 0 || n > LIN_SMALL;
  if (!h) {
    const int bprev = lm_ptr[l - 1];
    h = b / LIN_BUCKET != bprev / LIN_BUCKET || b - bprev > LIN_SMALL;
  }
  head[l] = h;
}

// An inactive edge (weight 0: g2o's level 1, which g2o never evaluates) must contribute exact zeros, also where its point sits at
// depth 0 and its projection is not finite (0 * inf = NaN).  Its linearisation runs like any other, without a divergent branch, and
// is then replaced by zeros; an active edge's values pass through unchanged.
__device__ __forceinline__ void drop_inactive(double w, ObsLin& L) {
  const bool on = w != 0.0;
  L.ex = on ? L.ex : 0.0; L.ey = on ? L.ey : 0.0; L.chi2 = on ? L.chi2 : 0.0;
#pragma unroll
  for (int i = 0; i < 6; i++) L.Jl[i] = on ? L.Jl[i] : 0.0;
#pragma unroll
  for (int i = 0; i < 12; i++) L.Jp[i] = on ? L.Jp[i] : 0.0;
}

// K1+K2 of one observation for the thread's slot t of the chunk [c0, c1): the 6x3 W row into s_w (row stride 19), and with
// hsum the 9 point-side terms (Hll upper, bl) into s_h and the robust chi2 into chi.  dbgW (debug export only): W as
// [18][Ep] SoA.  Returns the observation's landmark (-1 past the chunk).
__device__ __forceinline__ int lin_obs(int c0, int c1, const int* __restrict__ o_kf, const int* __restrict__ o_lm,
                                       const float2* __restrict__ o_uv, const float* __restrict__ o_w,
                                       const double* __restrict__ pose, const double* __restrict__ intr,
                                       const int* __restrict__ pose_slot, const double* __restrict__ pt, int robust, double delta,
                                       bool hsum, double* s_w, double* s_h, double& chi, double* __restrict__ dbgW, size_t Ep) {
  const int t = threadIdx.x;
  const int e = c0 + t;
  if (e >= c1) return -1;
  const int kf = o_kf[e];
  const int lm = o_lm[e];
  const float2 uv = o_uv[e];
  const float wf = o_w[e];
  const double w = fabs((double)wf);
  const bool rob = robust && !signbit(wf);
  const Pose T = load_pose(pose, kf);
  const double in4[4] = {__ldg(intr + 4 * (size_t)kf), __ldg(intr + 4 * (size_t)kf + 1),
                         __ldg(intr + 4 * (size_t)kf + 2), __ldg(intr + 4 * (size_t)kf + 3)};
  const double* X = pt + 3 * (size_t)lm;
  ObsLin L;
  linearize_obs(T, in4, X[0], X[1], X[2], (double)uv.x, (double)uv.y, w, L);
  drop_inactive(w, L);
  double rho0 = L.chi2, rho1 = 1.0;
  if (rob) huber(L.chi2, delta, rho0, rho1);
  const double wo = rho1 * w;                     // weightedOmega = rho'(chi2) * omega
  if (hsum) {
    chi += rho0;
    const double r0 = -wo * L.ex, r1 = -wo * L.ey;  // omega_r = -omega e * rho'
    double* h = s_h + t * 9;
    h[0] = wo * (L.Jl[0] * L.Jl[0] + L.Jl[3] * L.Jl[3]);
    h[1] = wo * (L.Jl[0] * L.Jl[1] + L.Jl[3] * L.Jl[4]);
    h[2] = wo * (L.Jl[0] * L.Jl[2] + L.Jl[3] * L.Jl[5]);
    h[3] = wo * (L.Jl[1] * L.Jl[1] + L.Jl[4] * L.Jl[4]);
    h[4] = wo * (L.Jl[1] * L.Jl[2] + L.Jl[4] * L.Jl[5]);
    h[5] = wo * (L.Jl[2] * L.Jl[2] + L.Jl[5] * L.Jl[5]);
    h[6] = L.Jl[0] * r0 + L.Jl[3] * r1;
    h[7] = L.Jl[1] * r0 + L.Jl[4] * r1;
    h[8] = L.Jl[2] * r0 + L.Jl[5] * r1;
  }
  // pose-landmark block W = Jp^T (wo I) Jl  (zero when the pose vertex is fixed)
  const double wz = __ldg(pose_slot + kf) >= 0 ? wo : 0.0;
#pragma unroll
  for (int r = 0; r < 6; r++) {
    const double a = wz * L.Jp[r], b = wz * L.Jp[6 + r];
#pragma unroll
    for (int c = 0; c < 3; c++) {
      const double v = a * L.Jl[c] + b * L.Jl[3 + c];
      s_w[t * 19 + r * 3 + c] = v;
      if (dbgW != nullptr) dbgW[(size_t)(r * 3 + c) * Ep + e] = v;
    }
  }
  return lm;
}

// K1..K4 first half, one CTA per unit of the landmark schedule (grid-stride over the units):
//   pass 1  per observation: residual, Huber weight, Jacobians, chi2; W row and the Hll / bl terms staged in shared memory;
//           per landmark a fixed-order sum of its terms (no atomics: deterministic)
//   factor  per landmark: LIN_H writes Hll / bl; LIN_Z factors Hll + lambda I = U^T U and writes g = U^-T bl
//   pass 2  (LIN_Z) per observation: Z = W U^-1 in place, written AoS through coalesced rows.  A landmark larger than a chunk
//           recomputes its W rows here, chunk by chunk.
// mode is a run-time argument on purpose: a Z-only launch (LIN_Z, recompute at the current state after lambda changed) then runs
// the same instructions as the fused one and gives bit-identical Z.
//   reads 20 B/obs + cache-resident gathers ; writes 144 B/obs (Z) + 72 B/landmark (Hll, bl) + 24 B/landmark (g)
enum { LIN_H = 1, LIN_Z = 2 };
__global__ void __launch_bounds__(LIN_TILE, 6) k_linearize(
    const int* __restrict__ units, int nunits, const int* __restrict__ lm_ptr, const int* __restrict__ o_kf,
    const int* __restrict__ o_lm, const float2* __restrict__ o_uv, const float* __restrict__ o_w, const double* __restrict__ pose,
    const double* __restrict__ intr, const int* __restrict__ pose_slot, const double* __restrict__ pt, int Pl, int robust,
    double delta, double lambda, int mode, double* __restrict__ Hll, double* __restrict__ bl, double* __restrict__ gvec,
    double* __restrict__ Z, double* __restrict__ chi2_partials, double* __restrict__ dbgW, size_t Ep) {
  __shared__ double s_w[LIN_TILE * 19];   // W rows, then Z rows in place (odd stride: conflict-free row access)
  __shared__ double s_h[LIN_TILE * 9];    // per observation the 9 terms; then per landmark, in its first slot, their sums, then U
  __shared__ double red[LIN_TILE / 32];
  const int t = threadIdx.x;
  double chi = 0.0;
  for (int c = blockIdx.x; c < nunits; c += gridDim.x) {
    const int l0 = units[c], nlm = units[c + 1] - l0;
    const int ob = lm_ptr[l0], oe = lm_ptr[l0 + nlm];
    const int nch = oe - ob > LIN_TILE ? (oe - ob + LIN_TILE - 1) / LIN_TILE : 1;   // > 1: the unit is one landmark
    int slot = 0;        // s_h slot of this thread's landmark
    double acc = 0.0;    // nch > 1: thread i < 9 carries term i over the chunks
    for (int k = 0; k < nch; k++) {
      const int c0 = ob + k * LIN_TILE, c1 = min(oe, c0 + LIN_TILE);
      const int lm = lin_obs(c0, c1, o_kf, o_lm, o_uv, o_w, pose, intr, pose_slot, pt, robust, delta, true, s_w, s_h, chi, dbgW, Ep);
      if (nch == 1 && lm >= 0) slot = __ldg(lm_ptr + lm) - ob;
      __syncthreads();
      for (int q = t; q < nlm * 9; q += LIN_TILE) {
        const int j = q / 9, i = q - 9 * j;
        const int b = max(__ldg(lm_ptr + l0 + j), c0), e = min(__ldg(lm_ptr + l0 + j + 1), c1);
        double v = 0.0;
        for (int o = b; o < e; o++) v += s_h[(o - c0) * 9 + i];
        if (nch == 1) {
          if (e > b) s_h[(b - c0) * 9 + i] = v;   // column i of this landmark's rows is read by this thread only
        } else {
          acc += v;
          if (k == nch - 1) s_h[i] = acc;
        }
      }
      __syncthreads();
    }
    if (t < nlm) {
      const int l = l0 + t, b = __ldg(lm_ptr + l);
      const bool empty = __ldg(lm_ptr + l + 1) == b;
      double* hs = s_h + (nch > 1 ? 0 : (b - ob) * 9);
      double d[9];
#pragma unroll
      for (int i = 0; i < 9; i++) d[i] = empty ? 0.0 : hs[i];
      if (mode & LIN_H) {
#pragma unroll
        for (int i = 0; i < 6; i++) Hll[(size_t)i * Pl + l] = d[i];
#pragma unroll
        for (int i = 0; i < 3; i++) bl[(size_t)i * Pl + l] = d[6 + i];
      }
      if (mode & LIN_Z) {
        d[0] += lambda; d[3] += lambda; d[5] += lambda;
        double u[6], g[3];
        chol3_upper(d, u);
        UTinv_times(u, d + 6, g);
        gvec[3 * (size_t)l] = g[0]; gvec[3 * (size_t)l + 1] = g[1]; gvec[3 * (size_t)l + 2] = g[2];
        if (!empty)
#pragma unroll
          for (int i = 0; i < 6; i++) hs[i] = u[i];
      }
    }
    __syncthreads();
    if (!(mode & LIN_Z)) continue;
    for (int k = 0; k < nch; k++) {
      const int c0 = ob + k * LIN_TILE, c1 = min(oe, c0 + LIN_TILE);
      if (nch > 1) {
        double unused = 0.0;
        lin_obs(c0, c1, o_kf, o_lm, o_uv, o_w, pose, intr, pose_slot, pt, robust, delta, false, s_w, s_h, unused, nullptr, Ep);
        __syncthreads();
      }
      if (c0 + t < c1) {
        const double* u = s_h + slot * 9;
#pragma unroll
        for (int r = 0; r < 6; r++) {
          double* row = s_w + t * 19 + r * 3;
          row_times_Uinv(u, row[0], row[1], row[2], row[0], row[1], row[2]);
        }
      }
      __syncthreads();
      const int n = (c1 - c0) * 18;
      double* out = Z + (size_t)c0 * 18;
      for (int i = t; i < n; i += LIN_TILE) out[i] = s_w[(i / 18) * 19 + (i % 18)];
      __syncthreads();
    }
  }
  const double tot = block_sum(chi, red);
  if (t == 0) chi2_partials[blockIdx.x] = tot;
}

// K1 on a (trial) state: robust chi2 only.  20 B/obs read.
__global__ void __launch_bounds__(TPB) k_residual(
    const int* __restrict__ o_kf, const int* __restrict__ o_lm, const float2* __restrict__ o_uv,
    const float* __restrict__ o_w, const double* __restrict__ pose, const double* __restrict__ intr,
    const double* __restrict__ pt, int E, int robust, double delta, double* __restrict__ chi2_partials) {
  __shared__ double red[TPB / 32];
  double chi_acc = 0.0;
  for (long long e = (long long)blockIdx.x * TPB + threadIdx.x; e < E; e += (long long)gridDim.x * TPB) {
    const int kf = o_kf[e];
    const int lm = o_lm[e];
    const float2 uv = o_uv[e];
    const float wf = o_w[e];
    const double w = fabs((double)wf);
    const Pose T = load_pose(pose, kf);
    const double in4[4] = {__ldg(intr + 4 * (size_t)kf), __ldg(intr + 4 * (size_t)kf + 1),
                           __ldg(intr + 4 * (size_t)kf + 2), __ldg(intr + 4 * (size_t)kf + 3)};
    const double* X = pt + 3 * (size_t)lm;
    double ex, ey, chi2, Xc[3];
    project_residual(T, in4, X[0], X[1], X[2], (double)uv.x, (double)uv.y, w, ex, ey, chi2, Xc);
    double rho0 = chi2, rho1;
    if (robust && !signbit(wf)) huber(chi2, delta, rho0, rho1);
    chi_acc += w != 0.0 ? rho0 : 0.0;   // an inactive edge adds nothing, even where its chi2 is not finite (drop_inactive)
  }
  const double tot = block_sum(chi_acc, red);
  if (threadIdx.x == 0) chi2_partials[blockIdx.x] = tot;
}

// per-edge report for the caller: plain chi2 at the last evaluated state, depth sign at the final estimate
__global__ void __launch_bounds__(TPB) k_edge_report(
    const int* __restrict__ o_kf, const int* __restrict__ o_lm, const float2* __restrict__ o_uv,
    const float* __restrict__ o_w, const double* __restrict__ pose_eval, const double* __restrict__ pt_eval,
    const double* __restrict__ pose_fin, const double* __restrict__ pt_fin, const double* __restrict__ intr, int E,
    double* __restrict__ chi2_out, uint8_t* __restrict__ depth_out) {
  const long long e = (long long)blockIdx.x * TPB + threadIdx.x;
  if (e >= E) return;
  const int kf = o_kf[e], lm = o_lm[e];
  const float2 uv = o_uv[e];
  const double w = fabs((double)o_w[e]);
  const double in4[4] = {intr[4 * (size_t)kf], intr[4 * (size_t)kf + 1], intr[4 * (size_t)kf + 2], intr[4 * (size_t)kf + 3]};
  double ex, ey, chi2, Xc[3];
  {
    const Pose T = load_pose(pose_eval, kf);
    const double* X = pt_eval + 3 * (size_t)lm;
    project_residual(T, in4, X[0], X[1], X[2], (double)uv.x, (double)uv.y, w, ex, ey, chi2, Xc);
    chi2_out[e] = chi2;
  }
  {
    const Pose T = load_pose(pose_fin, kf);
    const double* X = pt_fin + 3 * (size_t)lm;
    project_residual(T, in4, X[0], X[1], X[2], (double)uv.x, (double)uv.y, w, ex, ey, chi2, Xc);
    depth_out[e] = Xc[2] > 0.0 ? 1 : 0;
  }
}

// ------------------------------------------------------------------------------------------------------------
// per free pose: its observations packed as (u, v, signed weight, landmark) in diagonal-product-list order, so that the pose
// pass streams 16 coalesced bytes per observation instead of chasing four index arrays
__global__ void __launch_bounds__(128) k_pack_pose_obs(const uint2* __restrict__ prod, const unsigned* __restrict__ u_prod_ptr,
                                                       const int* __restrict__ u_diag, const unsigned* __restrict__ kobs_ptr,
                                                       const int* __restrict__ o_lm, const float2* __restrict__ o_uv,
                                                       const float* __restrict__ o_w, float4* __restrict__ kobs) {
  const int a = blockIdx.x;
  const unsigned beg = u_prod_ptr[u_diag[a]], n = u_prod_ptr[u_diag[a] + 1] - beg, dst = kobs_ptr[a];
  for (unsigned i = threadIdx.x; i < n; i += blockDim.x) {
    const unsigned e = prod[beg + i].x;
    const float2 uv = o_uv[e];
    kobs[dst + i] = make_float4(uv.x, uv.y, o_w[e], __int_as_float(o_lm[e]));
  }
}

// K2 pose side: one CTA per free pose; its observations are the product list of the diagonal Schur block (a,a).
__global__ void __launch_bounds__(128) k_pose_pass(
    const float4* __restrict__ kobs, const unsigned* __restrict__ kobs_ptr,
    const int* __restrict__ slot_pose, const double* __restrict__ pose, const double* __restrict__ intr,
    const double* __restrict__ pt, int robust, double delta, double* __restrict__ Hpp, double* __restrict__ bp) {
  __shared__ double red[27][4];
  const int a = blockIdx.x;
  const int kf = slot_pose[a];
  const unsigned beg = kobs_ptr[a], end = kobs_ptr[a + 1];
  const Pose T = load_pose(pose, kf);
  const double in4[4] = {intr[4 * (size_t)kf], intr[4 * (size_t)kf + 1], intr[4 * (size_t)kf + 2], intr[4 * (size_t)kf + 3]};
  double acc[27];
#pragma unroll
  for (int i = 0; i < 27; i++) acc[i] = 0.0;
  for (unsigned p = beg + threadIdx.x; p < end; p += blockDim.x) {
    const float4 ob = kobs[p];
    const int lm = __float_as_int(ob.w);
    const float wf = ob.z;
    const double w = fabs((double)wf);
    const double* X = pt + 3 * (size_t)lm;
    ObsLin L;
    linearize_obs(T, in4, X[0], X[1], X[2], (double)ob.x, (double)ob.y, w, L);
    drop_inactive(w, L);
    double rho0, rho1 = 1.0;
    if (robust && !signbit(wf)) huber(L.chi2, delta, rho0, rho1);
    const double wo = rho1 * w;
    const double r0 = -wo * L.ex, r1 = -wo * L.ey;
    int q = 0;
#pragma unroll
    for (int i = 0; i < 6; i++)
#pragma unroll
      for (int j = i; j < 6; j++) acc[q++] += wo * (L.Jp[i] * L.Jp[j] + L.Jp[6 + i] * L.Jp[6 + j]);
#pragma unroll
    for (int i = 0; i < 6; i++) acc[21 + i] += L.Jp[i] * r0 + L.Jp[6 + i] * r1;
  }
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
#pragma unroll
  for (int i = 0; i < 27; i++) {
    const double v = warp_sum(acc[i]);
    if (lane == 0) red[i][wid] = v;
  }
  __syncthreads();
  if (threadIdx.x < 27) {
    const double v = red[threadIdx.x][0] + red[threadIdx.x][1] + red[threadIdx.x][2] + red[threadIdx.x][3];
    if (threadIdx.x < 21) {
      // unpack upper-triangular index -> (i,j)
      int i = 0, q = threadIdx.x;
      while (q >= 6 - i) { q -= 6 - i; i++; }
      const int j = i + q;
      Hpp[(size_t)a * 36 + i * 6 + j] = v;
      Hpp[(size_t)a * 36 + j * 6 + i] = v;
    } else {
      bp[(size_t)a * 6 + (threadIdx.x - 21)] = v;
    }
  }
}

// max |diag| over Hpp and Hll -> bits of a non-negative double, atomicMax as unsigned long long
__global__ void __launch_bounds__(TPB) k_max_diag(const double* __restrict__ Hpp, int Kf, const double* __restrict__ Hll,
                                                  int Pl, unsigned long long* __restrict__ out) {
  double m = 0.0;
  const long long n1 = (long long)Kf * 6, n2 = (long long)Pl * 3;
  for (long long i = (long long)blockIdx.x * TPB + threadIdx.x; i < n1 + n2; i += (long long)gridDim.x * TPB) {
    double v;
    if (i < n1) {
      v = Hpp[(i / 6) * 36 + (i % 6) * 7];
    } else {
      const long long j = i - n1;
      const int d = (int)(j / Pl);  // 0,1,2 -> rows 0,3,5 of the packed upper triangle
      const int row = d == 0 ? 0 : (d == 1 ? 3 : 5);
      v = Hll[(size_t)row * Pl + (j % Pl)];
    }
    m = fmax(m, fabs(v));
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m = fmax(m, __shfl_xor_sync(0xffffffffu, m, o));
  if ((threadIdx.x & 31) == 0) atomicMax(out, (unsigned long long)__double_as_longlong(m));
}

// single-block deterministic sum of partials: out[0] = sum
__global__ void __launch_bounds__(1024) k_sum_partials(const double* __restrict__ partials, int n, double* __restrict__ out) {
  __shared__ double red[32];
  double v = 0.0;
  for (int i = threadIdx.x; i < n; i += blockDim.x) v += partials[i];
  const double t = block_sum(v, red);
  if (threadIdx.x == 0) out[0] = t;
}

// ------------------------------------------------------------------------------------------------------------
// K4: Schur products, tensor-core form.  One warp per upper block u = (a,b) walks the block's precomputed product list
// (register accumulation, no atomics):
//   acc[r][c] += sum_k Z_oa[r][k] * Z_ob[c][k]  over the list; diagonal blocks also build bneg_a = sum_o Z_o g_l(o).
// Outputs are written NEGATED (S = Hpp + lambda I - sum).  One product Z_oa (6x3) . Z_ob^T (3x6) is ONE
// mma.sync.m8n8k4.f64 whose operand fragments are exactly one coalesced 144-byte row each:
//   A (8x4 row-major): lane t holds A[t/4][t%4] = Z_oa[t/4][t%4]        rows 6,7 and column 3 are zero padding
//   B (4x8 col-major): lane t holds B[t%4][t/4] = Z_ob[t/4][t%4]        -> the same offset (t/4)*3 + t%4 into the row
//   C (8x8)          : lane t holds C[t/4][2*(t%4)], C[t/4][2*(t%4)+1]  accumulated in place over the product list
// i.e. 18 lanes x 8 B per operand (2 cache lines), no cross-lane reduction.  Diagonal blocks put g_l into B's column 6, so
// C[r][6] = sum_o Z_o[r][:] . g_l(o) = bneg comes out of the same instruction.  Two accumulator sets (products alternate) keep
// two MMA chains in flight; they are added in a fixed order: deterministic per list order.
// The UNROLL list entries of a batch come in with ONE coalesced load (lane j takes entry j) and reach the other lanes by shuffle,
// instead of UNROLL broadcast loads.  Off-diagonal blocks request the entries of batch k+1 before the rows of batch k, so the
// entry -> row dependence costs one memory latency per batch instead of two.  On H100 the kernel is bound by the rows it keeps in
// flight: the 2 * UNROLL rows of a batch are requested together, and UNROLL 16 at 66 registers runs a cfg5 launch in 9.6 ms against
// 11.3 at UNROLL 8 (48 registers), 10.0 at 32 and 12.7 at 4 (H100 80GB HBM3, 700 W).  (dmma_884: pcg.cuh)
// Holding every row of a batch in its own registers (96, 20 warps per SM) beats squeezing the batch into 66 registers (28 warps): fewer
// warps, but each keeps all 32 rows of its batch in flight, and a cfg5 launch took 8.3-8.6 ms against 9.5 (128-thread CTAs).  Capping
// it at 64 registers for 32 warps per SM (128, 64, 32 or 256-thread CTAs) gives 9.7-10.9 ms (H100 80GB HBM3, 700 W).
//
// Schedule: one CTA of SCHUR_WARPS warps per SM.  The upper blocks of a block row share its a-side rows of Z, so they run on one SM
// at the same time, and since every list is in landmark order (k_row_products) they walk those rows in the same direction: the
// a-side fetches of a row's blocks meet in L1.  The work is a row-major sequence of tasks (a task: the upper blocks of one row,
// longest list first; a row of more than SCHUR_TASK blocks is cut into several tasks, so that one long row - a loop closure, a
// merged map - cannot serialise the end of the launch).  CTAs take tasks from a global counter in order, which keeps the rows in
// progress across the device as narrow as with one warp per block; a CTA's warps take the blocks of its current task from a
// shared counter, and the warp that exhausts it takes the next task for the CTA while the others finish their blocks: no barrier.
// A cfg5 launch takes 7.5-7.9 ms against 8.3-8.7 with one warp per block and four blocks per CTA; two adjacent rows per task
// (tasks of up to 128 blocks) take 9.0 (H100 80GB HBM3, 700 W).
constexpr int SCHUR_WARPS = 20;                 // 640 threads x 96 registers fill the register file: the warps per SM of 5 x 128
constexpr int SCHUR_CTA = SCHUR_WARPS * 32;
constexpr int SCHUR_TASK = 64;                  // most blocks of one task
__device__ __forceinline__ void schur_block(int u, int lane, const uint2* __restrict__ prod, const unsigned* __restrict__ u_prod_ptr,
                                            const int* __restrict__ u_row, const int* __restrict__ u_col,
                                            const double* __restrict__ Z, const int* __restrict__ o_lm,
                                            const double* __restrict__ gvec, double* __restrict__ U_val, double* __restrict__ bneg) {
  constexpr int UNROLL = 16;  // products per batch; even: they alternate between the two accumulator sets; <= 32 (one entry per lane)
  const int m = lane >> 2, k = lane & 3;
  const bool ld = m < 6 && k < 3;
  constexpr int zs = 18;   // doubles per row of Z.  Padded rows (a 128-byte line per half-warp, 160 / 192 / 256-byte strides) were measured
                           // and are no faster
  // padding lanes read an element their own half-warp reads anyway (no extra line) and discard it
  const int off = ld ? m * 3 + k : (lane < 16 ? 0 : 12);
  const unsigned beg = u_prod_ptr[u], end = u_prod_ptr[u + 1];
  const int row = u_row[u];
  const bool diag = row == u_col[u];
  double c00 = 0.0, c01 = 0.0, c10 = 0.0, c11 = 0.0;
  unsigned p = beg;
  if (!diag) {
    uint2 nxv = make_uint2(0u, 0u);
    if (p + UNROLL <= end && lane < UNROLL) nxv = prod[p + lane];
    for (; p + UNROLL <= end; p += UNROLL) {
      uint2 pr[UNROLL];
#pragma unroll
      for (int j = 0; j < UNROLL; j++) { pr[j].x = __shfl_sync(0xffffffffu, nxv.x, j); pr[j].y = __shfl_sync(0xffffffffu, nxv.y, j); }
      if (p + 2 * UNROLL <= end && lane < UNROLL) nxv = prod[p + UNROLL + lane];
      double a[UNROLL], b[UNROLL];
#pragma unroll
      for (int j = 0; j < UNROLL; j++) {
        a[j] = Z[(size_t)pr[j].x * zs + off];
        b[j] = Z[(size_t)pr[j].y * zs + off];
      }
#pragma unroll
      for (int j = 0; j < UNROLL; j += 2) {
        dmma_884(c00, c01, ld ? a[j] : 0.0, ld ? b[j] : 0.0);
        dmma_884(c10, c11, ld ? a[j + 1] : 0.0, ld ? b[j + 1] : 0.0);
      }
    }
    for (; p < end; p++) {
      const uint2 pr = prod[p];
      const double a = Z[(size_t)pr.x * zs + off], b = Z[(size_t)pr.y * zs + off];
      if ((p - beg) & 1u) dmma_884(c10, c11, ld ? a : 0.0, ld ? b : 0.0);  // warp-uniform branch
      else dmma_884(c00, c01, ld ? a : 0.0, ld ? b : 0.0);
    }
  } else {
    // diagonal block (Kf of them): lanes 24..26 carry g_l in column 6 of B, so C[r][6] accumulates bneg
    const bool gl = m == 6 && k < 3;
    // batches of UNROLL products: entries by one coalesced load, then all rows, landmark ids and g_l of the batch in flight together
    for (; p + UNROLL <= end; p += UNROLL) {
      unsigned ex = 0u;
      if (lane < UNROLL) ex = prod[p + lane].x;
      unsigned e[UNROLL];
#pragma unroll
      for (int j = 0; j < UNROLL; j++) e[j] = __shfl_sync(0xffffffffu, ex, j);
      double a[UNROLL], g[UNROLL];
      int lm[UNROLL];
#pragma unroll
      for (int j = 0; j < UNROLL; j++) {
        a[j] = Z[(size_t)e[j] * zs + off];
        lm[j] = gl ? o_lm[e[j]] : 0;
      }
#pragma unroll
      for (int j = 0; j < UNROLL; j++) g[j] = gl ? gvec[3 * (size_t)lm[j] + k] : 0.0;
#pragma unroll
      for (int j = 0; j < UNROLL; j += 2) {
        dmma_884(c00, c01, ld ? a[j] : 0.0, gl ? g[j] : (ld ? a[j] : 0.0));
        dmma_884(c10, c11, ld ? a[j + 1] : 0.0, gl ? g[j + 1] : (ld ? a[j + 1] : 0.0));
      }
    }
    for (; p < end; p++) {
      const uint2 pr = prod[p];
      const double a = Z[(size_t)pr.x * zs + off];
      double b = a;   // a diagonal list holds (e, e) pairs only: one row serves both operands
      if (!ld) b = 0.0;
      if (gl) b = gvec[3 * (size_t)o_lm[pr.x] + k];
      if ((p - beg) & 1u) dmma_884(c10, c11, ld ? a : 0.0, b);
      else dmma_884(c00, c01, ld ? a : 0.0, b);
    }
  }
  c00 += c10; c01 += c11;
  if (ld) {
    U_val[(size_t)u * 36 + m * 6 + 2 * k] = -c00;
    U_val[(size_t)u * 36 + m * 6 + 2 * k + 1] = -c01;
  }
  if (diag && m < 6 && k == 3) bneg[(size_t)row * 6 + m] = -c00;  // C[m][6]
}

// task_ptr [ntasks+1]: each task's range in u_sched (the upper blocks, row-major, longest list first within a row); next_task: 0
// before the launch
__global__ void __launch_bounds__(SCHUR_CTA, 1) k_schur_mma(const uint2* __restrict__ prod, const unsigned* __restrict__ u_prod_ptr,
                                                         const int* __restrict__ u_row, const int* __restrict__ u_col,
                                                         const int* __restrict__ u_sched, const int* __restrict__ task_ptr,
                                                         int ntasks, int* __restrict__ next_task, const double* __restrict__ Z,
                                                         const int* __restrict__ o_lm, const double* __restrict__ gvec,
                                                         double* __restrict__ U_val, double* __restrict__ bneg) {
  __shared__ unsigned long long s_state;   // (current task << 32) | blocks of it handed out
  const int lane = threadIdx.x & 31;
  if (threadIdx.x == 0) s_state = (unsigned long long)atomicAdd(next_task, 1) << 32;
  __syncthreads();
  for (;;) {
    unsigned long long st = 0;
    if (lane == 0) st = atomicAdd(&s_state, 1ull);
    st = __shfl_sync(0xffffffffu, st, 0);
    const int t = (int)(st >> 32), i = (int)(unsigned)st;
    if (t >= ntasks) break;
    const int b0 = __ldg(task_ptr + t), n = __ldg(task_ptr + t + 1) - b0;
    if (i < n) {
      schur_block(__ldg(u_sched + b0 + i), lane, prod, u_prod_ptr, u_row, u_col, Z, o_lm, gvec, U_val, bneg);
    } else if (lane == 0) {
      if (i == n) atomicExch(&s_state, (unsigned long long)atomicAdd(next_task, 1) << 32);   // this warp moves the CTA on
      else while ((int)(*(volatile unsigned long long*)&s_state >> 32) == t) {}            // wait until that is done
    }
    __syncwarp();
  }
}

// S (full block-CSR) from the upper blocks: diagonal gets Hpp + lambda I, lower blocks are transposed copies.
__global__ void __launch_bounds__(TPB) k_finalize_S(const int* __restrict__ s_row, const int* __restrict__ s_col,
                                                    const int* __restrict__ csr_u, long long nnzb,
                                                    const double* __restrict__ U_val, const double* __restrict__ Hpp,
                                                    double lambda, double* __restrict__ s_val) {
  const long long i = (long long)blockIdx.x * TPB + threadIdx.x;
  if (i >= nnzb * 36) return;
  const long long pos = i / 36;
  const int ent = (int)(i % 36);
  const int a = s_row[pos], b = s_col[pos];
  const int u = csr_u[pos];
  double v;
  if (a <= b) {
    v = U_val[(size_t)u * 36 + ent];
    if (a == b) {
      v += Hpp[(size_t)a * 36 + ent];
      if (ent % 7 == 0) v += lambda;
    }
  } else {
    v = U_val[(size_t)u * 36 + (ent % 6) * 6 + ent / 6];
  }
  s_val[i] = v;
}

// block-Jacobi preconditioner: Minv_a = inverse(S_aa) by Cholesky; bschur = bp + bneg
__global__ void __launch_bounds__(128) k_block_jacobi(const int* __restrict__ s_diag, const double* __restrict__ s_val,
                                                      const double* __restrict__ bp, const double* __restrict__ bneg,
                                                      int Kf, double* __restrict__ Minv, double* __restrict__ bschur,
                                                      int* __restrict__ fail) {
  const int a = blockIdx.x * blockDim.x + threadIdx.x;
  if (a >= Kf) return;
  double A[36], Li[36];
  const double* src = s_val + (size_t)s_diag[a] * 36;
#pragma unroll
  for (int i = 0; i < 36; i++) A[i] = src[i];
  // Cholesky A = L L^T (lower), in place
  bool ok = true;
#pragma unroll
  for (int j = 0; j < 6; j++) {
    double d = A[j * 6 + j];
#pragma unroll
    for (int k = 0; k < j; k++) d -= A[j * 6 + k] * A[j * 6 + k];
    if (!(d > 0.0)) { ok = false; d = 1.0; }
    const double l = sqrt(d);
    A[j * 6 + j] = l;
    const double il = 1.0 / l;
#pragma unroll
    for (int i = j + 1; i < 6; i++) {
      double v = A[i * 6 + j];
#pragma unroll
      for (int k = 0; k < j; k++) v -= A[i * 6 + k] * A[j * 6 + k];
      A[i * 6 + j] = v * il;
    }
  }
  // Li = L^-1 (lower)
#pragma unroll
  for (int i = 0; i < 36; i++) Li[i] = 0.0;
#pragma unroll
  for (int c = 0; c < 6; c++) {
    Li[c * 6 + c] = 1.0 / A[c * 6 + c];
#pragma unroll
    for (int i = c + 1; i < 6; i++) {
      double v = 0.0;
#pragma unroll
      for (int k = c; k < i; k++) v -= A[i * 6 + k] * Li[k * 6 + c];
      Li[i * 6 + c] = v / A[i * 6 + i];
    }
  }
  // Minv = Li^T Li
#pragma unroll
  for (int i = 0; i < 6; i++)
#pragma unroll
    for (int j = 0; j < 6; j++) {
      double v = 0.0;
#pragma unroll
      for (int k = 0; k < 6; k++) v += Li[k * 6 + i] * Li[k * 6 + j];
      Minv[(size_t)a * 36 + i * 6 + j] = v;
    }
#pragma unroll
  for (int i = 0; i < 6; i++) bschur[(size_t)a * 6 + i] = bp[(size_t)a * 6 + i] + bneg[(size_t)a * 6 + i];
  if (!ok) atomicExch(fail, 1);
}

// ------------------------------------------------------------------------------------------------------------
// K6+K7 (poses): trial = exp(x) * T ; partial of sum x (lambda x + b) over pose unknowns
__global__ void __launch_bounds__(TPB) k_update_poses(const double* __restrict__ pose, const int* __restrict__ pose_slot,
                                                      const double* __restrict__ x, const double* __restrict__ bp, int K,
                                                      double lambda, double* __restrict__ pose_trial,
                                                      double* __restrict__ scale_partials) {
  __shared__ double red[TPB / 32];
  double acc = 0.0;
  for (int k = blockIdx.x * TPB + threadIdx.x; k < K; k += gridDim.x * TPB) {
    Pose T;
    const double* p = pose + 7 * (size_t)k;
    T.qx = p[0]; T.qy = p[1]; T.qz = p[2]; T.qw = p[3]; T.tx = p[4]; T.ty = p[5]; T.tz = p[6];
    const int s = pose_slot[k];
    if (s >= 0) {
      double u[6];
#pragma unroll
      for (int i = 0; i < 6; i++) {
        u[i] = x[(size_t)s * 6 + i];
        acc += u[i] * (lambda * u[i] + bp[(size_t)s * 6 + i]);
      }
      T = se3_exp_times(u, T);
    }
    double* o = pose_trial + 7 * (size_t)k;
    o[0] = T.qx; o[1] = T.qy; o[2] = T.qz; o[3] = T.qw; o[4] = T.tx; o[5] = T.ty; o[6] = T.tz;
  }
  const double t = block_sum(acc, red);
  if (threadIdx.x == 0) scale_partials[blockIdx.x] = t;
}

// K6+K7 (landmarks): xl = U^-1 (g - sum_o Z_o^T xp), trial point = point + xl, partial of sum xl (lambda xl + bl).
// One CTA per unit of the landmark schedule (grid-stride): one thread per observation forms Z_o^T x_kf(o) from its row, a
// fixed-order sum per landmark follows, and one thread per landmark solves and writes.
//   reads 148 B/obs (Z, o_kf) + 96 B/landmark (Hll, bl, point) ; writes 24 B/landmark (+ 24 with dx_out)
__global__ void __launch_bounds__(LIN_TILE) k_backsub_points(const int* __restrict__ units, int nunits, const int* __restrict__ lm_ptr,
                                                             const int* __restrict__ o_kf, const int* __restrict__ pose_slot,
                                                             const double* __restrict__ Z, const double* __restrict__ Hll,
                                                             const double* __restrict__ bl, const double* __restrict__ x,
                                                             const double* __restrict__ pt, int Pl, double lambda,
                                                             double* __restrict__ pt_trial, double* __restrict__ dx_out,
                                                             double* __restrict__ scale_partials) {
  __shared__ double s_t[LIN_TILE * 3];
  __shared__ double red[LIN_TILE / 32];
  const int t = threadIdx.x;
  double acc = 0.0;
  for (int c = blockIdx.x; c < nunits; c += gridDim.x) {
    const int l0 = units[c], nlm = units[c + 1] - l0;
    const int ob = lm_ptr[l0], oe = lm_ptr[l0 + nlm];
    const int nch = oe - ob > LIN_TILE ? (oe - ob + LIN_TILE - 1) / LIN_TILE : 1;   // > 1: the unit is one landmark (thread 0)
    double tl[3] = {0.0, 0.0, 0.0};
    for (int k = 0; k < nch; k++) {
      const int c0 = ob + k * LIN_TILE, c1 = min(oe, c0 + LIN_TILE);
      double v0 = 0.0, v1 = 0.0, v2 = 0.0;
      if (c0 + t < c1) {
        const int s = __ldg(pose_slot + o_kf[c0 + t]);
        if (s >= 0) {   // the warp's rows are contiguous: every byte of the lines it touches is used
          const double2* z2 = reinterpret_cast<const double2*>(Z + (size_t)(c0 + t) * 18);
          double z[18];
#pragma unroll
          for (int i = 0; i < 9; i++) { const double2 v = z2[i]; z[2 * i] = v.x; z[2 * i + 1] = v.y; }
#pragma unroll
          for (int r = 0; r < 6; r++) {
            const double xr = __ldg(x + (size_t)s * 6 + r);
            v0 += z[r * 3] * xr; v1 += z[r * 3 + 1] * xr; v2 += z[r * 3 + 2] * xr;
          }
        }
      }
      s_t[t * 3] = v0; s_t[t * 3 + 1] = v1; s_t[t * 3 + 2] = v2;
      __syncthreads();
      if (t < nlm) {
        const int l = l0 + t;
        const int b = max(__ldg(lm_ptr + l), c0), e = min(__ldg(lm_ptr + l + 1), c1);
        for (int o = b; o < e; o++) { tl[0] += s_t[(o - c0) * 3]; tl[1] += s_t[(o - c0) * 3 + 1]; tl[2] += s_t[(o - c0) * 3 + 2]; }
        if (k == nch - 1) {
          double d[6], u[6], b3[3], g[3], xl[3];
#pragma unroll
          for (int i = 0; i < 6; i++) d[i] = Hll[(size_t)i * Pl + l];
          d[0] += lambda; d[3] += lambda; d[5] += lambda;
          chol3_upper(d, u);
          b3[0] = bl[l]; b3[1] = bl[(size_t)Pl + l]; b3[2] = bl[2 * (size_t)Pl + l];
          UTinv_times(u, b3, g);
          const double gm[3] = {g[0] - tl[0], g[1] - tl[1], g[2] - tl[2]};
          Uinv_times(u, gm, xl);
#pragma unroll
          for (int cc = 0; cc < 3; cc++) {
            pt_trial[3 * (size_t)l + cc] = pt[3 * (size_t)l + cc] + xl[cc];
            acc += xl[cc] * (lambda * xl[cc] + b3[cc]);
            if (dx_out) dx_out[3 * (size_t)l + cc] = xl[cc];
          }
        }
      }
      __syncthreads();
    }
  }
  const double tt = block_sum(acc, red);
  if (t == 0) scale_partials[blockIdx.x] = tt;
}

// ------------------------------------------------------------------------------------------------------------
// structure building (once per create): covisibility bitmap -> block-CSR pattern -> Schur product lists
__global__ void __launch_bounds__(TPB) k_pattern_bitmap(const int* __restrict__ g_kf, const int* __restrict__ g_lm_of,
                                                        const int* __restrict__ g_lm_ptr, const int* __restrict__ pose_slot,
                                                        long long E, int words, unsigned* __restrict__ bitmap) {
  const long long e = (long long)blockIdx.x * TPB + threadIdx.x;
  if (e >= E) return;
  const int a = pose_slot[g_kf[e]];
  if (a < 0) return;
  const int lm = g_lm_of[e];
  const int beg = g_lm_ptr[lm], end = g_lm_ptr[lm + 1];
  for (int o = beg; o < end; o++) {
    const int b = pose_slot[g_kf[o]];
    if (b < 0) continue;
    unsigned* wp = bitmap + (size_t)a * words + (b >> 5);
    const unsigned bit = 1u << (b & 31);
    if (!(*(volatile unsigned*)wp & bit)) atomicOr(wp, bit);
  }
}

__global__ void __launch_bounds__(TPB) k_set_diag_bits(int Kf, int words, unsigned* __restrict__ bitmap) {
  const int a = blockIdx.x * TPB + threadIdx.x;
  if (a < Kf) atomicOr(bitmap + (size_t)a * words + (a >> 5), 1u << (a & 31));
}

// per row: exclusive popcount prefix per word + row total
__global__ void __launch_bounds__(TPB) k_row_prefix(const unsigned* __restrict__ bitmap, int Kf, int words,
                                                    int* __restrict__ word_prefix, int* __restrict__ row_count) {
  const int a = blockIdx.x * TPB + threadIdx.x;
  if (a >= Kf) return;
  int run = 0;
  for (int w = 0; w < words; w++) {
    word_prefix[(size_t)a * words + w] = run;
    run += __popc(bitmap[(size_t)a * words + w]);
  }
  row_count[a] = run;
}

__global__ void __launch_bounds__(TPB) k_fill_cols(const unsigned* __restrict__ bitmap, const int* __restrict__ word_prefix,
                                                   const int* __restrict__ s_rowptr, int Kf, int words,
                                                   int* __restrict__ s_col, int* __restrict__ s_row) {
  const long long i = (long long)blockIdx.x * TPB + threadIdx.x;
  if (i >= (long long)Kf * words) return;
  const int a = (int)(i / words), w = (int)(i % words);
  unsigned bits = bitmap[i];
  int pos = s_rowptr[a] + word_prefix[i];
  while (bits) {
    const int b = __ffs(bits) - 1;
    bits &= bits - 1;
    s_col[pos] = w * 32 + b;
    s_row[pos] = a;
    pos++;
  }
}

__device__ __forceinline__ int csr_pos(const unsigned* __restrict__ bitmap, const int* __restrict__ word_prefix,
                                       const int* __restrict__ s_rowptr, int words, int a, int b) {
  const size_t wi = (size_t)a * words + (b >> 5);
  return s_rowptr[a] + word_prefix[wi] + __popc(bitmap[wi] & ((1u << (b & 31)) - 1u));
}

// CSR position of the diagonal block of every row and the number of upper blocks (diagonal included) of the row
__global__ void __launch_bounds__(TPB) k_diag_pos(const unsigned* __restrict__ bitmap, const int* __restrict__ word_prefix,
                                                 const int* __restrict__ s_rowptr, int Kf, int words, int* __restrict__ s_diag,
                                                 int* __restrict__ upper_count) {
  const int a = blockIdx.x * TPB + threadIdx.x;
  if (a >= Kf) return;
  const int q = csr_pos(bitmap, word_prefix, s_rowptr, words, a, a);
  s_diag[a] = q;
  upper_count[a] = s_rowptr[a + 1] - q;
}

// Upper-block numbering (row-major over the entries with column >= row: the columns of a row are sorted, so its upper part is
// [s_diag[a], s_rowptr[a+1]) and numbers consecutively from u_rowstart[a]), the (row, column) of every upper block, and for every
// position of the full pattern the upper block that holds it (the transposed one for the lower triangle).
__global__ void __launch_bounds__(TPB) k_upper_index(const int* __restrict__ s_row, const int* __restrict__ s_col, long long nnzb,
                                                    const unsigned* __restrict__ bitmap, const int* __restrict__ word_prefix,
                                                    const int* __restrict__ s_rowptr, int words, const int* __restrict__ s_diag,
                                                    const int* __restrict__ u_rowstart, int* __restrict__ csr_u,
                                                    int* __restrict__ u_row, int* __restrict__ u_col, int* __restrict__ err) {
  const long long q = (long long)blockIdx.x * TPB + threadIdx.x;
  if (q >= nnzb) return;
  const int a = s_row[q], b = s_col[q];
  if (b >= a) {
    const int u = u_rowstart[a] + (int)(q - s_diag[a]);
    csr_u[q] = u; u_row[u] = a; u_col[u] = b;
  } else {
    if (!((bitmap[(size_t)b * words + (a >> 5)] >> (a & 31)) & 1u)) { atomicOr(err, 1); return; }  // pattern must be symmetric
    const int qb = csr_pos(bitmap, word_prefix, s_rowptr, words, b, a);
    csr_u[q] = u_rowstart[b] + (qb - s_diag[b]);
  }
}

// out[i] = in[i] - off  (local landmark ids / local observation offsets of a shard)
__global__ void __launch_bounds__(TPB) k_shift(const int* __restrict__ in, long long n, int off, int* __restrict__ out) {
  const long long i = (long long)blockIdx.x * TPB + threadIdx.x;
  if (i < n) out[i] = in[i] - off;
}

// Cuts the landmark schedule of k_linearize / k_backsub_points: units[r - 1] = i for every head i (head flags from k_lin_heads,
// rank = their inclusive scan), units[n] = n.
__global__ void __launch_bounds__(TPB) k_unit_ptr(const int* __restrict__ head, const int* __restrict__ rank, int n,
                                                  int* __restrict__ units) {
  const int i = blockIdx.x * TPB + threadIdx.x;
  if (i >= n) return;
  if (head[i]) units[rank[i] - 1] = i;
  if (i == n - 1) units[rank[i]] = n;
}

// Row key of every local observation for the stable grouping by block row: its pose slot, Kf for a fixed pose (sorted past the rows)
__global__ void __launch_bounds__(TPB) k_row_keys(const int* __restrict__ o_kf, const int* __restrict__ pose_slot, int E, int Kf,
                                                  int* __restrict__ key, int* __restrict__ idx) {
  const int e = blockIdx.x * TPB + threadIdx.x;
  if (e >= E) return;
  const int a = pose_slot[o_kf[e]];
  key[e] = a < 0 ? Kf : a;
  idx[e] = e;
}

// Count (fill == 0) or fill (fill == 1) the product lists of the upper blocks of block row a, one warp per row.  The warp walks
// row a's observations e in increasing order (landmark order: row_obs is a stable grouping of the observations by row), with the
// lanes over the observations o of e's landmark; every pair (e, o) with row(o) > a, and (e, e), goes to block (a, row(o)) at that
// block's cursor.  Only this warp touches row a's cursors, so they need no atomics, and every list comes out in increasing (e, o)
// order: deterministic by construction.  Lanes that hit the same block in one step (a keyframe observing a landmark twice) take
// consecutive slots in lane order.  A row of at most ROWP_CUR upper blocks keeps its cursors in shared memory, a longer one in
// cursor[] (zero before each pass); the count pass leaves every block's count in cursor[], the fill writes at u_prod_ptr[u] + slot.
constexpr int ROWP_CUR = 512;
__global__ void __launch_bounds__(128) k_row_products(const int* __restrict__ row_obs, const int* __restrict__ row_obs_ptr, int Kf,
                                                      const int* __restrict__ o_kf, const int* __restrict__ o_lm,
                                                      const int* __restrict__ lm_ptr, const int* __restrict__ pose_slot,
                                                      const unsigned* __restrict__ bitmap, const int* __restrict__ word_prefix,
                                                      const int* __restrict__ s_rowptr, const int* __restrict__ s_diag,
                                                      const int* __restrict__ u_diag, int nub, int words, int fill, unsigned* cursor,
                                                      const unsigned* __restrict__ u_prod_ptr, uint2* __restrict__ prod) {
  __shared__ unsigned s_cur[4][ROWP_CUR];
  const int a = (int)(((long long)blockIdx.x * 128 + threadIdx.x) >> 5);
  if (a >= Kf) return;  // warp-uniform
  const int lane = threadIdx.x & 31;
  const unsigned below = (1u << lane) - 1u;
  const int ua = u_diag[a], nu = (a + 1 < Kf ? u_diag[a + 1] : nub) - ua;
  const bool sh = nu <= ROWP_CUR;
  unsigned* cur = sh ? s_cur[threadIdx.x >> 5] : cursor + ua;   // cursor of upper block ua + i: cur[i]
  if (sh)
    for (int i = lane; i < nu; i += 32) cur[i] = 0u;
  __syncwarp();
  const int q0 = s_diag[a];   // CSR position of block ua
  const int rb = row_obs_ptr[a], re = row_obs_ptr[a + 1];
  for (int c0 = rb; c0 < re; c0 += 32) {
    // 32 observations of the row, their landmarks' observation ranges loaded together, then walked one by one
    int ce = 0, cb = 0, cn = 0;
    if (c0 + lane < re) {
      ce = row_obs[c0 + lane];
      const int lm = o_lm[ce];
      cb = lm_ptr[lm]; cn = lm_ptr[lm + 1];
    }
    const int nc = min(32, re - c0);
    for (int j = 0; j < nc; j++) {
      const int e = __shfl_sync(0xffffffffu, ce, j), beg = __shfl_sync(0xffffffffu, cb, j), end = __shfl_sync(0xffffffffu, cn, j);
      for (int o0 = beg; o0 < end; o0 += 32) {
        const int o = o0 + lane;
        int i = -1;
        if (o < end) {
          const int b = pose_slot[o_kf[o]];
          if (b > a || o == e) i = csr_pos(bitmap, word_prefix, s_rowptr, words, a, b) - q0;
        }
        const unsigned grp = __match_any_sync(0xffffffffu, i);
        unsigned base = 0;
        if (i >= 0) {
          base = cur[i];
          if (fill) prod[u_prod_ptr[ua + i] + base + __popc(grp & below)] = make_uint2((unsigned)e, (unsigned)o);
        }
        __syncwarp();   // every lane of a group has read the cursor before its first lane moves it
        if (i >= 0 && (grp & below) == 0u) cur[i] = base + __popc(grp);
        __syncwarp();   // and the new value is visible to the next step's reads
      }
    }
  }
  if (sh && !fill)
    for (int i = lane; i < nu; i += 32) cursor[ua + i] = cur[i];
}

// validation of the caller's observation arrays: flags[0] |= out-of-range / negative weight, flags[1] |= not grouped by landmark
__global__ void __launch_bounds__(TPB) k_check_obs(const int* __restrict__ kf, const int* __restrict__ mp,
                                                  const float* __restrict__ w, int E, int K, int P, int* __restrict__ flags) {
  int bad = 0, unsorted = 0;
  for (long long e = (long long)blockIdx.x * TPB + threadIdx.x; e < E; e += (long long)gridDim.x * TPB) {
    const int k = kf[e], m = mp[e];
    if (k < 0 || k >= K || m < 0 || m >= P || (w != nullptr && !(w[e] >= 0.0f))) bad = 1;
    if (e > 0 && mp[e - 1] > m) unsorted = 1;
  }
  if (bad) atomicOr(flags, 1);
  if (unsorted) atomicOr(flags + 1, 1);
}

// lm_ptr[l] = first observation of landmark l in the landmark-sorted observation list (lower bound), lm_ptr[P] = E
__global__ void __launch_bounds__(TPB) k_lm_ptr(const int* __restrict__ mp, int E, int P, int* __restrict__ lm_ptr) {
  const int l = blockIdx.x * TPB + threadIdx.x;
  if (l > P) return;
  int lo = 0, hi = E;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (mp[mid] < l) lo = mid + 1; else hi = mid;
  }
  lm_ptr[l] = lo;
}

__global__ void __launch_bounds__(TPB) k_apply_flags(const float* __restrict__ w_raw, const uint8_t* __restrict__ flags,
                                                     int E, float* __restrict__ o_w) {
  const long long e = (long long)blockIdx.x * TPB + threadIdx.x;
  if (e >= E) return;
  const uint8_t f = flags ? flags[e] : 0;
  float w = (f & 1) ? 0.0f : w_raw[e];
  if (f & 2) w = -w;  // -0.0f keeps the sign bit: inactive + no kernel
  o_w[e] = w;
}

}  // namespace ba
}  // namespace ccm

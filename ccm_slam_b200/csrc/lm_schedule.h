// lm_schedule.h — the Levenberg-Marquardt schedule of g2o's OptimizationAlgorithmLevenberg::solve with SparseOptimizer::optimize's
// stop rules (G/core/optimization_algorithm_levenberg.cpp:61-164, G/core/sparse_optimizer.cpp:354-419), host only, for the LM
// loops of global BA (ba_solver.cu) and the essential graph (pgo.cu).  The caller linearises, solves and evaluates each trial and
// keeps the estimate's buffers.  Every expression keeps the reference's order of evaluation: decisions and trace stay bit-identical.
#pragma once
#include <algorithm>
#include <cmath>
#include <limits>

#include "../../include/ccm_b200.h"

namespace ccm {

struct LmSchedule {
  int max_trials;                // trials per iteration; all of them rejected ends the optimisation
  double lambda = -1, ni = 2;
  int nBad = 0;                  // consecutive iterations that reduced chi2 by less than 1e-3 relative
  // the iteration in progress; lambda_used and the PCG's iterations / relative residual are the last trial's
  double iniChi = 0, currentChi = 0, rho = 0, lambda_used = 0, pcg_relres = 0;
  int qmax = 0, pcg_iters = 0;   // qmax: trials so far

  // first iteration: lambda_init when given, else 1e-5 of the largest diagonal entry of H
  void start(double lambda_init, double maxdiag) {
    lambda = lambda_init > 0 ? lambda_init : 1e-5 * maxdiag;
    ni = 2; nBad = 0;
  }

  void begin_iteration(double chi2) { iniChi = currentChi = chi2; rho = 0; qmax = 0; }

  // One trial at `lambda`: tempChi is the trial state's chi2, scale = sum x (lambda x + b) of its step; a failed linear solve
  // (solved == false) counts as chi2 = DBL_MAX.  True: the trial is accepted and the caller makes the trial state the estimate.
  bool trial(double tempChi, double scale, bool solved, int pcg_iters_, double pcg_relres_) {
    lambda_used = lambda; pcg_iters = pcg_iters_; pcg_relres = pcg_relres_;
    qmax++;
    if (!solved) tempChi = std::numeric_limits<double>::max();
    rho = currentChi - tempChi;
    scale += 1e-3;
    rho /= scale;
    if (rho > 0 && std::isfinite(tempChi)) {
      double alpha = 1. - std::pow((2 * rho - 1), 3);
      alpha = std::min(alpha, 2. / 3.);
      lambda *= std::max(1. / 3., alpha);
      ni = 2;
      currentChi = tempChi;
      return true;
    }
    lambda *= ni;
    ni *= 2;
    return false;
  }

  // another trial at the larger lambda: the last one was rejected and trials are left
  bool retry() const { return rho < 0 && qmax < max_trials; }

  // End of iteration `it`: its trace row (CCM_TRACE_COLS, while the caller's trace has room) and the final chi2 / lambda so far.
  // True: the optimisation stops (every trial rejected, a gain ratio of exactly 0, or the third iteration in a row of low gain).
  template <class Result>
  bool end_iteration(Result* r, int it) {
    if (r->trace && r->trace_len < r->trace_cap) {
      double* tr = r->trace + (size_t)r->trace_len * CCM_TRACE_COLS;
      tr[0] = it; tr[1] = lambda_used; tr[2] = currentChi; tr[3] = rho; tr[4] = qmax; tr[5] = lambda; tr[6] = pcg_iters; tr[7] = pcg_relres;
      r->trace_len++;
    }
    r->chi2_final = currentChi; r->lambda_final = lambda;
    if (qmax == max_trials || rho == 0) return true;
    if ((iniChi - currentChi) * 1e3 < iniChi) nBad++; else nBad = 0;
    return nBad >= 3;
  }
};

}  // namespace ccm

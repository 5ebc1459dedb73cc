// search_and_fuse_oracle.cpp — flat CPU oracle for the searches of LoopFinder / MapMerger::SearchAndFuse (TEST INFRASTRUCTURE, NOT
// PRODUCT).
//
// Every (corrected keyframe, loop point) pair over the state at the start of the member: the prelude of
// ORBmatcher::Fuse(pKF, Scw, vpPoints, th, vpReplacePoint) (S/ORBmatcher.cpp:1017-1069) written out as the reference writes it, in plain
// C++ float / double arithmetic (this file is compiled with -ffp-contract=off), with PredictScale's log(float) as std::log(float), i.e.
// the host's logf; then the reference-pinned window search of liboracle.so (orc_fuse_search, proj_oracle.cpp) over all points of one
// keyframe at once, without the chi-square gate.  The camera is the caller's split of Scw (ccm_fuse_kf::Tcw / Ow).  Nothing here comes
// from the product.  th and chi2 exist so that tests can build the wrong variants a fixture must reject (th = 3, the gate of
// Fuse(kf, points) switched on); SearchAndFuse itself is th = 4, chi2 = 0.
#include <cmath>
#include <cstdint>
#include <vector>

#include "ccm_b200.h"

extern "C" {
struct orc_grid;     // layout of ccm_feature_grid (proj_oracle.cpp)
struct orc_queries;  // layout of ccm_proj_queries
int orc_fuse_search(const orc_grid* g, const orc_queries* q, const float* inv_level_sigma2, int32_t* best_idx);
}

namespace {

struct Queries {
  std::vector<uint8_t> valid, desc;
  std::vector<float> uv, radius, angle;
  std::vector<int32_t> level;
  explicit Queries(size_t m) : valid(m, 0), desc(32 * m, 0), uv(2 * m, 0.f), radius(m, 0.f), angle(m, 0.f), level(m, 0) {}
};

// MapPoint::PredictScale(currentDist, pKF) (S/MapPoint.cpp:837-852)
int PredictScale(float mfMaxDistance, const float& currentDist, const ccm_fuse_kf* pKF) {
  float ratio;
  ratio = mfMaxDistance / currentDist;
  int nScale = std::ceil(std::log(ratio) / pKF->log_scale_factor);
  if (nScale < 0)
    nScale = 0;
  else if (nScale >= pKF->nlevels)
    nScale = pKF->nlevels - 1;
  return nScale;
}

// Fuse(Scw)'s prelude for point `row` into keyframe pKF; fills query i when every gate passes
void prelude(const ccm_fuse_kf* pKF, const ccm_fuse_points* pts, int row, float th, Queries& q, size_t i) {
  if (pts->skip[row]) return;   // pMP->isBad(); spAlreadyFound is the caller's, mbDoNotReplace is commented out (:1026-1027)
  const float* Tcw = pKF->Tcw;
  const float* p3Dw = pts->pos + 3 * (size_t)row;
  float p3Dc[3];
  for (int r = 0; r < 3; r++) p3Dc[r] = Tcw[4 * r] * p3Dw[0] + Tcw[4 * r + 1] * p3Dw[1] + Tcw[4 * r + 2] * p3Dw[2] + Tcw[4 * r + 3];
  if (p3Dc[2] < 0.0f) return;
  const float invz = 1.0 / p3Dc[2];
  const float x = p3Dc[0] * invz;
  const float y = p3Dc[1] * invz;
  const float u = pKF->fx * x + pKF->cx;
  const float v = pKF->fy * y + pKF->cy;
  const ccm_feature_grid& g = pKF->grid;
  if (!(u >= g.min_x && u < g.max_x && v >= g.min_y && v < g.max_y)) return;   // KeyFrame::IsInImage
  const float maxDistance = 1.2f * pts->max_distance[row];                     // GetMaxDistanceInvariance
  const float minDistance = 0.8f * pts->min_distance[row];                     // GetMinDistanceInvariance
  const float PO[3] = {p3Dw[0] - pKF->Ow[0], p3Dw[1] - pKF->Ow[1], p3Dw[2] - pKF->Ow[2]};
  const float dist3D = (float)std::sqrt((double)PO[0] * PO[0] + (double)PO[1] * PO[1] + (double)PO[2] * PO[2]);   // cv::norm
  if (dist3D < minDistance || dist3D > maxDistance) return;
  const float* Pn = pts->normal + 3 * (size_t)row;
  const double dot = (double)PO[0] * Pn[0] + (double)PO[1] * Pn[1] + (double)PO[2] * Pn[2];                     // Mat::dot
  if (dot < 0.5 * dist3D) return;
  const int nPredictedLevel = PredictScale(pts->max_distance[row], dist3D, pKF);
  q.valid[i] = 1;
  q.uv[2 * i] = u; q.uv[2 * i + 1] = v;
  q.radius[i] = th * pKF->scale_factors[nPredictedLevel];
  q.level[i] = nPredictedLevel;
  for (int b = 0; b < 32; b++) q.desc[32 * i + b] = pts->desc[32 * (size_t)row + b];
}

}  // namespace

// the contract of ccm_search_and_fuse on valid input (th = 4, chi2 = 0)
extern "C" void orc_search_and_fuse(const ccm_fuse_kf* kfs, int32_t n_kf, const ccm_fuse_points* pts, float th, int32_t chi2, int32_t* best) {
  const int m = pts->n;
  for (int k = 0; k < n_kf; k++) {
    Queries q((size_t)m);
    for (int i = 0; i < m; i++) prelude(&kfs[k], pts, i, th, q, (size_t)i);
    const ccm_proj_queries cq{m, q.valid.data(), q.uv.data(), q.radius.data(), q.level.data(), q.desc.data(), q.angle.data()};
    orc_fuse_search(reinterpret_cast<const orc_grid*>(&kfs[k].grid), reinterpret_cast<const orc_queries*>(&cq),
                    chi2 ? kfs[k].inv_level_sigma2 : nullptr, best + (size_t)k * m);
  }
}

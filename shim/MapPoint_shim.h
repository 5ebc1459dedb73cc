// MapPoint_shim.h — the batch entry of shim/MapPoint_shim.cpp, for the write-back loops of shim/Optimizer_shim.cpp.
#ifndef CCM_MAPPOINT_SHIM_H
#define CCM_MAPPOINT_SHIM_H
#include <vector>

#include <boost/shared_ptr.hpp>

namespace cslam {

class MapPoint;

// Computes mNormalVector / mfMinDistance / mfMaxDistance of every point in one ccm_normal_depth call and parks the results, per
// thread, for the MapPoint::UpdateNormalAndDepth() calls that follow.  new_pos [n][3]: the positions SetWorldPos will give the
// points before that call (nullptr: their current positions).  A parked value is used only while the point's position, observation
// count and reference keyframe still match; the member computes on the host otherwise.
void ccm_b200_prepare_normals(const std::vector<boost::shared_ptr<MapPoint> >& points, const float* new_pos);
// Drops every value parked on this thread.
void ccm_b200_clear_normals();
// Counts of MapPoint::UpdateNormalAndDepth() calls since the process started, by how they ended: a parked value written, a parked
// value found stale (then computed on the host), computed on the host.  A write-back loop after ccm_b200_prepare_normals should show
// one hit per point it wrote and nothing else.
void ccm_b200_normals_stats(unsigned long long* hits, unsigned long long* stale, unsigned long long* host);

// Clears the parked values when a write-back ends, by any path.
struct ParkedNormalsGuard {
  ParkedNormalsGuard() {}
  ~ParkedNormalsGuard() { ccm_b200_clear_normals(); }
  ParkedNormalsGuard(const ParkedNormalsGuard&) = delete;
  ParkedNormalsGuard& operator=(const ParkedNormalsGuard&) = delete;
};

}  // namespace cslam
#endif

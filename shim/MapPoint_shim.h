// MapPoint_shim.h — the batch entry of shim/MapPoint_shim.cpp, for the write-back loops of shim/Optimizer_shim.cpp.
#ifndef CCM_MAPPOINT_SHIM_H
#define CCM_MAPPOINT_SHIM_H
#include <stdint.h>

#include <vector>

#include <boost/shared_ptr.hpp>

namespace cslam {

class MapPoint;

// Computes mNormalVector / mfMinDistance / mfMaxDistance of every point in one ccm_normal_depth call and parks the results, per
// thread, for the MapPoint::UpdateNormalAndDepth() calls that follow.  new_pos [n][3]: the positions SetWorldPos will give the
// points before that call (nullptr: their current positions).  A parked value is used only while the point's position, observation
// count and reference keyframe still match; the member computes on the host otherwise.
void ccm_b200_prepare_normals(const std::vector<boost::shared_ptr<MapPoint> >& points, const float* new_pos);
// Parks values computed elsewhere for the MapPoint::UpdateNormalAndDepth() calls that follow, under the same snapshot rule: point i
// (status[i] != 0) gets normal [i][3], max_dist[i], min_dist[i], used while its position is pos[i][3] and its observation count and
// reference keyframe are what they are now.  ccm_b200_prepare_normals parks its own results through the same table.
void ccm_b200_park_normals(const std::vector<boost::shared_ptr<MapPoint> >& points, const float* pos, const float* normal,
                           const float* max_dist, const float* min_dist, const uint8_t* status);
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

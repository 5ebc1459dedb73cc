// MapPointDescriptor_shim.h — the batch entry of shim/MapPointDescriptor_shim.cpp, for the loops that call
// MapPoint::ComputeDistinctiveDescriptors on many points (INTEGRATION.md §4d).
#ifndef CCM_MAPPOINT_DESCRIPTOR_SHIM_H
#define CCM_MAPPOINT_DESCRIPTOR_SHIM_H
#include <vector>

#include <boost/shared_ptr.hpp>

#include "ccm_b200.h"

namespace cslam {

class MapPoint;

// Chooses mDescriptor of every point in one ccm_distinctive_descriptors call (ccm_kfstore_distinctive_descriptors when a store is
// registered) and parks the choice, per thread, for the MapPoint::ComputeDistinctiveDescriptors() calls that follow.  A parked choice
// is used only while the point's observation list is element for element the one it was computed from; the member computes on the
// host otherwise.
void ccm_b200_prepare_descriptors(const std::vector<boost::shared_ptr<MapPoint> >& points);
// ccm_b200_prepare_normals(points, nullptr) and ccm_b200_prepare_descriptors(points), for the sites that call both members on each
// point.  Needs shim/MapPoint_shim.cpp in the same link.
void ccm_b200_prepare_point_updates(const std::vector<boost::shared_ptr<MapPoint> >& points);
// Drops every choice parked on this thread.
void ccm_b200_clear_descriptors();
// The keyframe store that holds every keyframe's descriptors under its mUniqueId (nullptr: none; the rows go with the call).  Process-wide.
void ccm_b200_register_kfstore(ccm_kf_store* store);
// Counts of MapPoint::ComputeDistinctiveDescriptors() calls since the process started, by how they ended: a parked choice written, a
// parked choice found stale (then computed on the host), computed on the host.  A loop after ccm_b200_prepare_descriptors should show
// one hit per point it wrote and nothing else.
void ccm_b200_descriptors_stats(unsigned long long* hits, unsigned long long* stale, unsigned long long* host);

// Clears the parked choices when a loop ends, by any path.
struct ParkedDescriptorsGuard {
  ParkedDescriptorsGuard() {}
  ~ParkedDescriptorsGuard() { ccm_b200_clear_descriptors(); }
  ParkedDescriptorsGuard(const ParkedDescriptorsGuard&) = delete;
  ParkedDescriptorsGuard& operator=(const ParkedDescriptorsGuard&) = delete;
};

}  // namespace cslam
#endif

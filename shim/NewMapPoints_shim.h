// NewMapPoints_shim.h — what shim/NewMapPoints_shim.cpp offers besides the member it defines, LocalMapping::CreateNewMapPoints
// (INTEGRATION.md §4f).
#ifndef CCM_NEW_MAP_POINTS_SHIM_H
#define CCM_NEW_MAP_POINTS_SHIM_H

namespace cslam {

// Counts since the process started: library calls made by LocalMapping::CreateNewMapPoints, points it created, and points the
// library returned that were dropped because CheckNewKeyFrames() ended the member early.
void ccm_b200_new_map_points_stats(unsigned long long* calls, unsigned long long* created, unsigned long long* dropped);

}  // namespace cslam
#endif

// FuseNeighbours_shim.h — what shim/FuseNeighbours_shim.cpp offers besides the member it defines, LocalMapping::SearchInNeighbors
// (INTEGRATION.md §4g).
#ifndef CCM_FUSE_NEIGHBOURS_SHIM_H
#define CCM_FUSE_NEIGHBOURS_SHIM_H

namespace cslam {

// Counts since the process started: library calls made by LocalMapping::SearchInNeighbors, and pairs searched again on the host
// because the point's descriptor had changed since the call (or the point was not in the uploaded set).
void ccm_b200_fuse_neighbours_stats(unsigned long long* calls, unsigned long long* repairs);

}  // namespace cslam
#endif

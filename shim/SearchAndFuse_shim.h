// SearchAndFuse_shim.h — the drop-in for LoopFinder::SearchAndFuse (cslam/src/LoopFinder.cpp:709-734) and MapMerger::SearchAndFuse
// (cslam/src/MapMerger.cpp:574-598), INTEGRATION.md §4i.
#ifndef CCM_SEARCH_AND_FUSE_SHIM_H
#define CCM_SEARCH_AND_FUSE_SHIM_H
#include <vector>

#include <boost/shared_ptr.hpp>

#include "Sim3Correction_shim.h"   // Sim3CorrectionMap: the KeyFrameAndPose of LoopFinder.h / MapMerger.h

namespace cslam {

class MapPoint;

// The member body: for each keyframe of CorrectedPosesMap in map order, Fuse(pKF, Scw, vpLoopMapPoints, 4, vpReplacePoints) and then
// the replacements, with the searches of every keyframe made by one ccm_search_and_fuse call.  merge = false: LoopFinder's
// pRep->Replace(vpLoopMapPoints[i], true); merge = true: MapMerger's pRep->ReplaceAndLock(vpLoopMapPoints[i]).
void ccm_b200_search_and_fuse(const Sim3CorrectionMap& CorrectedPosesMap, const std::vector<boost::shared_ptr<MapPoint> >& vpLoopMapPoints,
                              bool merge);
// Counts since the process started: library calls, and points searched again on the host because their descriptor had changed.
void ccm_b200_search_and_fuse_stats(unsigned long long* calls, unsigned long long* repairs);

}  // namespace cslam
#endif

// Sim3Correction_shim.h — the drop-in for the Sim3 correction pass of LoopFinder::CorrectLoop (cslam/src/LoopFinder.cpp:568-613) and
// MapMerger::MergeMaps (cslam/src/MapMerger.cpp:349-395), INTEGRATION.md §4h.
#ifndef CCM_SIM3_CORRECTION_SHIM_H
#define CCM_SIM3_CORRECTION_SHIM_H
#include <map>
#include <set>
#include <utility>

#include <Eigen/StdVector>
#include <boost/shared_ptr.hpp>

#include "thirdparty/g2o/g2o/types/sim3.h"

namespace cslam {

class KeyFrame;

// the KeyFrameAndPose of LoopFinder.h:80-81 and MapMerger.h:80-81 (the same type in both classes)
typedef std::map<boost::shared_ptr<KeyFrame>, g2o::Sim3, std::less<boost::shared_ptr<KeyFrame> >,
                 Eigen::aligned_allocator<std::pair<const boost::shared_ptr<KeyFrame>, g2o::Sim3> > >
    Sim3CorrectionMap;

// Runs the whole pass over `corrected` in its map order with one ccm_sim3_correction call, then applies the results in the reference's
// order: each moved point's SetWorldPos, tag (mCorrectedByKF_LC / _MM = pCurKF->mId), mCorrectedReference_* = pCurKF->mUniqueId and
// UpdateNormalAndDepth() (its value parked, shim/MapPoint_shim.cpp); then each keyframe's SetPose([R t/s]), UpdateConnections() (its
// counter prepared by ccm_b200_prepare_connections) and, for a merge, mCorrected_MM = pCurKF->mId, or else changed->insert(mId).
// noncorrected[pKFi] as the reference reads it (a missing key reads the identity Sim3).  merge: MergeMaps' tags and bookkeeping;
// otherwise CorrectLoop's.  Each slot is checked live (null, isBad(), tag) before it is applied; a point whose live state disagrees
// with what was flattened is corrected on the host, as the reference does it, and counted as a fallback.
void ccm_b200_correct_sim3(const Sim3CorrectionMap& corrected, const Sim3CorrectionMap& noncorrected, boost::shared_ptr<KeyFrame> pCurKF,
                           bool merge, std::set<std::pair<size_t, size_t> >* changed);
// Counts since the process started: calls, points moved with the device's values, points corrected on the host instead.
void ccm_b200_sim3_correction_stats(unsigned long long* calls, unsigned long long* moved, unsigned long long* fallbacks);

}  // namespace cslam
#endif

// Stand-in for cslam::MapPoint as shim/KeyFrameCulling_shim.cpp sees it (TEST INFRASTRUCTURE): what LocalMapping::KeyFrameCullingV3
// reads and what KeyFrame::SetBadFlag reaches, with the reference's names and access (line numbers refer to
// cslam/include/cslam/MapPoint.h).  EraseObservation and SetBadFlag are restated for the server in oracle/ref_keyframe_culling_wrap.cpp;
// SetBadFlag's map bookkeeping after the observers' slots are nulled is not stood in for.  mObservations is ordered by keyframe mId.
#ifndef CCM_REF_STUB_KC_CSLAM_MAPPOINT_H
#define CCM_REF_STUB_KC_CSLAM_MAPPOINT_H
#include <map>
#include <mutex>

#include <cslam/KeyFrame.h>

namespace cslam {

class MapPoint : public boost::enable_shared_from_this<MapPoint> {   // MapPoint.h:78
 public:
  typedef boost::shared_ptr<KeyFrame> kfptr;
  typedef boost::shared_ptr<MapPoint> mpptr;
  kfptr GetReferenceKeyFrame() { std::unique_lock<std::mutex> lock(mMutexFeatures); return mpRefKF; }             // MapPoint.h:138
  std::map<kfptr, size_t, KfById> GetObservations() { std::unique_lock<std::mutex> lock(mMutexFeatures); return mObservations; }   // MapPoint.h:141
  int Observations() { std::unique_lock<std::mutex> lock(mMutexFeatures); return nObs; }                          // MapPoint.h:142
  void EraseObservation(kfptr pKF, bool bLock = false, bool bSuppressMapAction = false);                          // MapPoint.h:145
  void SetBadFlag(bool bSuppressMapAction = false);                                                              // MapPoint.h:151
  bool isBad() { std::unique_lock<std::mutex> lock(mMutexFeatures); return mbBad; }                              // MapPoint.h:152

  int nObs = 0;                                  // MapPoint.h:221

 protected:
  friend struct KcScene;
  std::map<kfptr, size_t, KfById> mObservations; // MapPoint.h:281
  kfptr mpRefKF;                                 // MapPoint.h:292
  bool mbBad = false;                            // MapPoint.h:299
  std::mutex mMutexFeatures;
};

}  // namespace cslam
#endif

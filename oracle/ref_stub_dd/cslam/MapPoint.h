// Stand-ins for cslam::MapPoint / KeyFrame as shim/MapPointDescriptor_shim.cpp and shim/MapPoint_shim.cpp see them together
// (TEST INFRASTRUCTURE).
//
// The same classes as oracle/ref_stub_mp (whose MapPoint.h explains why the real header is not used), plus what
// MapPoint::ComputeDistinctiveDescriptors and its batch preparation touch: KeyFrame::mDescriptors and mUniqueId, MapPoint::mDescriptor
// and GetDescriptor, and AddObservation with the reference's first-index-wins rule.  Both members are declared without a body: the two
// shims define them.  Line numbers refer to the real headers (MapPoint.cpp for the two bodies restated here).
#ifndef CCM_REF_STUB_DD_CSLAM_H
#define CCM_REF_STUB_DD_CSLAM_H
#include <boost/shared_ptr.hpp>
#include <map>
#include <mutex>
#include <vector>

#include <opencv2/core/core.hpp>

namespace cslam {

class KeyFrame;
class MapPoint;
struct NormalDepthProbe;

class KeyFrame {
 public:
  typedef boost::shared_ptr<KeyFrame> kfptr;
  cv::Mat GetCameraCenter() { std::unique_lock<std::mutex> lock(mMutexPose); return Ow.clone(); }   // KeyFrame.h:137
  bool isBad() { std::unique_lock<std::mutex> lock(mMutexConnections); return mbBad; }               // KeyFrame.h:194
  size_t mUniqueId = 0;                                                                              // KeyFrame.h:283 (const there)
  std::vector<cv::KeyPoint> mvKeysUn;                                                                // KeyFrame.h:326 (const there)
  cv::Mat mDescriptors;                                                                              // KeyFrame.h:327 (const there)
  int mnScaleLevels = 8;                                                                             // KeyFrame.h:337 (const there)
  std::vector<float> mvScaleFactors;                                                                 // KeyFrame.h:340 (const there)
  // storage
  cv::Mat Ow;                                                                                        // KeyFrame.h:383
  bool mbBad = false;                                                                                // KeyFrame.h:411
  std::mutex mMutexPose, mMutexConnections;                                                          // KeyFrame.h:417-418
};

class MapPoint {
 public:
  typedef boost::shared_ptr<KeyFrame> kfptr;
  typedef boost::shared_ptr<MapPoint> mpptr;
  // MapPoint.h:132-171
  void SetWorldPos(const cv::Mat& Pos, bool bLock, bool bIgnorePosMutex = false) {
    (void)bLock; (void)bIgnorePosMutex;
    std::unique_lock<std::mutex> lock(mMutexPos);
    Pos.copyTo(mWorldPos);
  }
  cv::Mat GetWorldPos() { std::unique_lock<std::mutex> lock(mMutexPos); return mWorldPos.clone(); }
  kfptr GetReferenceKeyFrame() { std::unique_lock<std::mutex> lock(mMutexFeatures); return mpRefKF; }
  std::map<kfptr, size_t> GetObservations() { std::unique_lock<std::mutex> lock(mMutexFeatures); return mObservations; }
  // MapPoint.h:144; the body's server-side part (MapPoint.cpp:417-428): a keyframe already observing the point keeps its index
  void AddObservation(kfptr pKF, size_t idx) {
    std::unique_lock<std::mutex> lock(mMutexFeatures);
    if (mObservations.count(pKF)) return;
    mObservations[pKF] = idx;
  }
  bool isBad() { std::unique_lock<std::mutex> lock(mMutexFeatures); std::unique_lock<std::mutex> lock2(mMutexPos); return mbBad; }   // MapPoint.h:152
  void ComputeDistinctiveDescriptors();                                                                                           // MapPoint.h:167
  cv::Mat GetDescriptor() { std::unique_lock<std::mutex> lock(mMutexFeatures); return mDescriptor.clone(); }                      // MapPoint.h:169
  void UpdateNormalAndDepth();                                                                                                    // MapPoint.h:171
  // scene construction and change (the reference goes through AddObservation / EraseObservation / SetBadFlag)
  void AddObservationForTest(kfptr pKF, size_t idx) { mObservations[pKF] = idx; }
  void EraseObservationForTest(kfptr pKF) { mObservations.erase(pKF); }
  void SetReferenceForTest(kfptr pKF) { mpRefKF = pKF; }
  void SetBadForTest(bool b) { mbBad = b; }

 protected:
  friend struct NormalDepthProbe;
  cv::Mat mWorldPos;                          // MapPoint.h:274
  std::map<kfptr, size_t> mObservations;      // MapPoint.h:281
  cv::Mat mNormalVector;                      // MapPoint.h:286
  cv::Mat mDescriptor;                        // MapPoint.h:289
  kfptr mpRefKF;                              // MapPoint.h:292
  bool mbBad = false;                         // MapPoint.h:299
  float mfMinDistance = 0.f;                  // MapPoint.h:304
  float mfMaxDistance = 0.f;                  // MapPoint.h:305
  std::mutex mMutexPos;                       // MapPoint.h:309
  std::mutex mMutexFeatures;                  // MapPoint.h:310
};

}  // namespace cslam
#endif

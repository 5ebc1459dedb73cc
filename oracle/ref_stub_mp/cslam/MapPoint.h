// Stand-ins for cslam::MapPoint / KeyFrame as shim/MapPoint_shim.cpp sees them (TEST INFRASTRUCTURE).
//
// The real cslam/include/cslam/MapPoint.h pulls in ROS messages, cereal, the communicator and the map; these classes carry exactly what
// MapPoint::UpdateNormalAndDepth and its batch preparation touch, with the reference's names and types (line numbers refer to the real
// headers).  MapPoint declares UpdateNormalAndDepth without defining it: the shim defines it.  The members it writes are protected, as
// in the reference; the test wrapper (oracle/ref_normal_depth_wrap.cpp) reads them through the friend NormalDepthProbe.
#ifndef CCM_REF_STUB_MP_CSLAM_H
#define CCM_REF_STUB_MP_CSLAM_H
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
  std::vector<cv::KeyPoint> mvKeysUn;                                                                // KeyFrame.h:326 (const there)
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
  bool isBad() { std::unique_lock<std::mutex> lock(mMutexFeatures); std::unique_lock<std::mutex> lock2(mMutexPos); return mbBad; }   // MapPoint.h:152
  void UpdateNormalAndDepth();                                                                                                    // MapPoint.h:171
  // scene construction (the reference sets these through AddObservation / the constructor)
  void AddObservationForTest(kfptr pKF, size_t idx) { mObservations[pKF] = idx; }
  void SetReferenceForTest(kfptr pKF) { mpRefKF = pKF; }
  void SetBadForTest(bool b) { mbBad = b; }

 protected:
  friend struct NormalDepthProbe;
  cv::Mat mWorldPos;                          // MapPoint.h:274
  std::map<kfptr, size_t> mObservations;      // MapPoint.h:281
  cv::Mat mNormalVector;                      // MapPoint.h:286
  kfptr mpRefKF;                              // MapPoint.h:292
  bool mbBad = false;                         // MapPoint.h:299
  float mfMinDistance = 0.f;                  // MapPoint.h:304
  float mfMaxDistance = 0.f;                  // MapPoint.h:305
  std::mutex mMutexPos;                       // MapPoint.h:309
  std::mutex mMutexFeatures;                  // MapPoint.h:310
};

}  // namespace cslam
#endif

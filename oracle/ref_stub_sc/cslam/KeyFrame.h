// Stand-ins for cslam::KeyFrame / MapPoint as shim/Sim3Correction_shim.cpp, shim/MapPoint_shim.cpp and the literal restatement of
// the two correction loops (oracle/ref_sim3_correction_wrap.cpp) see them (TEST INFRASTRUCTURE).  Real shared_ptr objects; the
// members are the reference's names and types (line numbers refer to the real headers).  KeyFrame::SetPose computes Twc and Ow as
// KeyFrame.cpp:298-306 does (f32, cv::gemm's left-to-right sums); UpdateConnections is defined by the wrapper, which logs the call and
// counts the keyframe's weights from mvpMapPoints; MapPoint::UpdateNormalAndDepth is defined by shim/MapPoint_shim.cpp.
#ifndef CCM_REF_STUB_SC_CSLAM_H
#define CCM_REF_STUB_SC_CSLAM_H
#include <boost/shared_ptr.hpp>
#include <map>
#include <mutex>
#include <utility>
#include <vector>

#include <cslam/estd.h>
#include <opencv2/core/core.hpp>

namespace cslam {

typedef std::pair<size_t, size_t> idpair;                                          // estd.h:69

class KeyFrame;
class MapPoint;
struct Sim3CorrectionProbe;

class KeyFrame {
 public:
  typedef boost::shared_ptr<KeyFrame> kfptr;
  typedef boost::shared_ptr<MapPoint> mpptr;
  void SetPose(const cv::Mat& Tcw_, bool bLock, bool bIgnorePoseMutex = false) {    // KeyFrame.h:133, KeyFrame.cpp:298-306
    (void)bLock; (void)bIgnorePoseMutex;
    std::unique_lock<std::mutex> lock(mMutexPose);
    Tcw_.copyTo(Tcw);
    Twc = cv::Mat::eye(4, 4, CV_32F);
    Ow = cv::Mat(3, 1, CV_32F);
    for (int r = 0; r < 3; r++) {
      float s = Tcw.at<float>(0, r) * Tcw.at<float>(0, 3);                          // Ow = -Rwc*tcw
      s = s + Tcw.at<float>(1, r) * Tcw.at<float>(1, 3);
      s = s + Tcw.at<float>(2, r) * Tcw.at<float>(2, 3);
      Ow.at<float>(r) = -s;
      for (int c = 0; c < 3; c++) Twc.at<float>(r, c) = Tcw.at<float>(c, r);
      Twc.at<float>(r, 3) = -s;
    }
  }
  cv::Mat GetPose() { std::unique_lock<std::mutex> lock(mMutexPose); return Tcw.clone(); }          // KeyFrame.h:135
  cv::Mat GetPoseInverse() { std::unique_lock<std::mutex> lock(mMutexPose); return Twc.clone(); }   // KeyFrame.h:136
  cv::Mat GetCameraCenter() { std::unique_lock<std::mutex> lock(mMutexPose); return Ow.clone(); }   // KeyFrame.h:137
  void UpdateConnections(bool bIgnoreMutex = false);                                               // KeyFrame.h:150
  std::vector<mpptr> GetMapPointMatches() { std::unique_lock<std::mutex> lock(mMutexFeatures); return mvpMapPoints; }   // KeyFrame.h:176
  bool isBad() { std::unique_lock<std::mutex> lock(mMutexConnections); return mbBad; }             // KeyFrame.h:194

  idpair mId;                                                                        // KeyFrame.h:282 (const there)
  size_t mUniqueId = 0;                                                              // KeyFrame.h:283
  idpair mCorrected_MM = idpair(size_t(-1), size_t(-1));                             // KeyFrame.h:316
  std::vector<cv::KeyPoint> mvKeysUn;                                                // KeyFrame.h:326 (const there)
  int mnScaleLevels = 8;                                                             // KeyFrame.h:337 (const there)
  std::vector<float> mvScaleFactors;                                                 // KeyFrame.h:340 (const there)
  cv::Mat Tcw, Twc, Ow;                                                              // KeyFrame.h:381-383
  std::vector<mpptr> mvpMapPoints;                                                   // KeyFrame.h:390
  std::map<kfptr, int> mConnectedKeyFrameWeights;                                    // KeyFrame.h:398
  bool mbBad = false;                                                                // KeyFrame.h:411
  std::mutex mMutexPose, mMutexConnections, mMutexFeatures;                          // KeyFrame.h:417-419
  int32_t mnRowForTest = -1;                                                         // the scene's row (not in the reference)
};

class MapPoint {
 public:
  typedef boost::shared_ptr<KeyFrame> kfptr;
  typedef boost::shared_ptr<MapPoint> mpptr;
  void SetWorldPos(const cv::Mat& Pos, bool bLock, bool bIgnorePosMutex = false) {  // MapPoint.h:132
    (void)bLock; (void)bIgnorePosMutex;
    std::unique_lock<std::mutex> lock(mMutexPos);
    Pos.copyTo(mWorldPos);
  }
  cv::Mat GetWorldPos() { std::unique_lock<std::mutex> lock(mMutexPos); return mWorldPos.clone(); }
  kfptr GetReferenceKeyFrame() { std::unique_lock<std::mutex> lock(mMutexFeatures); return mpRefKF; }
  std::map<kfptr, size_t> GetObservations() { std::unique_lock<std::mutex> lock(mMutexFeatures); return mObservations; }
  bool isBad() { std::unique_lock<std::mutex> lock(mMutexFeatures); std::unique_lock<std::mutex> lock2(mMutexPos); return mbBad; }   // MapPoint.h:152
  void UpdateNormalAndDepth();                                                                                                    // MapPoint.h:171
  void AddObservationForTest(kfptr pKF, size_t idx) { mObservations[pKF] = idx; }
  void SetReferenceForTest(kfptr pKF) { mpRefKF = pKF; }
  void SetBadForTest(bool b) { mbBad = b; }

  idpair mCorrectedByKF_LC = idpair(size_t(-1), size_t(-1));   // MapPoint.h:239
  size_t mCorrectedReference_LC = 0;                           // MapPoint.h:240
  idpair mCorrectedByKF_MM = idpair(size_t(-1), size_t(-1));   // MapPoint.h:245
  size_t mCorrectedReference_MM = 0;                           // MapPoint.h:246

 protected:
  friend struct Sim3CorrectionProbe;
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

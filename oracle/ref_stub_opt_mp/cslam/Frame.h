// Stand-ins for cslam::Frame / KeyFrame / MapPoint / Map / Communicator as shim/Optimizer_shim.cpp AND shim/MapPoint_shim.cpp see
// them together (TEST INFRASTRUCTURE).  The same classes as oracle/ref_stub_opt/cslam/Frame.h, with two differences:
//   * MapPoint declares UpdateNormalAndDepth() without a body (shim/MapPoint_shim.cpp defines it) and carries the members it writes,
//     mNormalVector / mfMinDistance / mfMaxDistance, and the two mutexes it locks (MapPoint.h:286,304-305,309-310);
//   * KeyFrame has GetCameraCenter(), mvScaleFactors and mnScaleLevels (KeyFrame.h:137,337,340).
// A MapPoint hands itself to MapPoint::on_destroy, when set, as the scene that holds it goes away: the wrapper
// (oracle/ref_optimizer_nd_wrap.cpp) reads there what the write-back left, without touching the driver of ref_optimizer_wrap.cpp.
// Original header comment:
//
// The real classes (cslam/include/cslam/{Frame,KeyFrame,MapPoint,Map}.h) pull in ROS, the communicator and message types.  These carry
// exactly the members the optimiser code touches, with the reference's names, types and signatures (line numbers in the comments refer
// to the real headers), plain storage behind them, and a record of what was asked of them (SetPose / SetWorldPos /
// UpdateNormalAndDepth / EraseObservation calls) for the tests to read.  oracle/ref_optimizer_wrap.cpp builds a map of them from flat
// arrays.  Used together with the reference's REAL cslam/Optimizer.h, Converter.h, Datatypes.h, estd.h, config.h.
#ifndef CCM_REF_STUB_OPT_MP_CSLAM_H
#define CCM_REF_STUB_OPT_MP_CSLAM_H
#include <boost/shared_ptr.hpp>
#include <map>
#include <mutex>
#include <set>
#include <vector>

#include <opencv2/core/core.hpp>

#include <cslam/config.h>
#include <cslam/estd.h>

namespace cslam {
using estd::idpair;

class KeyFrame;
class MapPoint;
class Map;
class Frame;

class MapPoint {
 public:
  typedef boost::shared_ptr<KeyFrame> kfptr;
  typedef boost::shared_ptr<MapPoint> mpptr;
  // MapPoint.h:132-171
  void SetWorldPos(const cv::Mat& Pos, bool bLock, bool bIgnorePosMutex = false) { (void)bLock; (void)bIgnorePosMutex; Pos.copyTo(mWorldPos); n_set_pos++; }
  cv::Mat GetWorldPos() { return mWorldPos.clone(); }
  kfptr GetReferenceKeyFrame() { return mpRefKF; }
  std::map<kfptr, size_t> GetObservations() { return mObservations; }
  void EraseObservation(kfptr pKF, bool bLock = false, bool bSuppressMapAction = false) { (void)bLock; (void)bSuppressMapAction; mObservations.erase(pKF); n_erased++; }
  int GetIndexInKeyFrame(kfptr pKF, bool bIgnoreMutex = false) { (void)bIgnoreMutex; return mObservations.count(pKF) ? (int)mObservations[pKF] : -1; }
  bool isBad() { return mbBad; }
  void UpdateNormalAndDepth();                                           // MapPoint.h:171, defined by shim/MapPoint_shim.cpp
  ~MapPoint() { if (on_destroy) on_destroy(*this); }
  static void (*on_destroy)(MapPoint&);
  // MapPoint.h:217-250
  idpair mId;
  size_t mUniqueId = 0;
  idpair mBALocalForKF;
  idpair mCorrectedByKF_LC;                                              // MapPoint.h:239-246
  size_t mCorrectedReference_LC = 0;
  idpair mCorrectedByKF_MM;
  size_t mCorrectedReference_MM = 0;
  idpair mBAGlobalForKF;
  cv::Mat mPosGBA;
  bool mbLoopCorrected = false;                                          // MapPoint.h:241
  static std::mutex mGlobalMutex;                                        // MapPoint.h:253
  // storage / record
  cv::Mat mWorldPos;
  std::map<kfptr, size_t> mObservations;
  kfptr mpRefKF;
  bool mbBad = false;
  int n_set_pos = 0, n_update_normal = 0, n_erased = 0;                  // n_update_normal stays 0: the member is the shim's
  cv::Mat mNormalVector;                                                 // MapPoint.h:286
  float mfMinDistance = 0.f, mfMaxDistance = 0.f;                        // MapPoint.h:304-305
  std::mutex mMutexPos, mMutexFeatures;                                  // MapPoint.h:309-310
};

// ORBextractor's mvScaleFactor for 8 levels at 1.2 (each level the previous one times the factor, in float)
inline std::vector<float> orb_scale_factors() {
  std::vector<float> s(8, 1.f);
  for (int l = 1; l < 8; l++) s[l] = s[l - 1] * 1.2f;
  return s;
}

class KeyFrame {
 public:
  typedef boost::shared_ptr<KeyFrame> kfptr;
  typedef boost::shared_ptr<MapPoint> mpptr;
  // KeyFrame.h:133-194
  void SetPose(const cv::Mat& Tcw_, bool bLock, bool bIgnorePoseMutex = false) { (void)bLock; (void)bIgnorePoseMutex; Tcw_.copyTo(Tcw); n_set_pose++; }
  cv::Mat GetPose() { return Tcw.clone(); }
  cv::Mat GetRotation() { return Tcw.rowRange(0, 3).colRange(0, 3).clone(); }
  cv::Mat GetTranslation() { return Tcw.rowRange(0, 3).col(3).clone(); }
  std::vector<kfptr> GetVectorCovisibleKeyFrames() { return mvpOrderedConnectedKeyFrames; }
  std::vector<kfptr> GetCovisiblesByWeight(const int& w) {
    std::vector<kfptr> out;
    for (size_t i = 0; i < mvpOrderedConnectedKeyFrames.size(); i++) if (mvOrderedWeights[i] >= w) out.push_back(mvpOrderedConnectedKeyFrames[i]);
    return out;
  }
  int GetWeight(kfptr pKF) {
    for (size_t i = 0; i < mvpOrderedConnectedKeyFrames.size(); i++) if (mvpOrderedConnectedKeyFrames[i] == pKF) return mvOrderedWeights[i];
    return 0;
  }
  kfptr GetParent(bool bIgnorePoseMutex = false) { (void)bIgnorePoseMutex; return mpParent; }
  std::set<kfptr> GetChilds() { return mspChildrens; }                   // KeyFrame.h:176
  cv::Mat GetCameraCenter() {                                            // KeyFrame.h:137; Ow as SetPose leaves it (KeyFrame.cpp:298-306)
    cv::Mat Rcw = Tcw.rowRange(0, 3).colRange(0, 3), tcw = Tcw.rowRange(0, 3).col(3);
    cv::Mat Rwc = Rcw.t();
    return -(Rwc * tcw);
  }
  std::vector<float> mvScaleFactors = orb_scale_factors();               // KeyFrame.h:340
  int mnScaleLevels = 8;                                                 // KeyFrame.h:337
  cv::Mat GetPoseInverse() {                                             // KeyFrame.h:136; Twc as SetPose leaves it (KeyFrame.cpp:298-306)
    cv::Mat Rcw = Tcw.rowRange(0, 3).colRange(0, 3), tcw = Tcw.rowRange(0, 3).col(3);
    cv::Mat Rwc = Rcw.t();
    cv::Mat Ow = -(Rwc * tcw);
    cv::Mat Twc = cv::Mat::eye(4, 4, CV_32F);
    for (int r = 0; r < 3; r++) {
      for (int c = 0; c < 3; c++) Twc.at<float>(r, c) = Rwc.at<float>(r, c);
      Twc.at<float>(r, 3) = Ow.at<float>(r);
    }
    return Twc;
  }
  bool hasChild(kfptr pKF) { return mspChildrens.count(pKF) != 0; }
  std::set<kfptr> GetLoopEdges() { return mspLoopEdges; }
  void EraseMapPointMatch(const size_t& idx, bool bLock = false) { (void)bLock; mvpMapPoints[idx] = mpptr(); n_erased++; }
  void EraseMapPointMatch(mpptr pMP, bool bLock = false) {
    (void)bLock;
    for (size_t i = 0; i < mvpMapPoints.size(); i++) if (mvpMapPoints[i] == pMP) mvpMapPoints[i] = mpptr();
    n_erased++;
  }
  std::vector<mpptr> GetMapPointMatches() { return mvpMapPoints; }
  bool isBad() { return mbBad; }
  // KeyFrame.h:129,282-342
  bool mbUpdatedByServer = false;
  idpair mId;
  size_t mUniqueId = 0;
  idpair mBALocalForKF;
  idpair mBAFixedForKF;
  cv::Mat mTcwGBA;
  cv::Mat mTcwBefGBA;                                                    // KeyFrame.h:311
  bool mbLoopCorrected = false;                                          // KeyFrame.h:313
  idpair mBAGlobalForKF;
  float fx = 0, fy = 0, cx = 0, cy = 0, invfx = 0, invfy = 0;
  std::vector<cv::KeyPoint> mvKeysUn;
  std::vector<float> mvInvLevelSigma2;
  cv::Mat mK;                                                            // KeyFrame.h:349
  // storage / record
  cv::Mat Tcw;
  std::vector<mpptr> mvpMapPoints;
  std::vector<kfptr> mvpOrderedConnectedKeyFrames;
  std::vector<int> mvOrderedWeights;
  kfptr mpParent;
  std::set<kfptr> mspChildrens, mspLoopEdges;
  bool mbBad = false;
  int n_set_pose = 0, n_erased = 0;
};

class Frame {
 public:
  typedef boost::shared_ptr<MapPoint> mpptr;
  void SetPose(cv::Mat Tcw) { mTcw = Tcw.clone(); n_set_pose++; }     // Frame.h:80
  int N = 0;
  static float fx, fy, cx, cy;                                           // Frame.h:116-119
  std::vector<cv::KeyPoint> mvKeysUn;
  std::vector<mpptr> mvpMapPoints;
  std::vector<bool> mvbOutlier;                                          // Frame.h:144
  cv::Mat mTcw, mK;                                                      // Frame.h:152
  std::vector<float> mvInvLevelSigma2;                                   // Frame.h:168
  int n_set_pose = 0;
};

class Map {
 public:
  typedef boost::shared_ptr<KeyFrame> kfptr;
  typedef boost::shared_ptr<MapPoint> mpptr;
  std::set<size_t> msuAssClients;                                        // Map.h:93
  size_t mMapId = 0;                                                     // Map.h:100
  mpptr GetMpPtr(size_t MpId, size_t ClientId) {                         // Map.h:121-122
    for (size_t i = 0; i < mps.size(); i++) if (mps[i]->mId == idpair(MpId, ClientId)) return mps[i];
    return mpptr();
  }
  mpptr GetMpPtr(idpair id) { return GetMpPtr(id.first, id.second); }
  std::vector<kfptr> GetAllKeyFrames() { return kfs; }                   // Map.h:132-133
  std::vector<mpptr> GetAllMapPoints() { return mps; }
  long unsigned int GetMaxKFidUnique() { long unsigned int m = 0; for (size_t i = 0; i < kfs.size(); i++) if (kfs[i]->mUniqueId > m) m = kfs[i]->mUniqueId; return m; }
  std::vector<kfptr> mvpKeyFrameOrigins;                                 // Map.h:163
  bool LockMapUpdate() { if (!locked) { locked = true; return true; } return false; }   // Map.h:175-177
  void UnLockMapUpdate() { if (!locked) throw estd::infrastructure_ex(); locked = false; }
  std::vector<kfptr> kfs;
  std::vector<mpptr> mps;
  bool locked = false;
};

class Communicator {};

}  // namespace cslam
#endif

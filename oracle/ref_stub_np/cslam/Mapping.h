// Stand-ins for cslam::LocalMapping / KeyFrame / MapPoint / Map as shim/NewMapPoints_shim.cpp sees them (TEST INFRASTRUCTURE).
//
// The real cslam/include/cslam/Mapping.h pulls in ROS, the communicator, the map and the whole front end; these classes carry exactly
// what LocalMapping::CreateNewMapPoints (cslam/src/Mapping.cpp:284-469) touches, with the reference's names and types (line numbers
// refer to the real headers).  LocalMapping declares CreateNewMapPoints without defining it: the shim defines it.  The members of
// MapPoint that the body calls after creating a point (ComputeDistinctiveDescriptors, UpdateNormalAndDepth) are other members of the
// library; here they only record that they ran, and in which order, in the point's call log.
#ifndef CCM_REF_STUB_NP_CSLAM_MAPPING_H
#define CCM_REF_STUB_NP_CSLAM_MAPPING_H
#include <boost/shared_ptr.hpp>
#include <list>
#include <map>
#include <mutex>
#include <set>
#include <string>
#include <utility>
#include <vector>

#include <opencv2/core/core.hpp>

#include "../../../ccm_slam_b200/csrc/new_points_math.cuh"

namespace DBoW2 {
typedef unsigned int NodeId;
typedef std::map<NodeId, std::vector<unsigned int> > FeatureVector;   // DBoW2/FeatureVector.h:22
}  // namespace DBoW2

namespace cv {
// cv::SVD::compute for the one use in CreateNewMapPoints: a 4x4 CV_32F matrix, vt.row(3) read.  OpenCV's result depends on its build
// (its own Jacobi iteration or LAPACK); the stand-in runs the arithmetic the library states (new_points_math.cuh), fills vt.row(3)
// and leaves w, u and the other rows of vt zero.
struct SVD {
  enum { MODIFY_A = 1, NO_UV = 2, FULL_UV = 4 };
  static void compute(const Mat& A, Mat& w, Mat& u, Mat& vt, int = 0) {
    float a[16], x[4];
    for (int r = 0; r < 4; r++) for (int c = 0; c < 4; c++) a[4 * r + c] = A.at<float>(r, c);
    ccm::newpts::svd4_null(a, x);
    w = Mat::zeros(4, 1, CV_32F); u = Mat::zeros(4, 4, CV_32F); vt = Mat::zeros(4, 4, CV_32F);
    for (int c = 0; c < 4; c++) vt.at<float>(3, c) = x[c];
  }
};
// Mat::inv() of an upper-triangular 3x3 camera matrix (ComputeF12, Mapping.cpp:565), in f32
inline Mat inv3(const Mat& K) {
  const float a = K.at<float>(0, 0), b = K.at<float>(0, 1), c = K.at<float>(0, 2), d = K.at<float>(1, 0), e = K.at<float>(1, 1),
              f = K.at<float>(1, 2), g = K.at<float>(2, 0), h = K.at<float>(2, 1), i = K.at<float>(2, 2);
  const float det = a * (e * i - f * h) - b * (d * i - f * g) + c * (d * h - e * g), s = 1.0f / det;
  Mat m(3, 3, CV_32F);
  m.at<float>(0, 0) = (e * i - f * h) * s; m.at<float>(0, 1) = (c * h - b * i) * s; m.at<float>(0, 2) = (b * f - c * e) * s;
  m.at<float>(1, 0) = (f * g - d * i) * s; m.at<float>(1, 1) = (a * i - c * g) * s; m.at<float>(1, 2) = (c * d - a * f) * s;
  m.at<float>(2, 0) = (d * h - e * g) * s; m.at<float>(2, 1) = (b * g - a * h) * s; m.at<float>(2, 2) = (a * e - b * d) * s;
  return m;
}
}  // namespace cv

namespace cslam {

class KeyFrame;
class MapPoint;
class Map;
struct Communicator {};
struct CentralControl { int mSysState = 0; };   // CentralControl.h (eSystemState there)

class KeyFrame {
 public:
  typedef boost::shared_ptr<KeyFrame> kfptr;
  typedef boost::shared_ptr<MapPoint> mpptr;
  cv::Mat GetRotation() { std::unique_lock<std::mutex> lock(mMutexPose); return Tcw.rowRange(0, 3).colRange(0, 3).clone(); }   // KeyFrame.h:139
  cv::Mat GetTranslation() { std::unique_lock<std::mutex> lock(mMutexPose); return Tcw.rowRange(0, 3).col(3).clone(); }         // KeyFrame.h:140
  cv::Mat GetCameraCenter() { std::unique_lock<std::mutex> lock(mMutexPose); return Ow.clone(); }                               // KeyFrame.h:137
  std::vector<kfptr> GetBestCovisibilityKeyFrames(const int& N) {                                                             // KeyFrame.h:152
    return (int)mvpOrderedConnectedKeyFrames.size() < N ? mvpOrderedConnectedKeyFrames
                                                        : std::vector<kfptr>(mvpOrderedConnectedKeyFrames.begin(), mvpOrderedConnectedKeyFrames.begin() + N);
  }
  mpptr GetMapPoint(const size_t& idx) { std::unique_lock<std::mutex> lock(mMutexFeatures); return mvpMapPoints[idx]; }         // KeyFrame.h:177
  void AddMapPoint(mpptr pMP, const size_t& idx, bool = false) { std::unique_lock<std::mutex> lock(mMutexFeatures); mvpMapPoints[idx] = pMP; }   // KeyFrame.h:170
  float ComputeSceneMedianDepth(const int) { return mMedianDepthForTest; }   // KeyFrame.h:198; computed from the map points there
  float fx, fy, cx, cy, invfx, invfy;            // KeyFrame.h:309
  int N = 0;                                     // KeyFrame.h:316
  std::vector<cv::KeyPoint> mvKeysUn;            // KeyFrame.h:326
  cv::Mat mDescriptors;                          // KeyFrame.h:327
  DBoW2::FeatureVector mFeatVec;                 // KeyFrame.h:331
  float mfScaleFactor = 1.2f;                    // KeyFrame.h:338
  std::vector<float> mvScaleFactors;             // KeyFrame.h:340
  std::vector<float> mvLevelSigma2;              // KeyFrame.h:341
  cv::Mat mK;                                    // KeyFrame.h:350
  // storage
  cv::Mat Tcw, Ow;                               // KeyFrame.h:380-383
  std::vector<mpptr> mvpMapPoints;               // KeyFrame.h:386
  std::vector<kfptr> mvpOrderedConnectedKeyFrames;   // KeyFrame.h:395
  float mMedianDepthForTest = 1.f;
  std::mutex mMutexPose, mMutexFeatures;
};

class MapPoint {
 public:
  typedef boost::shared_ptr<KeyFrame> kfptr;
  typedef boost::shared_ptr<MapPoint> mpptr;
  typedef boost::shared_ptr<Map> mapptr;
  typedef boost::shared_ptr<Communicator> commptr;
  MapPoint(const cv::Mat& Pos, kfptr pRefKF, mapptr pMap, size_t ClientId, commptr pComm, int SysState, size_t UniqueId)   // MapPoint.h:69
      : mWorldPos(Pos.clone()), mpRefKF(pRefKF), mClientId(ClientId), mSysState(SysState), mUniqueId(UniqueId) { (void)pMap; (void)pComm; }
  void AddObservation(kfptr pKF, size_t idx, bool = false) { mObservations[pKF] = idx; mLog += 'o'; }   // MapPoint.h:141
  void ComputeDistinctiveDescriptors() { mLog += 'd'; }                                                  // MapPoint.h:166
  void UpdateNormalAndDepth() { mLog += 'n'; }                                                           // MapPoint.h:171
  cv::Mat mWorldPos;
  std::map<kfptr, size_t> mObservations;
  kfptr mpRefKF;
  size_t mClientId, mUniqueId;
  int mSysState;
  std::string mLog;   // the members called on this point, in order
};

class Map {
 public:
  typedef boost::shared_ptr<MapPoint> mpptr;
  void AddMapPoint(mpptr pMP) { pMP->mLog += 'm'; mvpAdded.push_back(pMP); }   // Map.h:90
  std::vector<mpptr> mvpAdded;
};

class LocalMapping {
 public:
  typedef boost::shared_ptr<KeyFrame> kfptr;
  typedef boost::shared_ptr<MapPoint> mpptr;
  typedef boost::shared_ptr<Map> mapptr;
  typedef boost::shared_ptr<Communicator> commptr;
  typedef boost::shared_ptr<CentralControl> ccptr;
  void CreateNewMapPoints();                                   // Mapping.h:97
  cv::Mat ComputeF12(kfptr& pKF1, kfptr& pKF2);                // Mapping.h:106
  cv::Mat SkewSymmetricMatrix(const cv::Mat& v);               // Mapping.h:107
  // Mapping.h:88; there it reads mlNewKeyFrames under its mutex.  Here the n-th call answers true when n == mForceAtPoll (1-based)
  bool CheckNewKeyFrames() { return ++mPolls == mForceAtPoll; }
  ccptr mpCC;                                                  // Mapping.h:113
  mapptr mpMap;                                                // Mapping.h:114
  commptr mpComm;                                              // Mapping.h:115
  size_t mClientId = 0;                                        // Mapping.h:121
  kfptr mpCurrentKeyFrame;                                     // Mapping.h:131
  std::list<mpptr> mlpRecentAddedMapPoints;                    // Mapping.h:132
  int mPolls = 0, mForceAtPoll = -1;
};

}  // namespace cslam
#endif

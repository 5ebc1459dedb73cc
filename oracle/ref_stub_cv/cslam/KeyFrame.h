// Stand-ins for cslam::KeyFrame / MapPoint / Map / KeyFrameDatabase as shim/KeyFrameConnections_shim.cpp sees them
// (TEST INFRASTRUCTURE).
//
// The reference's KeyFrame.h needs ROS messages, cereal, DBoW2 and the communicator, so KeyFrame.cpp does not build here.  These
// classes carry exactly what KeyFrame::UpdateConnections and its batch preparation touch, with the reference's types: real shared_ptr
// objects (boost::shared_ptr is std::shared_ptr in oracle/ref_stub), std::map<kfptr,int> ordered by the pointer, std::set<kfptr>.
// UpdateConnections is declared without a body (the shim defines it); AddConnection, UpdateBestCovisibles, AddChild, EraseConnection
// and SetBadFlag are defined by oracle/ref_covis_wrap.cpp.  Line numbers refer to the real headers.
#ifndef CCM_REF_STUB_CV_CSLAM_H
#define CCM_REF_STUB_CV_CSLAM_H
#include <boost/shared_ptr.hpp>
#include <map>
#include <mutex>
#include <set>
#include <utility>
#include <vector>

#include <cslam/estd.h>
#include <opencv2/core/core.hpp>

namespace cslam {

using namespace estd;
typedef std::pair<size_t, size_t> idpair;                                          // estd.h:69
enum eSystemState { NOTYPE = -1, CLIENT = 0, SERVER = 1 };                          // Datatypes.h:24-28

class KeyFrame;
class MapPoint;

class Map {
 public:
  typedef boost::shared_ptr<KeyFrame> kfptr;
  size_t mMapId = 0;                                                                 // Map.h:100
  void EraseKeyFrame(kfptr pKF) { mErased.insert(pKF); }                             // Map.h:107
  kfptr GetKfPtr(size_t KfId, size_t ClientId, bool bIgnoreMutex = false) {          // Map.h:118
    (void)bIgnoreMutex;
    std::map<idpair, kfptr>::iterator it = mmpKeyFrames.find(std::make_pair(KfId, ClientId));
    return it == mmpKeyFrames.end() ? kfptr() : it->second;
  }
  std::map<idpair, kfptr> mmpKeyFrames;   // the map's keyframes by mId (the first row of an mId wins)
  std::set<kfptr> mErased;
};

class KeyFrameDatabase {
 public:
  void erase(boost::shared_ptr<KeyFrame> pKF) { (void)pKF; }                         // Database.h:71
};

class KeyFrame : public boost::enable_shared_from_this<KeyFrame> {
 public:
  typedef boost::shared_ptr<KeyFrame> kfptr;
  typedef boost::shared_ptr<MapPoint> mpptr;
  typedef boost::shared_ptr<Map> mapptr;
  typedef boost::shared_ptr<KeyFrameDatabase> dbptr;

  void SetPose(const cv::Mat& Tcw_, bool bLock, bool bIgnorePoseMutex = false) {    // KeyFrame.h:133
    (void)bLock; (void)bIgnorePoseMutex;
    std::unique_lock<std::mutex> lock(mMutexPose);
    Tcw_.copyTo(Tcw);
  }
  void AddConnection(kfptr pKF, const int& weight);                                  // KeyFrame.h:148
  void EraseConnection(kfptr pKF);                                                   // KeyFrame.h:149
  void UpdateConnections(bool bIgnoreMutex = false);                                 // KeyFrame.h:150
  void UpdateBestCovisibles();                                                       // KeyFrame.h:151
  void AddChild(kfptr pKF);                                                          // KeyFrame.h:159
  void AddMapPoint(mpptr pMP, const size_t& idx, bool bLock = false) {               // KeyFrame.h:171
    (void)bLock;
    std::unique_lock<std::mutex> lock(mMutexFeatures);
    mvpMapPoints[idx] = pMP;
  }
  void SetBadFlag(bool bSuppressMapAction = false, bool bNoParent = false);          // KeyFrame.h:193
  bool isBad() { std::unique_lock<std::mutex> lock(mMutexConnections); return mbBad; }   // KeyFrame.h:194

  bool mbFromServer = false;                                                         // KeyFrame.h:128
  idpair mId;                                                                        // KeyFrame.h:282 (const there)
  mapptr mpMap;                                                                      // KeyFrame.h:374
  eSystemState mSysState = SERVER;                                                   // KeyFrame.h:376
  dbptr mpKeyFrameDB;                                                                // KeyFrame.h:377
  cv::Mat Tcw;                                                                       // KeyFrame.h:381
  std::vector<mpptr> mvpMapPoints;                                                   // KeyFrame.h:390
  std::map<kfptr, int> mConnectedKeyFrameWeights;                                    // KeyFrame.h:398
  std::vector<kfptr> mvpOrderedConnectedKeyFrames;                                   // KeyFrame.h:399
  std::vector<int> mvOrderedWeights;                                                 // KeyFrame.h:400
  bool mbFirstConnection = true;                                                     // KeyFrame.h:403
  kfptr mpParent;                                                                    // KeyFrame.h:404
  std::set<kfptr> mspChildrens;                                                      // KeyFrame.h:405
  bool mbBad = false;                                                                // KeyFrame.h:411
  std::mutex mMutexPose, mMutexConnections, mMutexFeatures;                          // KeyFrame.h:417-419
  int32_t mnRowForTest = -1;                                                         // the scene's row (not in the reference)
};

class MapPoint {
 public:
  typedef boost::shared_ptr<KeyFrame> kfptr;
  std::map<kfptr, size_t> GetObservations() { std::unique_lock<std::mutex> lock(mMutexFeatures); return mObservations; }   // MapPoint.h:141
  int Observations() { std::unique_lock<std::mutex> lock(mMutexFeatures); return nObs; }                                   // MapPoint.h:142
  void EraseObservation(kfptr pKF, bool bLock = false, bool bSuppressMapAction = false) {                                  // MapPoint.h:145
    (void)bLock; (void)bSuppressMapAction;
    std::unique_lock<std::mutex> lock(mMutexFeatures);
    if (mObservations.erase(pKF)) nObs--;
  }
  bool isBad() { std::unique_lock<std::mutex> lock(mMutexFeatures); return mbBad; }                                         // MapPoint.h:152
  // scene construction and change (the reference goes through AddObservation / EraseObservation / SetBadFlag)
  void AddObservationForTest(kfptr pKF, size_t idx) { if (!mObservations.count(pKF)) nObs++; mObservations[pKF] = idx; }
  void ReplaceObserverForTest(kfptr from, kfptr to) {
    size_t idx = mObservations[from];
    mObservations.erase(from);
    mObservations[to] = idx;
  }
  void SetBadForTest(bool b) { mbBad = b; }

 protected:
  int nObs = 0;                                                                       // MapPoint.h:221
  std::map<kfptr, size_t> mObservations;                                              // MapPoint.h:281
  bool mbBad = false;                                                                 // MapPoint.h:299
  std::mutex mMutexFeatures;                                                          // MapPoint.h:310
};

}  // namespace cslam
#endif

// Stand-ins for cslam::KeyFrame / MapPoint / Map / Converter as shim/SearchAndFuse_shim.cpp and the literal restatement of both
// SearchAndFuse bodies (oracle/ref_search_and_fuse_wrap.cpp) see them (TEST INFRASTRUCTURE).  Real shared_ptr objects; the members carry
// the reference's names and types (line numbers refer to the real sources).  Restated from cslam/src/KeyFrame.cpp / MapPoint.cpp:
// GetMapPoints, GetFeaturesInArea, the slot members, AddObservation, EraseObservation and SetBadFlag (monocular).  Replace and
// ReplaceAndLock are restated in the wrapper.  Two differences, the same for the shim and the restatement:
//   * mObservations is ordered by keyframe id, not by address, so that two copies of one scene walk Replace's loop in one order;
//   * ComputeDistinctiveDescriptors (another member of the library) is a fixed rule that changes the bytes: the descriptor becomes the
//     keyframe descriptor of the point's first observation.
// Every member that takes a lock flag appends one letter to the point's (or keyframe's) log: lower case unlocked, upper case locked.
#ifndef CCM_REF_STUB_SF_CSLAM_H
#define CCM_REF_STUB_SF_CSLAM_H
#include <boost/shared_ptr.hpp>
#include <cmath>
#include <map>
#include <memory>
#include <mutex>
#include <set>
#include <string>
#include <vector>

#include <cslam/estd.h>
#include <opencv2/core/core.hpp>

namespace cslam {

class KeyFrame;
class MapPoint;

struct KfById {
  bool operator()(const boost::shared_ptr<KeyFrame>& a, const boost::shared_ptr<KeyFrame>& b) const;
};

inline char lock_letter(char c, bool bLock) { return bLock ? (char)(c - 'a' + 'A') : c; }

class KeyFrame {
 public:
  typedef boost::shared_ptr<KeyFrame> kfptr;
  typedef boost::shared_ptr<MapPoint> mpptr;
  std::set<mpptr> GetMapPoints();                                                                                              // KeyFrame.cpp:569-582
  std::vector<mpptr> GetMapPointMatches() { std::unique_lock<std::mutex> lock(mMutexFeatures); return mvpMapPoints; }          // KeyFrame.h:176
  mpptr GetMapPoint(const size_t& idx) { std::unique_lock<std::mutex> lock(mMutexFeatures); return mvpMapPoints[idx]; }         // KeyFrame.h:177
  void AddMapPoint(mpptr pMP, const size_t& idx, bool bLock = false) { mLog += lock_letter('a', bLock); mvpMapPoints[idx] = pMP; }     // KeyFrame.cpp:714
  void EraseMapPointMatch(const size_t& idx, bool bLock = false) { mLog += lock_letter('e', bLock); mvpMapPoints[idx] = nullptr; }     // KeyFrame.cpp:727
  void ReplaceMapPointMatch(const size_t& idx, mpptr pMP, bool bLock = false) { mLog += lock_letter('r', bLock); mvpMapPoints[idx] = pMP; }   // KeyFrame.cpp:758
  bool IsEmpty() { return mbIsEmpty; }                                                                                        // KeyFrame.h:195
  bool IsInImage(const float& x, const float& y) const { return (x >= mnMinX && x < mnMaxX && y >= mnMinY && y < mnMaxY); }   // KeyFrame.cpp:1203
  // KeyFrame::GetFeaturesInArea (KeyFrame.cpp:1162-1201) over mGrid as AssignFeaturesToGrid fills it
  std::vector<size_t> GetFeaturesInArea(const float& x, const float& y, const float& r) const {
    std::vector<size_t> vIndices;
    const int nMinCellX = std::max(0, (int)floor((x - mnMinX - r) * mfGridElementWidthInv));
    if (nMinCellX >= mnGridCols) return vIndices;
    const int nMaxCellX = std::min((int)mnGridCols - 1, (int)ceil((x - mnMinX + r) * mfGridElementWidthInv));
    if (nMaxCellX < 0) return vIndices;
    const int nMinCellY = std::max(0, (int)floor((y - mnMinY - r) * mfGridElementHeightInv));
    if (nMinCellY >= mnGridRows) return vIndices;
    const int nMaxCellY = std::min((int)mnGridRows - 1, (int)ceil((y - mnMinY + r) * mfGridElementHeightInv));
    if (nMaxCellY < 0) return vIndices;
    for (int ix = nMinCellX; ix <= nMaxCellX; ix++)
      for (int iy = nMinCellY; iy <= nMaxCellY; iy++) {
        const std::vector<size_t>& vCell = mGrid[ix][iy];
        for (size_t j = 0, jend = vCell.size(); j < jend; j++) {
          const cv::KeyPoint& kpUn = mvKeysUn[vCell[j]];
          const float distx = kpUn.pt.x - x;
          const float disty = kpUn.pt.y - y;
          if (fabs(distx) < r && fabs(disty) < r) vIndices.push_back(vCell[j]);
        }
      }
    return vIndices;
  }
  void AssignFeaturesToGrid() {   // KeyFrame.cpp:206-226 with PosInGrid (round of the float expression)
    mGrid.assign(mnGridCols, std::vector<std::vector<size_t> >(mnGridRows));
    for (int i = 0; i < N; i++) {
      const int px = (int)round((mvKeysUn[i].pt.x - mnMinX) * mfGridElementWidthInv);
      const int py = (int)round((mvKeysUn[i].pt.y - mnMinY) * mfGridElementHeightInv);
      if (px < 0 || px >= mnGridCols || py < 0 || py >= mnGridRows) continue;
      mGrid[px][py].push_back(i);
    }
  }
  size_t mId = 0;                                // KeyFrame.h:227 (an idpair there)
  float fx, fy, cx, cy;                          // KeyFrame.h:309
  int N = 0;                                     // KeyFrame.h:316
  std::vector<cv::KeyPoint> mvKeysUn;            // KeyFrame.h:326
  cv::Mat mDescriptors;                          // KeyFrame.h:327
  int mnScaleLevels = 8;                         // KeyFrame.h:337
  float mfLogScaleFactor = 0.f;                  // KeyFrame.h:339
  std::vector<float> mvScaleFactors, mvInvLevelSigma2;   // KeyFrame.h:340-343
  int mnMinX = 0, mnMinY = 0, mnMaxX = 0, mnMaxY = 0;    // KeyFrame.h:345-348
  int mnGridCols = 64, mnGridRows = 48;                  // KeyFrame.h:301-302
  float mfGridElementWidthInv = 0.f, mfGridElementHeightInv = 0.f;   // KeyFrame.h:303-304
  std::vector<std::vector<std::vector<size_t> > > mGrid; // KeyFrame.h:389
  std::vector<mpptr> mvpMapPoints;               // KeyFrame.h:386
  bool mbIsEmpty = false;                        // KeyFrame.h:412
  std::string mLog;                              // the slot members called on this keyframe, in order
  std::mutex mMutexFeatures;
};

inline bool KfById::operator()(const boost::shared_ptr<KeyFrame>& a, const boost::shared_ptr<KeyFrame>& b) const { return a->mId < b->mId; }

class Map {
 public:
  typedef boost::shared_ptr<MapPoint> mpptr;
  void EraseMapPoint(mpptr pMP);   // Map.h:91
};

class MapPoint {
 public:
  typedef boost::shared_ptr<KeyFrame> kfptr;
  typedef boost::shared_ptr<MapPoint> mpptr;
  typedef boost::shared_ptr<Map> mapptr;
  cv::Mat GetWorldPos() { std::unique_lock<std::mutex> lock(mMutexPos); return mWorldPos.clone(); }     // MapPoint.h:134
  cv::Mat GetNormal() { std::unique_lock<std::mutex> lock(mMutexPos); return mNormalVector.clone(); }   // MapPoint.h:135
  cv::Mat GetDescriptor() { std::unique_lock<std::mutex> lock(mMutexFeatures); return mDescriptor.clone(); }   // MapPoint.h:167
  float GetMinDistanceInvariance() { return 0.8f * mfMinDistance; }   // MapPoint.cpp:825
  float GetMaxDistanceInvariance() { return 1.2f * mfMaxDistance; }   // MapPoint.cpp:831
  int PredictScale(const float& currentDist, kfptr pKF) {             // MapPoint.cpp:837-852
    float ratio;
    ratio = mfMaxDistance / currentDist;
    int nScale = std::ceil(std::log(ratio) / pKF->mfLogScaleFactor);
    if (nScale < 0) nScale = 0;
    else if (nScale >= pKF->mnScaleLevels) nScale = pKF->mnScaleLevels - 1;
    return nScale;
  }
  bool isBad() { return mbBad; }                                                          // MapPoint.h:152
  int Observations() { return nObs; }                                                     // MapPoint.h:146
  bool IsInKeyFrame(kfptr pKF) { return mObservations.count(pKF) > 0; }                   // MapPoint.cpp:571
  int GetIndexInKeyFrame(kfptr pKF) { return mObservations.count(pKF) ? (int)mObservations[pKF] : -1; }   // MapPoint.cpp:562
  void AddObservation(kfptr pKF, size_t idx, bool bLock = false) {                        // MapPoint.cpp:417-440
    mLog += lock_letter('o', bLock);
    if (mObservations.count(pKF)) return;
    mObservations[pKF] = idx;
    nObs++;
  }
  void EraseObservation(kfptr pKF, bool bLock = false) {                                  // MapPoint.cpp:442-510, monocular
    mLog += lock_letter('x', bLock);
    bool bBad = false;
    if (mObservations.count(pKF)) {
      nObs--;
      mObservations.erase(pKF);
      if (nObs <= 2) bBad = true;
    }
    if (bBad) SetBadFlag();
  }
  void SetBadFlag() {                                                                     // MapPoint.cpp:520-548
    mLog += 'b';
    std::map<kfptr, size_t, KfById> obs = mObservations;
    mbBad = true;
    mObservations.clear();
    for (auto& o : obs) o.first->EraseMapPointMatch(o.second);
    mpMap->EraseMapPoint(self());
  }
  void IncreaseVisible(int n = 1) { mnVisible += n; }
  void IncreaseFound(int n = 1) { mnFound += n; }
  void ComputeDistinctiveDescriptors() {   // stand-in rule (see the top of this file)
    mLog += 'd';
    if (mbBad || mObservations.empty()) return;
    const auto& o = *mObservations.begin();
    mDescriptor = o.first->mDescriptors.row((int)o.second).clone();
  }
  void Replace(mpptr pMP, bool bLock = false);   // MapPoint.cpp:583-678, restated in oracle/ref_search_and_fuse_wrap.cpp
  void ReplaceAndLock(mpptr pMP);                // MapPoint.cpp:680-720, restated in oracle/ref_search_and_fuse_wrap.cpp
  mpptr self() { return mSelf.lock(); }

  size_t mId = 0;                                // MapPoint.h:233 (an idpair there)
  bool mbDoNotReplace = false;                   // MapPoint.h:158
  cv::Mat mWorldPos, mNormalVector, mDescriptor;
  std::map<kfptr, size_t, KfById> mObservations;
  int nObs = 0, mnVisible = 1, mnFound = 1;
  bool mbBad = false;
  mpptr mpReplaced;
  mapptr mpMap;
  std::weak_ptr<MapPoint> mSelf;
  std::string mLog;   // the members called on this point, in order

 protected:
  float mfMinDistance = 0.f, mfMaxDistance = 0.f;   // MapPoint.h:206-207 (protected there too)
  std::mutex mMutexPos, mMutexFeatures;
  friend struct SfSceneAccess;
};

inline std::set<KeyFrame::mpptr> KeyFrame::GetMapPoints() {
  std::unique_lock<std::mutex> lock(mMutexFeatures);
  std::set<mpptr> s;
  for (size_t i = 0, iend = mvpMapPoints.size(); i < iend; i++) {
    if (!mvpMapPoints[i]) continue;
    mpptr pMP = mvpMapPoints[i];
    if (!pMP->isBad()) s.insert(pMP);
  }
  return s;
}

inline void Map::EraseMapPoint(mpptr pMP) { pMP->mLog += 'e'; }

}  // namespace cslam
#endif

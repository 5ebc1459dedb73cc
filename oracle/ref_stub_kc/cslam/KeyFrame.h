// Stand-in for cslam::KeyFrame as shim/KeyFrameCulling_shim.cpp sees it (TEST INFRASTRUCTURE).
//
// The real header pulls in ROS, the communicator and the whole front end; this class carries what LocalMapping::KeyFrameCullingV3
// (cslam/src/Mapping.cpp:771-863) touches, with the reference's names and access (line numbers refer to cslam/include/cslam/KeyFrame.h).
// SetBadFlag is restated in oracle/ref_keyframe_culling_wrap.cpp for the server, up to the parts this member reaches: the connection
// and spanning-tree surgery and the map and database erasure are not stood in for (they change nothing the member reads).  KcScene, the
// test's scene builder, is a friend so that it can set and read the protected flags.
#ifndef CCM_REF_STUB_KC_CSLAM_KEYFRAME_H
#define CCM_REF_STUB_KC_CSLAM_KEYFRAME_H
#include <boost/shared_ptr.hpp>
#include <cstddef>
#include <mutex>
#include <utility>
#include <vector>

#include <opencv2/core/core.hpp>

namespace cslam {

class MapPoint;
typedef std::pair<size_t, size_t> idpair;

class KeyFrame : public boost::enable_shared_from_this<KeyFrame> {   // KeyFrame.h:81
 public:
  typedef boost::shared_ptr<KeyFrame> kfptr;
  typedef boost::shared_ptr<MapPoint> mpptr;
  std::vector<kfptr> GetVectorCovisibleKeyFrames() { std::unique_lock<std::mutex> lock(mMutexConnections); return mvpOrderedConnectedKeyFrames; }   // KeyFrame.h:153
  void EraseMapPointMatch(const size_t& idx, bool = false) { std::unique_lock<std::mutex> lock(mMutexFeatures); mvpMapPoints[idx] = nullptr; }   // KeyFrame.h:172
  std::vector<mpptr> GetMapPointMatches() { std::unique_lock<std::mutex> lock(mMutexFeatures); return mvpMapPoints; }                          // KeyFrame.h:176
  void SetBadFlag(bool bSuppressMapAction = false, bool bNoParent = false);                                                                  // KeyFrame.h:193
  bool isBad() { std::unique_lock<std::mutex> lock(mMutexConnections); return mbBad; }                                                     // KeyFrame.h:194

  idpair mId;                                    // KeyFrame.h:282
  std::vector<cv::KeyPoint> mvKeysUn;            // KeyFrame.h:326

 protected:
  friend struct KcScene;
  std::vector<mpptr> mvpMapPoints;               // KeyFrame.h:390
  std::vector<kfptr> mvpOrderedConnectedKeyFrames;   // KeyFrame.h:395
  bool mbNotErase = false;                       // KeyFrame.h:409
  bool mbToBeErased = false;                     // KeyFrame.h:410
  bool mbBad = false;                            // KeyFrame.h:411
  std::mutex mMutexConnections, mMutexFeatures;
};

struct KfById {   // mObservations is ordered by mId here, not by address, so that two copies of one scene walk it in one order
  bool operator()(const boost::shared_ptr<KeyFrame>& a, const boost::shared_ptr<KeyFrame>& b) const { return a->mId < b->mId; }
};

}  // namespace cslam
#endif

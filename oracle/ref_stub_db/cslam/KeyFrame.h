// Stand-ins for the classes the reference's cslam/src/Database.cpp reads (TEST INFRASTRUCTURE): KeyFrame, Map, Frame, MapPoint with
// the reference's member names and types (cslam/include/cslam/KeyFrame.h:123,152-154,282,301-307,330; Map.h:93,158; Frame.h:134,156;
// MapPoint.h mId).  The query-side state — connected keyframes, covisibility lists, the map — is filled by oracle/ref_kfdb_wrap.cpp.
// cslam/Database.h, config.h, estd.h, ORBVocabulary.h and the DBoW2 headers are the reference's own.
#ifndef CCM_REF_STUB_DB_CSLAM_H
#define CCM_REF_STUB_DB_CSLAM_H
#include <boost/shared_ptr.hpp>

#include <map>
#include <set>
#include <vector>

#include <cslam/ORBVocabulary.h>
#include <cslam/config.h>
#include <cslam/estd.h>
#include <thirdparty/DBoW2/DBoW2/BowVector.h>

namespace cslam {
using estd::idpair;
class KeyFrame;
class Map {
 public:
  typedef boost::shared_ptr<KeyFrame> kfptr;
  std::set<size_t> msuAssClients;
  std::map<idpair, kfptr> mmpKeyFrames;
  std::map<idpair, kfptr> GetMmpKeyFrames() { return mmpKeyFrames; }
};
class KeyFrame {
 public:
  typedef boost::shared_ptr<KeyFrame> kfptr;
  typedef boost::shared_ptr<Map> mapptr;
  KeyFrame()
      : mLoopQuery(defpair), mMatchQuery(defpair), mnLoopWords(0), mLoopScore(0.f), mRelocQuery(defpair), mnRelocWords(0), mRelocScore(0.f) {}
  mapptr GetMapptr() { return mpMap; }
  std::set<kfptr> GetConnectedKeyFrames() { return mspConnected; }
  std::vector<kfptr> GetBestCovisibilityKeyFrames(const int& N) {
    return (int)mvpCovis.size() > N ? std::vector<kfptr>(mvpCovis.begin(), mvpCovis.begin() + N) : mvpCovis;
  }
  idpair mId;
  size_t mUniqueId;
  idpair mLoopQuery;
  idpair mMatchQuery;
  int mnLoopWords;
  float mLoopScore;
  idpair mRelocQuery;
  int mnRelocWords;
  float mRelocScore;
  DBoW2::BowVector mBowVec;
  // stand-in state
  mapptr mpMap;
  std::set<kfptr> mspConnected;
  std::vector<kfptr> mvpCovis;
};
class Frame {
 public:
  DBoW2::BowVector mBowVec;
  idpair mId;
};
class MapPoint {
 public:
  idpair mId;
};
}  // namespace cslam
#endif

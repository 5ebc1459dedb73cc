// Stand-in for cslam::LocalMapping as shim/KeyFrameCulling_shim.cpp sees it (TEST INFRASTRUCTURE): the members KeyFrameCullingV3
// (cslam/src/Mapping.cpp:771-863) reads and writes, with the reference's names, types and access (line numbers refer to
// cslam/include/cslam/Mapping.h).  params::mapping::mfRedundancyThres is a constant here, with the shipped config's value.
#ifndef CCM_REF_STUB_KC_CSLAM_MAPPING_H
#define CCM_REF_STUB_KC_CSLAM_MAPPING_H
#include <list>
#include <set>

#include <cslam/KeyFrame.h>
#include <cslam/Map.h>
#include <cslam/MapPoint.h>

namespace cslam {

typedef double fptype;                           // config.h:37

namespace params { namespace mapping {
extern fptype mfRedundancyThres;                 // config.h:234 (Mapping.RedThres: 0.98, conf/config.yaml:81); the test may set it
} }

class LocalMapping {
 public:
  typedef boost::shared_ptr<KeyFrame> kfptr;     // Mapping.h:68
  typedef boost::shared_ptr<MapPoint> mpptr;     // Mapping.h:69
  typedef boost::shared_ptr<Map> mapptr;         // Mapping.h:70

 protected:
  friend struct KcScene;
  void KeyFrameCullingV3();                      // Mapping.h:128
  mapptr mpMap;                                  // Mapping.h:144
  std::list<kfptr> mlpRecentAddedKFs;            // Mapping.h:156
  std::set<kfptr> mspKFsCheckedForCulling;       // Mapping.h:157
  size_t mAddedKfs = 0, mCulledKfs = 0;          // Mapping.h:178
};

}  // namespace cslam
#endif

// Stand-in for cslam::Map as shim/KeyFrameCulling_shim.cpp sees it (TEST INFRASTRUCTURE): GetRandKfPtr (cslam/include/cslam/Map.h:120)
// answers a scripted list of keyframes in turn instead of rand() (a null pointer once the list is used up), so that the member's pick
// and its second try are the test's choice.
#ifndef CCM_REF_STUB_KC_CSLAM_MAP_H
#define CCM_REF_STUB_KC_CSLAM_MAP_H
#include <cstddef>
#include <vector>

#include <cslam/KeyFrame.h>

namespace cslam {

class Map {
 public:
  typedef boost::shared_ptr<KeyFrame> kfptr;
  kfptr GetRandKfPtr() { return mNext < mvScript.size() ? mvScript[mNext++] : kfptr(); }   // Map.h:120
  std::vector<kfptr> mvScript;
  size_t mNext = 0;
};

}  // namespace cslam
#endif

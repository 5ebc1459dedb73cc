// Stand-in for the part of cslam/include/cslam/estd.h that shim/MapPoint_shim.cpp uses (TEST INFRASTRUCTURE): the exception type the
// reference's components throw on an infrastructure failure (estd.h:74-81).  The real header pulls in OpenCV's full interface.
#ifndef CCM_REF_STUB_MP_ESTD_H
#define CCM_REF_STUB_MP_ESTD_H
#include <exception>

namespace estd {
class infrastructure_ex : public std::exception {
 public:
  virtual const char* what() const throw() { return "EXCEPTION: Bad Infrastructure"; }
};
}  // namespace estd
#endif

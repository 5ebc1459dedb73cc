// ccm_search_and_fuse_double.cpp — the device entry point ccm_search_and_fuse doubled on the CPU for the shim tests that run without a
// device (TEST INFRASTRUCTURE): linked with -Bsymbolic into _ref/libsearch_and_fuse_shim.so, it answers the shim's call with the
// library's host entry point, which the tests hold bit for bit equal to the device (tests/test_gpu_search_and_fuse.py).
#include "ccm_b200.h"

extern "C" int ccm_search_and_fuse(const ccm_fuse_kf* kfs, int32_t n_kf, const ccm_fuse_points* pts, int32_t* best, int32_t* n_settled) {
  return ccm_search_and_fuse_host(kfs, n_kf, pts, best, n_settled);
}

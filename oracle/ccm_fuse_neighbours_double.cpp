// ccm_fuse_neighbours_double.cpp — the device entry point ccm_fuse_neighbours doubled on the CPU for the shim tests that run without
// a device (TEST INFRASTRUCTURE): linked with -Bsymbolic into _ref/libfuse_neighbours_shim.so, it answers the shim's call with the
// library's host entry point, which the tests hold bit for bit equal to the device (tests/test_gpu_fuse_neighbours.py).
#include "ccm_b200.h"

extern "C" int ccm_fuse_neighbours(const ccm_fuse_kf* cur, const ccm_fuse_kf* targets, int32_t n_targets, const ccm_fuse_points* pts,
                                   const int32_t* cur_point, const int32_t* cand, int32_t n_cand, int32_t* fwd_best, int32_t* bwd_best,
                                   int32_t* n_settled) {
  return ccm_fuse_neighbours_host(cur, targets, n_targets, pts, cur_point, cand, n_cand, fwd_best, bwd_best, n_settled);
}

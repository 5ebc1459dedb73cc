// ccm_normal_depth_double.cpp — TEST INFRASTRUCTURE: a CPU double of the device entry point ccm_normal_depth (include/ccm_b200.h),
// so that shim/MapPoint_shim.cpp can be linked and run without a GPU.  The values come from the oracle (normal_depth_oracle.cpp);
// ccm_normal_depth_host stays the product library's own.  Linked with -Bsymbolic in front of libccm_b200.so (oracle/Makefile).
#include <cstdint>

#include "ccm_b200.h"

extern "C" int orc_normal_depth(int32_t n_kf, const float* kf_centre, const uint8_t* kf_bad, int32_t n_mp, const float* mp_pos,
                                const int64_t* obs_ptr, const int32_t* obs_kf, const int32_t* mp_ref, const float* mp_scale_ref,
                                const float* mp_scale_last, float* normal, float* max_dist, float* min_dist, uint8_t* status);

static int g_device_calls = 0;

extern "C" int ccm_normal_depth(int32_t n_kf, const float* kf_centre, const uint8_t* kf_bad, int32_t n_mp, const float* mp_pos,
                                const int64_t* obs_ptr, const int32_t* obs_kf, const int32_t* mp_ref, const float* mp_scale_ref,
                                const float* mp_scale_last, float* normal, float* max_dist, float* min_dist, uint8_t* status) {
  g_device_calls++;
  return orc_normal_depth(n_kf, kf_centre, kf_bad, n_mp, mp_pos, obs_ptr, obs_kf, mp_ref, mp_scale_ref, mp_scale_last, normal, max_dist,
                          min_dist, status) == 0 ? CCM_OK : CCM_ERR_INVALID;
}

extern "C" int nd_double_device_calls() { return g_device_calls; }

// ccm_sim3_correction_double.cpp — TEST INFRASTRUCTURE: a CPU double of the device entry point ccm_sim3_correction (include/ccm_b200.h),
// so that shim/Sim3Correction_shim.cpp runs on a machine without a GPU: the flat oracle (orc_sim3_correction of liboracle.so) answers the call.
// Linked with -Bsymbolic into the shim test library ahead of libccm_b200.so; the GPU suite links the real entry point instead.
#include <cstdint>

#include "ccm_b200.h"

extern "C" int orc_sim3_correction(int32_t, const float*, const uint8_t*, int32_t, const int32_t*, const double*, const double*, const int64_t*,
                                   const int32_t*, int32_t, const float*, const uint8_t*, const int64_t*, const int32_t*, const int32_t*,
                                   const float*, const float*, float*, float*, int32_t*, float*, float*, float*, float*, uint8_t*);

static unsigned long long g_calls = 0;
extern "C" unsigned long long sc_double_device_calls() { return g_calls; }

extern "C" int ccm_sim3_correction(int32_t n_kf, const float* kf_centre, const uint8_t* kf_bad, int32_t n_e, const int32_t* entry_kf,
                                   const double* entry_Siw_new, const double* entry_Siw_old, const int64_t* slot_ptr, const int32_t* slot_mp,
                                   int32_t n_mp, const float* mp_pos, const uint8_t* mp_skip, const int64_t* obs_ptr, const int32_t* obs_kf,
                                   const int32_t* mp_ref, const float* mp_scale_ref, const float* mp_scale_last, float* entry_Tcw,
                                   float* entry_centre, int32_t* mp_entry, float* mp_pos_out, float* normal, float* max_dist, float* min_dist,
                                   uint8_t* status) {
  g_calls++;
  return orc_sim3_correction(n_kf, kf_centre, kf_bad, n_e, entry_kf, entry_Siw_new, entry_Siw_old, slot_ptr, slot_mp, n_mp, mp_pos, mp_skip,
                             obs_ptr, obs_kf, mp_ref, mp_scale_ref, mp_scale_last, entry_Tcw, entry_centre, mp_entry, mp_pos_out, normal,
                             max_dist, min_dist, status) == 0 ? CCM_OK : CCM_ERR_INVALID;
}

// ccm_keyframe_culling_double.cpp — the device entry point ccm_keyframe_culling doubled on the CPU for the shim tests that run without
// a device (TEST INFRASTRUCTURE): linked with -Bsymbolic into _ref/libkeyframe_culling_shim.so, it answers the shim's call with the
// library's host entry point, which the tests hold bit for bit equal to the device (tests/test_gpu_keyframe_culling.py).
#include "ccm_b200.h"

extern "C" int ccm_keyframe_culling(int32_t n_kf, const uint8_t* kf_bad, int32_t n_c, const int32_t* cand_kf, const uint8_t* cand_not_erase,
                                    const int64_t* slot_ptr, const int32_t* slot_mp, const int32_t* slot_octave, int32_t n_mp,
                                    const uint8_t* mp_bad, const int32_t* mp_nobs, const int32_t* mp_ref, const int64_t* obs_ptr,
                                    const int32_t* obs_kf, const int32_t* obs_octave, int32_t th_obs, double red_thres, uint8_t* cull,
                                    int32_t* n_mps, int32_t* n_red, int32_t* n_settled) {
  return ccm_keyframe_culling_host(n_kf, kf_bad, n_c, cand_kf, cand_not_erase, slot_ptr, slot_mp, slot_octave, n_mp, mp_bad, mp_nobs, mp_ref,
                                   obs_ptr, obs_kf, obs_octave, th_obs, red_thres, cull, n_mps, n_red, n_settled);
}

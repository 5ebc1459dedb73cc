// ccm_covis_double.cpp — TEST INFRASTRUCTURE: a CPU double of the device entry point ccm_covisibility (include/ccm_b200.h), so that
// shim/KeyFrameConnections_shim.cpp can be linked and run without a GPU.  The values come from the oracle (covis_oracle.cpp);
// ccm_covisibility_host stays the product library's own.  Linked with -Bsymbolic in front of libccm_b200.so (oracle/Makefile).
#include <cstdint>

#include "ccm_b200.h"

extern "C" int orc_covisibility(int32_t n_kf, const uint64_t* kf_id, const uint32_t* kf_rank, int32_t n_b, const int32_t* batch,
                                const int64_t* kf_mp_ptr, const int32_t* kf_mp, int32_t n_mp, const uint8_t* mp_bad, const int64_t* obs_ptr,
                                const int32_t* obs_kf, int32_t th, int64_t capacity, int64_t* conn_ptr, int32_t* conn_kf, int32_t* conn_w,
                                int32_t* n_sel, int32_t* sel_kf, int32_t* sel_w, uint8_t* status, int64_t* total);

static int g_device_calls = 0;

extern "C" int ccm_covisibility(int32_t n_kf, const uint64_t* kf_id, const uint32_t* kf_rank, int32_t n_b, const int32_t* batch,
                                const int64_t* kf_mp_ptr, const int32_t* kf_mp, int32_t n_mp, const uint8_t* mp_bad, const int64_t* obs_ptr,
                                const int32_t* obs_kf, int32_t th, int64_t capacity, int64_t* conn_ptr, int32_t* conn_kf, int32_t* conn_w,
                                int32_t* n_sel, int32_t* sel_kf, int32_t* sel_w, uint8_t* status, int64_t* total) {
  g_device_calls++;
  return orc_covisibility(n_kf, kf_id, kf_rank, n_b, batch, kf_mp_ptr, kf_mp, n_mp, mp_bad, obs_ptr, obs_kf, th, capacity, conn_ptr, conn_kf,
                          conn_w, n_sel, sel_kf, sel_w, status, total) == 0
             ? CCM_OK
             : CCM_ERR_INVALID;
}

extern "C" int cv_double_device_calls() { return g_device_calls; }

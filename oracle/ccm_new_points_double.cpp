// ccm_new_points_double.cpp — TEST INFRASTRUCTURE: a CPU double of the device entry point ccm_new_map_points (include/ccm_b200.h), so
// that shim/NewMapPoints_shim.cpp can be linked and run without a GPU.  The values come from the sequential oracle
// (new_points_oracle.cpp).  Linked with -Bsymbolic in front of libccm_b200.so (oracle/new_points.mk).
#include <cstdint>

#include "ccm_b200.h"

extern "C" int orc_new_map_points(const ccm_newpts_view* cur, const ccm_newpts_neighbour* nb, int32_t n_nb, ccm_new_point* out,
                                  int32_t capacity, int32_t* n_out, int32_t* best2, uint8_t* verdict, int32_t mutate);

static int g_device_calls = 0;

extern "C" int ccm_new_map_points(const ccm_newpts_view* cur, const ccm_newpts_neighbour* nb, int32_t n_nb, ccm_new_point* out,
                                  int32_t capacity, int32_t* n_out, int32_t* best2, uint8_t* verdict) {
  g_device_calls++;
  return orc_new_map_points(cur, nb, n_nb, out, capacity, n_out, best2, verdict, 0) == 0 ? CCM_OK : CCM_ERR_INVALID;
}

extern "C" int np_double_device_calls() { return g_device_calls; }

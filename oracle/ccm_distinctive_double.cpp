// ccm_distinctive_double.cpp — TEST INFRASTRUCTURE: CPU doubles of the device entry points ccm_distinctive_descriptors and
// ccm_kfstore_distinctive_descriptors (include/ccm_b200.h), so that shim/MapPointDescriptor_shim.cpp can be linked and run without a
// GPU.  The values come from the oracle (distinctive_oracle.cpp); ccm_distinctive_descriptors_host stays the product library's own.
// The store double holds descriptors put through dd_double_store_put under their uid; any non-null ccm_kf_store* names it.
// Linked with -Bsymbolic in front of libccm_b200.so (oracle/Makefile).
#include <cstddef>
#include <cstdint>
#include <map>
#include <vector>

#include "ccm_b200.h"

extern "C" int orc_distinctive_descriptors(int32_t n_kf, const uint8_t* kf_bad, int32_t n_mp, const int64_t* obs_ptr, const int32_t* obs_kf,
                                           const uint8_t* obs_desc, int32_t* best, int32_t* best_median, uint8_t* desc_out);

static int g_device_calls = 0, g_store_calls = 0;
static std::map<uint64_t, std::vector<uint8_t> > g_store;

extern "C" int ccm_distinctive_descriptors(int32_t n_kf, const uint8_t* kf_bad, int32_t n_mp, const int64_t* obs_ptr, const int32_t* obs_kf,
                                           const uint8_t* obs_desc, int32_t* best, int32_t* best_median, uint8_t* desc_out) {
  g_device_calls++;
  return orc_distinctive_descriptors(n_kf, kf_bad, n_mp, obs_ptr, obs_kf, obs_desc, best, best_median, desc_out) == 0 ? CCM_OK : CCM_ERR_INVALID;
}

extern "C" int ccm_kfstore_distinctive_descriptors(ccm_kf_store* store, int32_t n_kf, const uint64_t* kf_uid, const uint8_t* kf_bad, int32_t n_mp,
                                                   const int64_t* obs_ptr, const int32_t* obs_kf, const int32_t* obs_feat, int32_t* best,
                                                   int32_t* best_median, uint8_t* desc_out) {
  g_store_calls++;
  if (!store || n_mp < 0) return CCM_ERR_INVALID;
  const int64_t E = n_mp ? obs_ptr[n_mp] : 0;
  std::vector<uint8_t> desc((size_t)E * 32 + 32, 0);
  for (int64_t j = 0; j < E; j++) {
    if (obs_kf[j] < 0 || obs_kf[j] >= n_kf) return CCM_ERR_INVALID;
    if (kf_bad[obs_kf[j]]) continue;
    std::map<uint64_t, std::vector<uint8_t> >::const_iterator it = g_store.find(kf_uid[obs_kf[j]]);
    if (it == g_store.end() || obs_feat[j] < 0 || (size_t)obs_feat[j] * 32 >= it->second.size()) return CCM_ERR_INVALID;
    for (int b = 0; b < 32; b++) desc[32 * j + b] = it->second[32 * (size_t)obs_feat[j] + b];
  }
  return orc_distinctive_descriptors(n_kf, kf_bad, n_mp, obs_ptr, obs_kf, desc.data(), best, best_median, desc_out) == 0 ? CCM_OK
                                                                                                                         : CCM_ERR_INVALID;
}

extern "C" void dd_double_store_put(uint64_t uid, int32_t n, const uint8_t* desc) { g_store[uid].assign(desc, desc + 32 * (size_t)n); }
extern "C" void dd_double_store_clear() { g_store.clear(); }
extern "C" int dd_double_device_calls() { return g_device_calls; }
extern "C" int dd_double_store_calls() { return g_store_calls; }

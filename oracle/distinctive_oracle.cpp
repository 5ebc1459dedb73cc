// distinctive_oracle.cpp — TEST INFRASTRUCTURE: the checker's own restatement of MapPoint::ComputeDistinctiveDescriptors
// (cslam/src/MapPoint.cpp:929-994) over the flat arrays of ccm_distinctive_descriptors (include/ccm_b200.h).  Written from the
// reference body, not from the product's distinctive.cu: every row of the N x N distance matrix is built and sorted in full, the
// median is element (N-1)/2 of the sorted row, the first strictly smaller median wins.  Rows are kept one at a time (any N).
#include <algorithm>
#include <climits>
#include <cstdint>
#include <cstring>
#include <vector>

// ORBmatcher::DescriptorDistance (cslam/src/ORBmatcher.cpp:1653-1669): popcount of the xor, 8 words of 32 bits
static int hamming256(const uint8_t* a, const uint8_t* b) {
  int d = 0;
  for (int i = 0; i < 32; i++) {
    unsigned x = (unsigned)(a[i] ^ b[i]);
    while (x) { d += (int)(x & 1u); x >>= 1; }
  }
  return d;
}

extern "C" int orc_distinctive_descriptors(int32_t n_kf, const uint8_t* kf_bad, int32_t n_mp, const int64_t* obs_ptr, const int32_t* obs_kf,
                                           const uint8_t* obs_desc, int32_t* best, int32_t* best_median, uint8_t* desc_out) {
  if (n_kf < 0 || n_mp < 0) return -1;
  for (int32_t i = 0; i < n_mp; i++)
    for (int64_t j = obs_ptr[i]; j < obs_ptr[i + 1]; j++)
      if (obs_kf[j] < 0 || obs_kf[j] >= n_kf) return -1;
  std::vector<int64_t> pos;
  std::vector<int> row;
  for (int32_t i = 0; i < n_mp; i++) {
    pos.clear();
    for (int64_t j = obs_ptr[i]; j < obs_ptr[i + 1]; j++)
      if (!kf_bad[obs_kf[j]]) pos.push_back(j);                      // if(!pKF->isBad()) vDescriptors.push_back(...)
    const size_t N = pos.size();
    int32_t b = -1, m = 0;
    if (N) {
      int best_median_v = INT_MAX;
      size_t best_idx = 0;
      row.resize(N);
      for (size_t a = 0; a < N; a++) {
        for (size_t c = 0; c < N; c++) row[c] = a == c ? 0 : hamming256(obs_desc + 32 * pos[a], obs_desc + 32 * pos[c]);
        std::sort(row.begin(), row.end());
        const int median = row[(N - 1) / 2];
        if (median < best_median_v) { best_median_v = median; best_idx = a; }
      }
      b = (int32_t)(pos[best_idx] - obs_ptr[i]); m = best_median_v;
    }
    best[i] = b;
    if (best_median) best_median[i] = m;
    if (desc_out) {
      if (b >= 0) std::memcpy(desc_out + 32 * (size_t)i, obs_desc + 32 * (obs_ptr[i] + b), 32);
      else std::memset(desc_out + 32 * (size_t)i, 0, 32);
    }
  }
  return 0;
}

// covis_oracle.cpp — TEST INFRASTRUCTURE: our restatement of the counting and the two orders of KeyFrame::UpdateConnections
// (cslam/src/KeyFrame.cpp:629-711) over the flat arrays of include/ccm_b200.h's ccm_covisibility, written independently of
// ccm_slam_b200/csrc/covis.cu: a std::map keyed by rank plays KFcounter, the selection is std::sort over (weight, rank) pairs read
// back from the end, and pKFmax is found by the reference's own strict-maximum scan.  Same signature and outputs as the product entry
// points; returns 0, -1 on bad input, -2 when capacity is below the total (written to *total).
#include <algorithm>
#include <cstdint>
#include <map>
#include <utility>
#include <vector>

extern "C" int orc_covisibility(int32_t n_kf, const uint64_t* kf_id, const uint32_t* kf_rank, int32_t n_b, const int32_t* batch,
                                const int64_t* kf_mp_ptr, const int32_t* kf_mp, int32_t n_mp, const uint8_t* mp_bad, const int64_t* obs_ptr,
                                const int32_t* obs_kf, int32_t th, int64_t capacity, int64_t* conn_ptr, int32_t* conn_kf, int32_t* conn_w,
                                int32_t* n_sel, int32_t* sel_kf, int32_t* sel_w, uint8_t* status, int64_t* total) {
  if (n_kf < 0 || n_b < 0 || n_mp < 0) return -1;
  std::vector<int32_t> row_of(n_kf, -1);
  for (int32_t k = 0; k < n_kf; k++) {
    if (kf_rank[k] >= (uint32_t)n_kf || row_of[kf_rank[k]] >= 0) return -1;
    row_of[kf_rank[k]] = k;
  }
  std::vector<std::map<uint32_t, int> > counters(n_b);
  int64_t T = 0;
  for (int32_t b = 0; b < n_b; b++) {
    const int32_t self = batch[b];
    if (self < 0 || self >= n_kf) return -1;
    std::map<uint32_t, int>& KFcounter = counters[b];
    for (int64_t j = kf_mp_ptr[b]; j < kf_mp_ptr[b + 1]; j++) {
      const int32_t p = kf_mp[j];
      if (p < -1 || p >= n_mp) return -1;
      if (p == -1 || mp_bad[p]) continue;
      for (int64_t q = obs_ptr[p]; q < obs_ptr[p + 1]; q++) {
        const int32_t k = obs_kf[q];
        if (k < 0 || k >= n_kf) return -1;
        if (kf_id[k] != kf_id[self]) KFcounter[kf_rank[k]]++;
      }
    }
    T += (int64_t)KFcounter.size();
  }
  *total = T;
  if (capacity < T) return -2;
  int64_t at = 0;
  conn_ptr[0] = 0;
  for (int32_t b = 0; b < n_b; b++) {
    const std::map<uint32_t, int>& KFcounter = counters[b];
    int nmax = 0;
    int32_t pKFmax = -1;
    std::vector<std::pair<int, uint32_t> > vPairs;
    const int64_t base = at;
    for (std::map<uint32_t, int>::const_iterator mit = KFcounter.begin(); mit != KFcounter.end(); ++mit, ++at) {
      conn_kf[at] = row_of[mit->first];
      conn_w[at] = mit->second;
      sel_kf[at] = -1;
      sel_w[at] = 0;
      if (mit->second > nmax) { nmax = mit->second; pKFmax = row_of[mit->first]; }
      if (mit->second >= th) vPairs.push_back(std::make_pair(mit->second, mit->first));
    }
    conn_ptr[b + 1] = at;
    status[b] = KFcounter.empty() ? 0 : 1;
    if (KFcounter.empty()) { n_sel[b] = 0; continue; }
    if (vPairs.empty()) {
      sel_kf[base] = pKFmax;
      sel_w[base] = nmax;
      n_sel[b] = 1;
      continue;
    }
    std::sort(vPairs.begin(), vPairs.end());
    for (size_t i = 0; i < vPairs.size(); i++) {
      const std::pair<int, uint32_t>& e = vPairs[vPairs.size() - 1 - i];
      sel_kf[base + i] = row_of[e.second];
      sel_w[base + i] = e.first;
    }
    n_sel[b] = (int32_t)vPairs.size();
  }
  return 0;
}

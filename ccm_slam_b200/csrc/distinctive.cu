// distinctive.cu — map-point descriptors, behind ccm_distinctive_descriptors / ccm_distinctive_descriptors_host /
// ccm_kfstore_distinctive_descriptors (include/ccm_b200.h).
//
//   MapPoint::ComputeDistinctiveDescriptors   cslam/src/MapPoint.cpp:929-994
//
// Per point: the observers that are not bad, in the order given, form D (N rows of 32 bytes); d(i,j) is the 256-bit Hamming distance;
// row i's median is the ((N-1)/2)-th smallest of d(i, 0..N-1) (d(i,i) = 0 included, the lower middle for even N); the chosen row is
// the first with the strictly smallest median.  Everything is an integer: the device, the host entry point and the reference agree
// exactly or not at all.
//
// Shape.  k_dd_classify counts each point's survivors, checks its rows, writes the untouched points (N = 0) and scatters the others'
// ids into three lists by N:
//   N <= 32     k_dd_warp: one warp per point; lane i holds row i in 8 registers, d(i,j) comes from 8 shuffles and 8 popcounts and
//               goes to a 32 x 32 shared tile; lane i then bisects its column for the median.
//   N <= 1024   k_dd_cta: one CTA per point, the survivors' rows and list positions staged in shared memory (36 KB);
//   N > 1024    k_dd_cta again, the rows read from global memory (through L1/L2) at their list positions, bad observers skipped inline.
// In the CTA path thread i finds row i's median by a 9-step bisection on the value (distances lie in 0..256): count d(i,j) <= v,
// recomputing the popcounts on each pass, so no row is stored.  The first minimum is a min-reduction over the key
// median << 32 | position: positions grow with the survivor index, so the smallest key is the reference's BestIdx whatever the schedule.
// Results are written back by point id; the list order (atomics) does not reach them.
#include <climits>
#include <string>
#include <vector>

#include "common.cuh"

using namespace ccm;

namespace ccm {
// kf_store.cu: the device address of each uid's first descriptor and its feature count (nullptr / -1: the store does not hold the uid)
void kfstore_resolve(ccm_kf_store* s, int32_t n, const uint64_t* uid, std::vector<const uint4*>& base, std::vector<int32_t>& n_feat,
                     int* device);
}  // namespace ccm

namespace {

constexpr int WARP_MAX = 32;     // N <= WARP_MAX: k_dd_warp
constexpr int STAGE_MAX = 1024;  // N <= STAGE_MAX: k_dd_cta with the rows in shared memory
constexpr int CTA = 256;
constexpr unsigned FULL = 0xffffffffu;
constexpr int32_t NO_BAD = 0x7f7f7f7f;  // the bad-point slot's initial value (a byte memset): larger than any point id

// where observation j's descriptor lives: 32 bytes uploaded with the call ...
struct FromHost {
  const uint4* desc;
  const int32_t* obs_kf;
  __device__ bool ok(int64_t, int32_t) const { return true; }
  __device__ const uint4* row(int64_t j) const { return desc + 2 * j; }
};
// ... or feature obs_feat[j] of keyframe row obs_kf[j] in the store's slabs
struct FromStore {
  const uint4* const* base;
  const int32_t* n_feat;
  const int32_t* feat;
  const int32_t* obs_kf;
  __device__ bool ok(int64_t j, int32_t k) const { return feat[j] >= 0 && feat[j] < n_feat[k]; }
  __device__ const uint4* row(int64_t j) const { return base[obs_kf[j]] + 2 * (size_t)feat[j]; }
};

__device__ __forceinline__ int dist(const uint4& a0, const uint4& a1, const uint4& b0, const uint4& b1) {
  return __popc(a0.x ^ b0.x) + __popc(a0.y ^ b0.y) + __popc(a0.z ^ b0.z) + __popc(a0.w ^ b0.w) + __popc(a1.x ^ b1.x) + __popc(a1.y ^ b1.y) +
         __popc(a1.z ^ b1.z) + __popc(a1.w ^ b1.w);
}

__device__ __forceinline__ unsigned long long warp_min(unsigned long long v) {
#pragma unroll
  for (int o = 16; o; o >>= 1) v = min(v, __shfl_xor_sync(FULL, v, o));
  return v;
}

__device__ __forceinline__ void write_untouched(int p, int32_t* best, int32_t* median, uint4* desc_out) {
  best[p] = -1; median[p] = 0;
  desc_out[2 * (size_t)p] = make_uint4(0, 0, 0, 0); desc_out[2 * (size_t)p + 1] = make_uint4(0, 0, 0, 0);
}

// survivors of every point, the range checks (*bad_point = the smallest failing point id; it is then left out of every list), the
// untouched points, and the three lists (lists[c * n ..], counts[c])
template <class Src>
__global__ void __launch_bounds__(CTA) k_dd_classify(int n, int n_kf, const uint8_t* __restrict__ kf_bad, const int64_t* __restrict__ obs_ptr,
                                                     const int32_t* __restrict__ obs_kf, Src src, int32_t* __restrict__ n_surv,
                                                     int32_t* __restrict__ lists, int32_t* __restrict__ counts, int32_t* __restrict__ bad_point,
                                                     int32_t* __restrict__ best, int32_t* __restrict__ median, uint4* __restrict__ desc_out) {
  const int lane = threadIdx.x & 31;
  for (int base = blockIdx.x * CTA; base < n; base += gridDim.x * CTA) {   // uniform per block: the ballots below see full warps
    const int i = base + threadIdx.x;
    int cls = -1;
    if (i < n) {
      int N = 0;
      bool ok = true;
      for (int64_t j = obs_ptr[i]; j < obs_ptr[i + 1]; j++) {
        const int32_t k = obs_kf[j];
        if ((unsigned)k >= (unsigned)n_kf) { ok = false; break; }
        if (kf_bad[k]) continue;                                   // if(!pKF->isBad()) vDescriptors.push_back(...)
        if (!src.ok(j, k)) { ok = false; break; }
        N++;
      }
      if (!ok) { atomicMin(bad_point, i); N = 0; }
      n_surv[i] = N;
      if (N == 0) {
        if (ok) write_untouched(i, best, median, desc_out);
      } else {
        cls = N <= WARP_MAX ? 0 : N <= STAGE_MAX ? 1 : 2;
      }
    }
#pragma unroll
    for (int c = 0; c < 3; c++) {
      const unsigned m = __ballot_sync(FULL, cls == c);
      if (!m) continue;
      const int leader = __ffs(m) - 1;
      int off = 0;
      if (lane == leader) off = atomicAdd(&counts[c], __popc(m));
      off = __shfl_sync(FULL, off, leader);
      if (cls == c) lists[(size_t)c * n + off + __popc(m & ((1u << lane) - 1))] = i;
    }
  }
}

// N <= 32: one warp per point.  The minimum of 4 CTAs per SM (17 KB of shared memory each) lifts ptxas's register target from 32,
// where it spilled one word, to 64.
template <class Src>
__global__ void __launch_bounds__(CTA, 4) k_dd_warp(const int32_t* __restrict__ list, const int32_t* __restrict__ count,
                                                 const uint8_t* __restrict__ kf_bad, const int64_t* __restrict__ obs_ptr,
                                                 const int32_t* __restrict__ obs_kf, Src src, const int32_t* __restrict__ n_surv,
                                                 int32_t* __restrict__ best, int32_t* __restrict__ median, uint4* __restrict__ desc_out) {
  constexpr int W = CTA / 32;
  __shared__ uint16_t sd[W][32 * 32];   // d(i, j) at [j * 32 + i]: lane i reads its own column, conflict-free
  __shared__ int32_t spos[W][32];       // survivor i's position in the caller's list
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const unsigned lt = (1u << lane) - 1;
  const int m = *count;
  for (int t = blockIdx.x * W + w; t < m; t += gridDim.x * W) {   // uniform per warp
    const int p = list[t];
    const int64_t b = obs_ptr[p], e = obs_ptr[p + 1];
    const int N = n_surv[p];
    int got = 0;
    for (int64_t c0 = b; c0 < e; c0 += 32) {
      const int64_t j = c0 + lane;
      const bool keep = j < e && !kf_bad[obs_kf[j]];
      const unsigned mk = __ballot_sync(FULL, keep);
      if (keep) spos[w][got + __popc(mk & lt)] = (int32_t)(j - b);
      got += __popc(mk);
    }
    __syncwarp();
    uint4 a0 = make_uint4(0, 0, 0, 0), a1 = a0;
    if (lane < N) { const uint4* r = src.row(b + spos[w][lane]); a0 = r[0]; a1 = r[1]; }
    for (int j = 0; j < N; j++) {
      uint4 b0, b1;
      b0.x = __shfl_sync(FULL, a0.x, j); b0.y = __shfl_sync(FULL, a0.y, j); b0.z = __shfl_sync(FULL, a0.z, j); b0.w = __shfl_sync(FULL, a0.w, j);
      b1.x = __shfl_sync(FULL, a1.x, j); b1.y = __shfl_sync(FULL, a1.y, j); b1.z = __shfl_sync(FULL, a1.z, j); b1.w = __shfl_sync(FULL, a1.w, j);
      sd[w][j * 32 + lane] = (uint16_t)dist(a0, a1, b0, b1);
    }
    __syncwarp();
    unsigned long long key = ~0ull;
    if (lane < N) {
      const int k = (N - 1) / 2;                                   // vDists[0.5*(N-1)]
      int lo = 0, hi = 256;
      while (lo < hi) {                                            // smallest v with #{j : d(i,j) <= v} > k
        const int mid = (lo + hi) >> 1;
        int c = 0;
        for (int j = 0; j < N; j++) c += sd[w][j * 32 + lane] <= mid;
        if (c > k) hi = mid; else lo = mid + 1;
      }
      key = (unsigned long long)lo << 32 | (unsigned)lane;
    }
    key = warp_min(key);
    const int bi = (int)(key & 0xffffffffu);
    if (lane == bi) {
      best[p] = spos[w][bi]; median[p] = (int32_t)(key >> 32);
      desc_out[2 * (size_t)p] = a0; desc_out[2 * (size_t)p + 1] = a1;
    }
    __syncwarp();                                                  // spos / sd are refilled for the next point
  }
}

// N > 32: one CTA per point; rows staged in shared memory up to STAGE_MAX, read in place beyond
template <class Src>
__global__ void __launch_bounds__(CTA) k_dd_cta(const int32_t* __restrict__ list_mid, const int32_t* __restrict__ list_big,
                                                const int32_t* __restrict__ counts, const uint8_t* __restrict__ kf_bad,
                                                const int64_t* __restrict__ obs_ptr, const int32_t* __restrict__ obs_kf, Src src,
                                                const int32_t* __restrict__ n_surv, int32_t* __restrict__ best, int32_t* __restrict__ median,
                                                uint4* __restrict__ desc_out) {
  __shared__ uint4 sdesc[2 * STAGE_MAX];
  __shared__ int32_t spos[STAGE_MAX];
  __shared__ int32_t wsum[CTA / 32];
  __shared__ unsigned long long wkey[CTA / 32];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const int n_mid = counts[1], n_all = n_mid + counts[2];
  for (int t = blockIdx.x; t < n_all; t += gridDim.x) {            // uniform per block
    const int p = t < n_mid ? list_mid[t] : list_big[t - n_mid];
    const int64_t b = obs_ptr[p], e = obs_ptr[p + 1];
    const int N = n_surv[p], k = (N - 1) / 2;
    const bool staged = N <= STAGE_MAX;
    unsigned long long key = ~0ull;
    if (staged) {
      int got = 0;
      for (int64_t c0 = b; c0 < e; c0 += CTA) {
        const int64_t j = c0 + threadIdx.x;
        const bool keep = j < e && !kf_bad[obs_kf[j]];
        const unsigned mk = __ballot_sync(FULL, keep);
        if (lane == 0) wsum[w] = __popc(mk);
        __syncthreads();
        int off = got, tot = 0;
        for (int q = 0; q < CTA / 32; q++) { off += q < w ? wsum[q] : 0; tot += wsum[q]; }
        if (keep) {
          const int r = off + __popc(mk & ((1u << lane) - 1));
          const uint4* row = src.row(j);
          spos[r] = (int32_t)(j - b); sdesc[2 * r] = row[0]; sdesc[2 * r + 1] = row[1];
        }
        got += tot;
        __syncthreads();
      }
      for (int i = threadIdx.x; i < N; i += CTA) {
        const uint4 a0 = sdesc[2 * i], a1 = sdesc[2 * i + 1];
        int lo = 0, hi = 256;
        while (lo < hi) {
          const int mid = (lo + hi) >> 1;
          int c = 0;
          for (int j = 0; j < N && c <= k; j++) c += dist(a0, a1, sdesc[2 * j], sdesc[2 * j + 1]) <= mid;
          if (c > k) hi = mid; else lo = mid + 1;
        }
        key = min(key, (unsigned long long)lo << 32 | (unsigned)spos[i]);
      }
    } else {
      for (int64_t q = b + threadIdx.x; q < e; q += CTA) {
        if (kf_bad[obs_kf[q]]) continue;
        const uint4* ra = src.row(q);
        const uint4 a0 = ra[0], a1 = ra[1];
        int lo = 0, hi = 256;
        while (lo < hi) {
          const int mid = (lo + hi) >> 1;
          int c = 0;
          for (int64_t j = b; j < e && c <= k; j++) {
            if (kf_bad[obs_kf[j]]) continue;
            const uint4* rb = src.row(j);
            c += dist(a0, a1, rb[0], rb[1]) <= mid;
          }
          if (c > k) hi = mid; else lo = mid + 1;
        }
        key = min(key, (unsigned long long)lo << 32 | (unsigned)(q - b));
      }
    }
    key = warp_min(key);
    if (lane == 0) wkey[w] = key;
    __syncthreads();
    if (threadIdx.x == 0) {
      for (int q = 1; q < CTA / 32; q++) key = min(key, wkey[q]);
      const int pos = (int)(key & 0xffffffffu);
      best[p] = pos; median[p] = (int32_t)(key >> 32);
      const uint4* row = src.row(b + pos);
      desc_out[2 * (size_t)p] = row[0]; desc_out[2 * (size_t)p + 1] = row[1];
    }
    __syncthreads();                                               // sdesc / spos / wkey are refilled for the next point
  }
}

void check_shape(const std::string& f, int32_t n_kf, const uint8_t* kf_bad, int32_t n_mp, const int64_t* obs_ptr, const int32_t* obs_kf,
                 const void* obs_data, int32_t* best) {
  CCM_REQUIRE(n_kf >= 0 && n_mp >= 0, f + ": negative size");
  CCM_REQUIRE(n_kf == 0 || kf_bad, f + ": null kf_bad");
  CCM_REQUIRE(n_mp == 0 || (obs_ptr && best), f + ": null point array");
  if (n_mp == 0) return;
  CCM_REQUIRE(obs_ptr[0] == 0, f + ": obs_ptr[0] must be 0");
  for (int32_t i = 0; i < n_mp; i++) CCM_REQUIRE(obs_ptr[i + 1] >= obs_ptr[i], f + ": obs_ptr is not monotone");
  CCM_REQUIRE(obs_ptr[n_mp] == 0 || (obs_kf && obs_data), f + ": null observation array");
  for (int32_t i = 0; i < n_mp; i++) CCM_REQUIRE(obs_ptr[i + 1] - obs_ptr[i] <= INT32_MAX, f + ": more than 2^31 observers of one point");
}

inline int popc_host(uint32_t x) { return __builtin_popcount(x); }

// the message for the smallest failing point, found again on the host (n_feat == nullptr: the host-buffer variant)
std::string bad_point_message(const std::string& f, int32_t p, int32_t n_kf, const uint8_t* kf_bad, const int64_t* obs_ptr,
                              const int32_t* obs_kf, const int32_t* obs_feat, const int32_t* n_feat, const uint64_t* kf_uid) {
  for (int64_t j = obs_ptr[p]; j < obs_ptr[p + 1]; j++) {
    const int32_t k = obs_kf[j];
    const std::string at = f + ": point " + std::to_string(p) + ", observer " + std::to_string(j - obs_ptr[p]);
    if (k < 0 || k >= n_kf) return at + ": keyframe row " + std::to_string(k) + " out of range";
    if (kf_bad[k] || !n_feat) continue;
    if (n_feat[k] < 0) return at + ": keyframe uid " + std::to_string(kf_uid[k]) + " is not in the store";
    if (obs_feat[j] < 0 || obs_feat[j] >= n_feat[k])
      return at + ": feature index " + std::to_string(obs_feat[j]) + " out of range (keyframe uid " + std::to_string(kf_uid[k]) + " has " +
             std::to_string(n_feat[k]) + ")";
  }
  return f + ": point " + std::to_string(p) + ": bad observer";
}

// classify + both compute kernels on stream s; the outputs reach the caller's buffers only when every point passed its checks
template <class Src>
void run_device(const std::string& f, cudaStream_t s, int32_t n_kf, const uint8_t* kf_bad, int32_t n_mp, const int64_t* obs_ptr,
                const int32_t* obs_kf, const int32_t* obs_feat, const int32_t* n_feat, const uint64_t* kf_uid, const DevBuf<uint8_t>& d_bad,
                const DevBuf<int64_t>& d_ptr, const DevBuf<int32_t>& d_obs, const Src& src, int32_t* best, int32_t* best_median,
                uint8_t* desc_out) {
  DevBuf<int32_t> d_nsurv, d_lists, d_best, d_med, d_counts;
  DevBuf<uint4> d_desc;
  d_nsurv.alloc(n_mp); d_lists.alloc((size_t)3 * n_mp); d_best.alloc(n_mp); d_med.alloc(n_mp); d_desc.alloc((size_t)2 * n_mp);
  d_counts.alloc(4);
  CCM_CUDA(cudaMemsetAsync(d_counts.p, 0, 3 * sizeof(int32_t), s));
  CCM_CUDA(cudaMemsetAsync(d_counts.p + 3, 0x7f, sizeof(int32_t), s));
  const int sms = sm_count();
  k_dd_classify<<<grid_size(n_mp, CTA), CTA, 0, s>>>(n_mp, n_kf, d_bad.p, d_ptr.p, d_obs.p, src, d_nsurv.p, d_lists.p,
                                                      d_counts.p, d_counts.p + 3, d_best.p, d_med.p, d_desc.p);
  CCM_LAUNCHED();
  k_dd_warp<<<grid_size(n_mp, CTA / 32), CTA, 0, s>>>(d_lists.p, d_counts.p, d_bad.p, d_ptr.p, d_obs.p, src, d_nsurv.p,
                                                      d_best.p, d_med.p, d_desc.p);
  CCM_LAUNCHED();
  k_dd_cta<<<std::min(n_mp, sms * 6), CTA, 0, s>>>(d_lists.p + n_mp, d_lists.p + 2 * (size_t)n_mp, d_counts.p, d_bad.p, d_ptr.p, d_obs.p, src,
                                                   d_nsurv.p, d_best.p, d_med.p, d_desc.p);
  CCM_LAUNCHED();
  int32_t bad = NO_BAD;
  CCM_CUDA(cudaMemcpyAsync(&bad, d_counts.p + 3, sizeof(int32_t), cudaMemcpyDeviceToHost, s));
  CCM_CUDA(cudaStreamSynchronize(s));
  if (bad != NO_BAD) throw Error(CCM_ERR_INVALID, bad_point_message(f, bad, n_kf, kf_bad, obs_ptr, obs_kf, obs_feat, n_feat, kf_uid));
  d_best.download(best, n_mp, s);
  if (best_median) d_med.download(best_median, n_mp, s);
  if (desc_out) CCM_CUDA(cudaMemcpyAsync(desc_out, d_desc.p, (size_t)n_mp * 32, cudaMemcpyDeviceToHost, s));
  CCM_CUDA(cudaStreamSynchronize(s));
}

}  // namespace

extern "C" int ccm_distinctive_descriptors_host(int32_t n_kf, const uint8_t* kf_bad, int32_t n_mp, const int64_t* obs_ptr, const int32_t* obs_kf,
                                                const uint8_t* obs_desc, int32_t* best, int32_t* best_median, uint8_t* desc_out) {
  return guarded([&] {
    const std::string f = "ccm_distinctive_descriptors_host";
    check_shape(f, n_kf, kf_bad, n_mp, obs_ptr, obs_kf, obs_desc, best);
    for (int32_t i = 0; i < n_mp; i++)
      for (int64_t j = obs_ptr[i]; j < obs_ptr[i + 1]; j++)
        if (obs_kf[j] < 0 || obs_kf[j] >= n_kf) throw Error(CCM_ERR_INVALID, bad_point_message(f, i, n_kf, kf_bad, obs_ptr, obs_kf, nullptr, nullptr, nullptr));
    std::vector<int64_t> keep;
    std::vector<uint32_t> rows;
    for (int32_t i = 0; i < n_mp; i++) {
      keep.clear(); rows.clear();
      for (int64_t j = obs_ptr[i]; j < obs_ptr[i + 1]; j++) {
        if (kf_bad[obs_kf[j]]) continue;
        keep.push_back(j);
        uint32_t w[8];
        memcpy(w, obs_desc + 32 * (size_t)j, 32);
        rows.insert(rows.end(), w, w + 8);
      }
      const int64_t N = (int64_t)keep.size();
      int32_t bi = -1, bm = 0;
      if (N) {
        const int64_t k = (N - 1) / 2;
        int64_t best_i = 0;
        int best_med = INT_MAX;
        int64_t hist[257];
        for (int64_t a = 0; a < N; a++) {                             // row a's k-th smallest from a 257-bin histogram
          memset(hist, 0, sizeof hist);
          const uint32_t* ra = &rows[8 * a];
          for (int64_t c = 0; c < N; c++) {
            const uint32_t* rc = &rows[8 * c];
            int d = 0;
            for (int q = 0; q < 8; q++) d += popc_host(ra[q] ^ rc[q]);
            hist[d]++;
          }
          int v = 0;
          for (int64_t acc = hist[0]; acc <= k; acc += hist[++v]) {}
          if (v < best_med) { best_med = v; best_i = a; }
        }
        bi = (int32_t)(keep[best_i] - obs_ptr[i]); bm = best_med;
      }
      best[i] = bi;
      if (best_median) best_median[i] = bm;
      if (desc_out) {
        if (bi >= 0) memcpy(desc_out + 32 * (size_t)i, obs_desc + 32 * (size_t)(obs_ptr[i] + bi), 32);
        else memset(desc_out + 32 * (size_t)i, 0, 32);
      }
    }
  });
}

extern "C" int ccm_distinctive_descriptors(int32_t n_kf, const uint8_t* kf_bad, int32_t n_mp, const int64_t* obs_ptr, const int32_t* obs_kf,
                                           const uint8_t* obs_desc, int32_t* best, int32_t* best_median, uint8_t* desc_out) {
  return guarded([&] {
    const std::string f = "ccm_distinctive_descriptors";
    check_shape(f, n_kf, kf_bad, n_mp, obs_ptr, obs_kf, obs_desc, best);
    ensure_device();
    if (n_mp == 0) return;
    const int64_t E = obs_ptr[n_mp];
    const CallStream g;
    DevBuf<uint8_t> d_bad;
    DevBuf<int64_t> d_ptr;
    DevBuf<int32_t> d_obs;
    DevBuf<uint4> d_desc;
    if (n_kf) d_bad.upload(kf_bad, n_kf, g.s); else d_bad.alloc(1);
    if (E) { d_obs.upload(obs_kf, (size_t)E, g.s); d_desc.alloc((size_t)2 * E);
             CCM_CUDA(cudaMemcpyAsync(d_desc.p, obs_desc, (size_t)E * 32, cudaMemcpyHostToDevice, g.s)); }
    else { d_obs.alloc(1); d_desc.alloc(2); }
    d_ptr.upload(obs_ptr, (size_t)n_mp + 1, g.s);
    run_device(f, g.s, n_kf, kf_bad, n_mp, obs_ptr, obs_kf, nullptr, nullptr, nullptr, d_bad, d_ptr, d_obs, FromHost{d_desc.p, d_obs.p}, best,
               best_median, desc_out);
  });
}

extern "C" int ccm_kfstore_distinctive_descriptors(ccm_kf_store* store, int32_t n_kf, const uint64_t* kf_uid, const uint8_t* kf_bad, int32_t n_mp,
                                                   const int64_t* obs_ptr, const int32_t* obs_kf, const int32_t* obs_feat, int32_t* best,
                                                   int32_t* best_median, uint8_t* desc_out) {
  return guarded([&] {
    const std::string f = "ccm_kfstore_distinctive_descriptors";
    CCM_REQUIRE(store, f + ": null store");
    CCM_REQUIRE(n_kf == 0 || kf_uid, f + ": null kf_uid");
    check_shape(f, n_kf, kf_bad, n_mp, obs_ptr, obs_kf, obs_feat, best);
    ensure_device();
    if (n_mp == 0) return;
    std::vector<const uint4*> base;
    std::vector<int32_t> n_feat;
    int device = 0;
    kfstore_resolve(store, n_kf, kf_uid, base, n_feat, &device);
    CCM_CUDA(cudaSetDevice(device));
    const int64_t E = obs_ptr[n_mp];
    const CallStream g;
    DevBuf<uint8_t> d_bad;
    DevBuf<int64_t> d_ptr;
    DevBuf<int32_t> d_obs, d_feat, d_nfeat;
    DevBuf<const uint4*> d_base;
    if (n_kf) { d_bad.upload(kf_bad, n_kf, g.s); d_nfeat.upload(n_feat.data(), n_kf, g.s); d_base.upload(base.data(), n_kf, g.s); }
    else { d_bad.alloc(1); d_nfeat.alloc(1); d_base.alloc(1); }
    if (E) { d_obs.upload(obs_kf, (size_t)E, g.s); d_feat.upload(obs_feat, (size_t)E, g.s); }
    else { d_obs.alloc(1); d_feat.alloc(1); }
    d_ptr.upload(obs_ptr, (size_t)n_mp + 1, g.s);
    run_device(f, g.s, n_kf, kf_bad, n_mp, obs_ptr, obs_kf, obs_feat, n_feat.data(), kf_uid, d_bad, d_ptr, d_obs,
               FromStore{d_base.p, d_nfeat.p, d_feat.p, d_obs.p}, best, best_median, desc_out);
  });
}

// covis.cu — covisibility weights, behind ccm_covisibility / ccm_covisibility_host (include/ccm_b200.h).
//
//   KeyFrame::UpdateConnections, steps 1-2 and the orders of steps 4-5   cslam/src/KeyFrame.cpp:629-711
//
// Per batch keyframe b (row self = batch[b]): for every entry of its point list that is not null and whose point is not bad (a point
// at two indices counts twice), every observer k of the point with kf_id[k] != kf_id[self] (the idpair, not the row; bad observers
// count) adds 1 to counter[k].  The counter leaves in ascending kf_rank (std::map<kfptr,int>'s order when kf_rank is the address
// rank); the selection is every entry with weight >= th by (weight, rank) descending, or, when none reaches th, the first entry of
// the counter with the largest weight.  Integers only: the device and the host entry point agree exactly or not at all.
//
// Shape.  Two passes over the same kernels, so that the caller's capacity is checked before anything is written:
//   k_cv_shared   one CTA per batch keyframe: an open-addressing table of TAB slots in shared memory keyed by observer row, counts
//                 by shared atomics.  Pass 1 validates every row and writes the number of distinct observers d[b], or flags the
//                 keyframe dense[b] when more than LIMIT distinct observers arrive (it then goes to k_cv_dense; nothing is
//                 truncated).  Pass 2 counts again the keyframes not flagged, compacts the table and places each entry by counting
//                 the entries of smaller rank.
//   k_cv_dense    the keyframes that overflowed: one CTA per keyframe with a dense counter of n_kf words in global memory indexed by
//                 rank, so the compaction scan is already in rank order.  Pass 1 writes d[b], pass 2 the entries.
// The selection places each entry by counting the selected entries that precede it in (weight, rank) descending.  Keys (row, rank)
// are unique within a counter, so every position is fixed whatever the schedule.
#include <algorithm>
#include <climits>
#include <string>
#include <utility>
#include <vector>

#include "common.cuh"

using namespace ccm;

namespace {

constexpr int CTA = 256;
constexpr int LOG_TAB = 11;
constexpr int TAB = 1 << LOG_TAB;      // shared table slots
constexpr int LIMIT = TAB / 2;         // distinct observers on the shared path; the load factor stays below 1/2 + CTA/TAB
constexpr unsigned FULL = 0xffffffffu;
constexpr int32_t NO_BAD = 0x7f7f7f7f;

struct Scene {
  int32_t n_kf, n_b, n_mp, th;
  const uint64_t* kf_id;
  const uint32_t* kf_rank;
  const int32_t* inv_rank;
  const int32_t* batch;
  const int64_t* kf_mp_ptr;
  const int32_t* kf_mp;
  const uint8_t* mp_bad;
  const int64_t* obs_ptr;
  const int32_t* obs_kf;
};

struct Out {
  const int64_t* conn_ptr;
  int32_t *conn_kf, *conn_w, *n_sel, *sel_kf, *sel_w;
  uint8_t* status;
};

// visits every counted observer of batch keyframe b, threads striding over its point list; false on a row out of range
template <class F>
__device__ __forceinline__ bool for_each_observer(const Scene& s, int b, uint64_t sid, F&& f) {
  bool ok = true;
  for (int64_t j = s.kf_mp_ptr[b] + threadIdx.x; j < s.kf_mp_ptr[b + 1]; j += CTA) {
    const int32_t p = s.kf_mp[j];
    if (p < -1 || p >= s.n_mp) { ok = false; continue; }
    if (p < 0 || s.mp_bad[p]) continue;                        // if(!pMP) continue; if(pMP->isBad()) continue;
    for (int64_t q = s.obs_ptr[p]; q < s.obs_ptr[p + 1]; q++) {
      const int32_t k = s.obs_kf[q];
      if ((unsigned)k >= (unsigned)s.n_kf) { ok = false; break; }
      if (s.kf_id[k] == sid) continue;                         // if(mit->first->mId == this->mId) continue;
      f(k);
    }
  }
  return ok;
}

// one block-wide exclusive scan of a flag per thread; returns this thread's offset, *total the block's sum
__device__ __forceinline__ int block_scan(bool flag, int* wsum, int* total) {
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const unsigned m = __ballot_sync(FULL, flag);
  if (lane == 0) wsum[w] = __popc(m);
  __syncthreads();
  int off = 0, tot = 0;
  for (int q = 0; q < CTA / 32; q++) { off += q < w ? wsum[q] : 0; tot += wsum[q]; }
  __syncthreads();
  *total = tot;
  return off + __popc(m & ((1u << lane) - 1));
}

// the selection of batch keyframe b from its d entries (row, weight, rank), any order; sh: 3 shared scratch words
__device__ void write_selection(const Scene& s, const Out& o, int b, int d, const int32_t* e_row, const int32_t* e_w, const uint32_t* e_rank,
                                int* sh) {
  const int64_t base = o.conn_ptr[b];
  if (threadIdx.x == 0) { sh[0] = 0; sh[1] = 0; sh[2] = INT_MAX; }
  __syncthreads();
  int n_ge = 0;
  for (int t = threadIdx.x; t < d; t += CTA) {
    n_ge += e_w[t] >= s.th;
    atomicMax(&sh[1], e_w[t]);
  }
  atomicAdd(&sh[0], n_ge);
  __syncthreads();
  const int n_sel = sh[0], wmax = sh[1];
  if (n_sel > 0) {                                             // sort(vPairs) read back through push_front: (w, rank) descending
    for (int t = threadIdx.x; t < d; t += CTA) {
      const int w = e_w[t];
      if (w < s.th) continue;
      const uint32_t r = e_rank[t];
      int pos = 0;
      for (int u = 0; u < d; u++) pos += e_w[u] >= s.th && (e_w[u] > w || (e_w[u] == w && e_rank[u] > r));
      o.sel_kf[base + pos] = e_row[t]; o.sel_w[base + pos] = w;
    }
  } else {                                                     // (nmax, pKFmax): the first strict maximum in rank order
    for (int t = threadIdx.x; t < d; t += CTA)
      if (e_w[t] == wmax) atomicMin(&sh[2], (int)e_rank[t]);
    __syncthreads();
    for (int t = threadIdx.x; t < d; t += CTA)
      if (e_w[t] == wmax && (int)e_rank[t] == sh[2]) { o.sel_kf[base] = e_row[t]; o.sel_w[base] = wmax; }
  }
  const int used = n_sel > 0 ? n_sel : (d > 0 ? 1 : 0);
  for (int t = used + threadIdx.x; t < d; t += CTA) { o.sel_kf[base + t] = -1; o.sel_w[base + t] = 0; }
  if (threadIdx.x == 0) { o.n_sel[b] = used; o.status[b] = d > 0; }
  __syncthreads();
}

__device__ __forceinline__ bool table_add(int* key, int* cnt, int* n_dist, int k) {
  unsigned h = ((unsigned)k * 2654435761u) >> (32 - LOG_TAB);
  for (int probe = 0; probe < TAB; probe++) {
    int cur = ((volatile int*)key)[h];
    if (cur == -1) {
      cur = atomicCAS(&key[h], -1, k);
      if (cur == -1) {
        if (atomicAdd(n_dist, 1) >= LIMIT) return false;
        atomicAdd(&cnt[h], 1);
        return true;
      }
    }
    if (cur == k) { atomicAdd(&cnt[h], 1); return true; }
    h = (h + 1) & (TAB - 1);
  }
  return false;
}

// WRITE = false: validate, d[b] = distinct observers or -1 and dense[b] = 1 past LIMIT; WRITE = true: the outputs of every b with
// dense[b] = 0 (d[b] then holds k_cv_dense's count for the others, so it cannot tell the paths apart)
template <bool WRITE>
__global__ void __launch_bounds__(CTA) k_cv_shared(Scene s, Out o, int32_t* __restrict__ d_out, uint8_t* __restrict__ dense,
                                                   int32_t* __restrict__ bad_b) {
  __shared__ int key[TAB], cnt[TAB];
  __shared__ int32_t e_row[LIMIT], e_w[LIMIT];
  __shared__ uint32_t e_rank[LIMIT];
  __shared__ int n_dist, ovf, err, sh[3];
  for (int b = blockIdx.x; b < s.n_b; b += gridDim.x) {         // uniform per block
    if (WRITE && dense[b]) continue;
    for (int t = threadIdx.x; t < TAB; t += CTA) { key[t] = -1; cnt[t] = 0; }
    if (threadIdx.x == 0) { n_dist = 0; ovf = 0; err = (unsigned)s.batch[b] >= (unsigned)s.n_kf; }
    __syncthreads();
    if (err) {
      if (threadIdx.x == 0) { atomicMin(bad_b, b); d_out[b] = 0; dense[b] = 0; }
      __syncthreads();
      continue;
    }
    const uint64_t sid = s.kf_id[s.batch[b]];
    const bool ok = for_each_observer(s, b, sid, [&](int k) {
      if (((volatile int*)&ovf)[0]) return;
      if (!table_add(key, cnt, &n_dist, k)) ovf = 1;
    });
    if (!ok) err = 1;
    __syncthreads();
    if (!WRITE) {
      if (threadIdx.x == 0) {
        if (err) atomicMin(bad_b, b);
        d_out[b] = err ? 0 : ovf ? -1 : n_dist;
        dense[b] = !err && ovf;
      }
      __syncthreads();
      continue;
    }
    if (threadIdx.x == 0) n_dist = 0;
    __syncthreads();
    for (int t = threadIdx.x; t < TAB; t += CTA)
      if (key[t] >= 0) {
        const int e = atomicAdd(&n_dist, 1);                    // < LIMIT: pass 1 found at most LIMIT keys here
        if (e < LIMIT) { e_row[e] = key[t]; e_w[e] = cnt[t]; e_rank[e] = s.kf_rank[key[t]]; }
      }
    __syncthreads();
    const int d = n_dist;
    const int64_t base = o.conn_ptr[b];
    for (int t = threadIdx.x; t < d; t += CTA) {                // KFcounter: ascending rank
      const uint32_t r = e_rank[t];
      int pos = 0;
      for (int u = 0; u < d; u++) pos += e_rank[u] < r;
      o.conn_kf[base + pos] = e_row[t]; o.conn_w[base + pos] = e_w[t];
    }
    write_selection(s, o, b, d, e_row, e_w, e_rank, sh);
  }
}

// the keyframes of list[0 .. n_list): a dense counter by rank per CTA (cnt_all + blockIdx.x * n_kf; rank_all likewise holds the
// compacted entries' ranks for the selection)
template <bool WRITE>
__global__ void __launch_bounds__(CTA) k_cv_dense(Scene s, Out o, const int32_t* __restrict__ list, int n_list, int32_t* __restrict__ d_out,
                                                  int32_t* __restrict__ cnt_all, uint32_t* __restrict__ rank_all) {
  __shared__ int wsum[CTA / 32], sh[3];
  int32_t* cnt = cnt_all + (size_t)blockIdx.x * s.n_kf;
  uint32_t* e_rank = rank_all + (size_t)blockIdx.x * s.n_kf;
  for (int t = blockIdx.x; t < n_list; t += gridDim.x) {
    const int b = list[t];
    for (int r = threadIdx.x; r < s.n_kf; r += CTA) cnt[r] = 0;
    __syncthreads();
    for_each_observer(s, b, s.kf_id[s.batch[b]], [&](int k) { atomicAdd(&cnt[s.kf_rank[k]], 1); });
    __syncthreads();
    const int64_t base = WRITE ? o.conn_ptr[b] : 0;
    int d = 0;
    for (int r0 = 0; r0 < s.n_kf; r0 += CTA) {                   // compaction in rank order: KFcounter as it stands
      const int r = r0 + threadIdx.x;
      const int v = r < s.n_kf ? cnt[r] : 0;
      int tot;
      const int at = d + block_scan(v > 0, wsum, &tot);
      if (WRITE && v > 0) { o.conn_kf[base + at] = s.inv_rank[r]; o.conn_w[base + at] = v; e_rank[at] = (uint32_t)r; }
      d += tot;
    }
    if (!WRITE) {
      if (threadIdx.x == 0) d_out[b] = d;
      continue;
    }
    __syncthreads();
    write_selection(s, o, b, d, o.conn_kf + base, o.conn_w + base, e_rank, sh);
  }
}

void check_shape(const std::string& f, int32_t n_kf, const uint64_t* kf_id, const uint32_t* kf_rank, int32_t n_b, const int32_t* batch,
                 const int64_t* kf_mp_ptr, const int32_t* kf_mp, int32_t n_mp, const uint8_t* mp_bad, const int64_t* obs_ptr,
                 const int32_t* obs_kf, int64_t capacity, int64_t* conn_ptr, int32_t* conn_kf, int32_t* conn_w, int32_t* n_sel,
                 int32_t* sel_kf, int32_t* sel_w, uint8_t* status, int64_t* total) {
  CCM_REQUIRE(n_kf >= 0 && n_b >= 0 && n_mp >= 0 && capacity >= 0, f + ": negative size");
  CCM_REQUIRE(total, f + ": null total");
  CCM_REQUIRE(n_kf == 0 || (kf_id && kf_rank), f + ": null keyframe array");
  CCM_REQUIRE(n_mp == 0 || (mp_bad && obs_ptr), f + ": null point array");
  CCM_REQUIRE(batch && kf_mp_ptr && conn_ptr && (n_b == 0 || (n_sel && status)), f + ": null batch array");
  CCM_REQUIRE(capacity == 0 || (conn_kf && conn_w && sel_kf && sel_w), f + ": null output array");
  std::vector<uint8_t> seen(n_kf, 0);
  for (int32_t k = 0; k < n_kf; k++) {
    CCM_REQUIRE(kf_rank[k] < (uint32_t)n_kf && !seen[kf_rank[k]], f + ": kf_rank is not a permutation of 0 .. n_kf-1 (row " + std::to_string(k) + ")");
    seen[kf_rank[k]] = 1;
  }
  CCM_REQUIRE(kf_mp_ptr[0] == 0, f + ": kf_mp_ptr[0] must be 0");
  for (int32_t b = 0; b < n_b; b++) CCM_REQUIRE(kf_mp_ptr[b + 1] >= kf_mp_ptr[b], f + ": kf_mp_ptr is not monotone");
  CCM_REQUIRE(kf_mp_ptr[n_b] == 0 || kf_mp, f + ": null kf_mp");
  if (n_mp) {
    CCM_REQUIRE(obs_ptr[0] == 0, f + ": obs_ptr[0] must be 0");
    for (int32_t i = 0; i < n_mp; i++) CCM_REQUIRE(obs_ptr[i + 1] >= obs_ptr[i], f + ": obs_ptr is not monotone");
    CCM_REQUIRE(obs_ptr[n_mp] == 0 || obs_kf, f + ": null obs_kf");
  }
}

// the first row out of range met by batch keyframe b, as a message naming it; "" when there is none
std::string row_error(const std::string& f, int32_t b, int32_t n_kf, const uint64_t* kf_id, const int32_t* batch, const int64_t* kf_mp_ptr,
                      const int32_t* kf_mp, int32_t n_mp, const uint8_t* mp_bad, const int64_t* obs_ptr, const int32_t* obs_kf) {
  const std::string at = f + ": batch keyframe " + std::to_string(b) + " (row " + std::to_string(batch[b]);
  if (batch[b] < 0 || batch[b] >= n_kf) return at + "): keyframe row out of range";
  const std::string who = at + ", id " + std::to_string(kf_id[batch[b]]) + ")";
  for (int64_t j = kf_mp_ptr[b]; j < kf_mp_ptr[b + 1]; j++) {
    const int32_t p = kf_mp[j];
    if (p < -1 || p >= n_mp) return who + ", map point index " + std::to_string(j - kf_mp_ptr[b]) + ": point row " + std::to_string(p) + " out of range";
    if (p < 0 || mp_bad[p]) continue;
    for (int64_t q = obs_ptr[p]; q < obs_ptr[p + 1]; q++)
      if (obs_kf[q] < 0 || obs_kf[q] >= n_kf)
        return who + ", point row " + std::to_string(p) + ", observer " + std::to_string(q - obs_ptr[p]) + ": keyframe row " +
               std::to_string(obs_kf[q]) + " out of range";
  }
  return "";
}

}  // namespace

extern "C" int ccm_covisibility_host(int32_t n_kf, const uint64_t* kf_id, const uint32_t* kf_rank, int32_t n_b, const int32_t* batch,
                                     const int64_t* kf_mp_ptr, const int32_t* kf_mp, int32_t n_mp, const uint8_t* mp_bad, const int64_t* obs_ptr,
                                     const int32_t* obs_kf, int32_t th, int64_t capacity, int64_t* conn_ptr, int32_t* conn_kf, int32_t* conn_w,
                                     int32_t* n_sel, int32_t* sel_kf, int32_t* sel_w, uint8_t* status, int64_t* total) {
  return guarded([&] {
    const std::string f = "ccm_covisibility_host";
    check_shape(f, n_kf, kf_id, kf_rank, n_b, batch, kf_mp_ptr, kf_mp, n_mp, mp_bad, obs_ptr, obs_kf, capacity, conn_ptr, conn_kf, conn_w, n_sel,
                sel_kf, sel_w, status, total);
    for (int32_t b = 0; b < n_b; b++) {
      const std::string e = row_error(f, b, n_kf, kf_id, batch, kf_mp_ptr, kf_mp, n_mp, mp_bad, obs_ptr, obs_kf);
      if (!e.empty()) throw Error(CCM_ERR_INVALID, e);
    }
    std::vector<int32_t> inv(n_kf), cnt(n_kf, 0), touched;
    for (int32_t k = 0; k < n_kf; k++) inv[kf_rank[k]] = k;
    std::vector<int64_t> ptr(n_b + 1, 0);
    std::vector<int32_t> ck, cw, ns(n_b), sk, sw;
    for (int32_t b = 0; b < n_b; b++) {
      const uint64_t sid = kf_id[batch[b]];
      touched.clear();
      for (int64_t j = kf_mp_ptr[b]; j < kf_mp_ptr[b + 1]; j++) {
        const int32_t p = kf_mp[j];
        if (p < 0 || mp_bad[p]) continue;
        for (int64_t q = obs_ptr[p]; q < obs_ptr[p + 1]; q++) {
          const int32_t k = obs_kf[q];
          if (kf_id[k] == sid) continue;
          if (cnt[kf_rank[k]]++ == 0) touched.push_back((int32_t)kf_rank[k]);
        }
      }
      std::sort(touched.begin(), touched.end());
      const size_t at = ck.size();
      int wmax = 0, first_max = -1, n_ge = 0;
      for (size_t t = 0; t < touched.size(); t++) {
        const int w = cnt[touched[t]];
        ck.push_back(inv[touched[t]]); cw.push_back(w);
        if (w > wmax) { wmax = w; first_max = (int)t; }
        n_ge += w >= th;
        cnt[touched[t]] = 0;
      }
      std::vector<std::pair<int, int32_t> > sel;                  // (weight, rank), placed by descending order below
      for (size_t t = 0; t < touched.size(); t++)
        if (cw[at + t] >= th) sel.push_back(std::make_pair(cw[at + t], touched[t]));
      std::sort(sel.begin(), sel.end());
      for (size_t t = sel.size(); t-- > 0;) { sk.push_back(inv[sel[t].second]); sw.push_back(sel[t].first); }
      if (n_ge == 0 && first_max >= 0) { sk.push_back(ck[at + first_max]); sw.push_back(wmax); }
      ns[b] = n_ge > 0 ? n_ge : (first_max >= 0 ? 1 : 0);
      sk.resize(ck.size(), -1); sw.resize(ck.size(), 0);
      ptr[b + 1] = (int64_t)ck.size();
    }
    *total = ptr[n_b];
    if (capacity < ptr[n_b])
      throw Error(CCM_ERR_INVALID, f + ": capacity " + std::to_string(capacity) + " below the " + std::to_string(ptr[n_b]) + " entries needed");
    std::copy(ptr.begin(), ptr.end(), conn_ptr);
    std::copy(ck.begin(), ck.end(), conn_kf); std::copy(cw.begin(), cw.end(), conn_w);
    std::copy(sk.begin(), sk.end(), sel_kf); std::copy(sw.begin(), sw.end(), sel_w);
    for (int32_t b = 0; b < n_b; b++) { n_sel[b] = ns[b]; status[b] = ptr[b + 1] > ptr[b]; }
  });
}

extern "C" int ccm_covisibility(int32_t n_kf, const uint64_t* kf_id, const uint32_t* kf_rank, int32_t n_b, const int32_t* batch,
                                const int64_t* kf_mp_ptr, const int32_t* kf_mp, int32_t n_mp, const uint8_t* mp_bad, const int64_t* obs_ptr,
                                const int32_t* obs_kf, int32_t th, int64_t capacity, int64_t* conn_ptr, int32_t* conn_kf, int32_t* conn_w,
                                int32_t* n_sel, int32_t* sel_kf, int32_t* sel_w, uint8_t* status, int64_t* total) {
  return guarded([&] {
    const std::string f = "ccm_covisibility";
    check_shape(f, n_kf, kf_id, kf_rank, n_b, batch, kf_mp_ptr, kf_mp, n_mp, mp_bad, obs_ptr, obs_kf, capacity, conn_ptr, conn_kf, conn_w, n_sel,
                sel_kf, sel_w, status, total);
    ensure_device();
    if (n_b == 0) { *total = 0; conn_ptr[0] = 0; return; }
    const int64_t M = kf_mp_ptr[n_b], E = n_mp ? obs_ptr[n_mp] : 0;
    const CallStream g;
    std::vector<int32_t> inv(std::max(n_kf, 1), 0);
    for (int32_t k = 0; k < n_kf; k++) inv[kf_rank[k]] = k;
    DevBuf<uint64_t> d_id;
    DevBuf<uint32_t> d_rank;
    DevBuf<int32_t> d_inv, d_batch, d_mp, d_obs, d_d, d_bad;
    DevBuf<int64_t> d_mptr, d_optr, d_cptr;
    DevBuf<uint8_t> d_mpbad, d_dense;
    if (n_kf) { d_id.upload(kf_id, n_kf, g.s); d_rank.upload(kf_rank, n_kf, g.s); } else { d_id.alloc(1); d_rank.alloc(1); }
    d_inv.upload(inv.data(), inv.size(), g.s);
    d_batch.upload(batch, n_b, g.s);
    d_mptr.upload(kf_mp_ptr, (size_t)n_b + 1, g.s);
    if (M) d_mp.upload(kf_mp, (size_t)M, g.s); else d_mp.alloc(1);
    if (n_mp) { d_mpbad.upload(mp_bad, n_mp, g.s); d_optr.upload(obs_ptr, (size_t)n_mp + 1, g.s); } else { d_mpbad.alloc(1); d_optr.alloc(1); }
    if (E) d_obs.upload(obs_kf, (size_t)E, g.s); else d_obs.alloc(1);
    d_d.alloc(n_b); d_dense.alloc(n_b); d_bad.alloc(1);
    CCM_CUDA(cudaMemsetAsync(d_bad.p, 0x7f, sizeof(int32_t), g.s));
    const Scene sc{n_kf, n_b, n_mp, th, d_id.p, d_rank.p, d_inv.p, d_batch.p, d_mptr.p, d_mp.p, d_mpbad.p, d_optr.p, d_obs.p};
    const int sms = sm_count();
    const int grid = std::min(n_b, sms * 8);
    k_cv_shared<false><<<grid, CTA, 0, g.s>>>(sc, Out{}, d_d.p, d_dense.p, d_bad.p);
    CCM_LAUNCHED();
    std::vector<int32_t> d(n_b);
    int32_t bad = NO_BAD;
    d_d.download(d.data(), n_b, g.s);
    CCM_CUDA(cudaMemcpyAsync(&bad, d_bad.p, sizeof(int32_t), cudaMemcpyDeviceToHost, g.s));
    CCM_CUDA(cudaStreamSynchronize(g.s));
    if (bad != NO_BAD) throw Error(CCM_ERR_INVALID, row_error(f, bad, n_kf, kf_id, batch, kf_mp_ptr, kf_mp, n_mp, mp_bad, obs_ptr, obs_kf));
    std::vector<int32_t> over;
    for (int32_t b = 0; b < n_b; b++) if (d[b] < 0) over.push_back(b);
    DevBuf<int32_t> d_over, d_cnt;
    DevBuf<uint32_t> d_erank;
    int g_dense = 0;
    if (!over.empty()) {                                         // counters past LIMIT distinct observers
      g_dense = (int)std::min<int64_t>({(int64_t)over.size(), (int64_t)sms, std::max<int64_t>(1, (int64_t(1) << 28) / (8 * (int64_t)n_kf))});
      d_over.upload(over.data(), over.size(), g.s);
      d_cnt.alloc((size_t)g_dense * n_kf); d_erank.alloc((size_t)g_dense * n_kf);
      k_cv_dense<false><<<g_dense, CTA, 0, g.s>>>(sc, Out{}, d_over.p, (int)over.size(), d_d.p, d_cnt.p, d_erank.p);
      CCM_LAUNCHED();
      d_d.download(d.data(), n_b, g.s);
      CCM_CUDA(cudaStreamSynchronize(g.s));
    }
    std::vector<int64_t> ptr(n_b + 1, 0);
    for (int32_t b = 0; b < n_b; b++) ptr[b + 1] = ptr[b] + d[b];
    *total = ptr[n_b];
    if (capacity < ptr[n_b])
      throw Error(CCM_ERR_INVALID, f + ": capacity " + std::to_string(capacity) + " below the " + std::to_string(ptr[n_b]) + " entries needed");
    const int64_t T = std::max<int64_t>(ptr[n_b], 1);
    DevBuf<int32_t> d_ck, d_cw, d_ns, d_sk, d_sw;
    DevBuf<uint8_t> d_st;
    d_cptr.upload(ptr.data(), ptr.size(), g.s);
    d_ck.alloc(T); d_cw.alloc(T); d_sk.alloc(T); d_sw.alloc(T); d_ns.alloc(n_b); d_st.alloc(n_b);
    const Out o{d_cptr.p, d_ck.p, d_cw.p, d_ns.p, d_sk.p, d_sw.p, d_st.p};
    k_cv_shared<true><<<grid, CTA, 0, g.s>>>(sc, o, d_d.p, d_dense.p, d_bad.p);
    CCM_LAUNCHED();
    if (g_dense) {
      k_cv_dense<true><<<g_dense, CTA, 0, g.s>>>(sc, o, d_over.p, (int)over.size(), d_d.p, d_cnt.p, d_erank.p);
      CCM_LAUNCHED();
    }
    std::copy(ptr.begin(), ptr.end(), conn_ptr);
    d_ck.download(conn_kf, ptr[n_b], g.s); d_cw.download(conn_w, ptr[n_b], g.s);
    d_sk.download(sel_kf, ptr[n_b], g.s); d_sw.download(sel_w, ptr[n_b], g.s);
    d_ns.download(n_sel, n_b, g.s); d_st.download(status, n_b, g.s);
    CCM_CUDA(cudaStreamSynchronize(g.s));
  });
}

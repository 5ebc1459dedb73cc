// kf_db.cu — device-resident keyframe database (place-recognition candidate queries) behind ccm_kfdb_* (include/ccm_b200.h).
//
// Replaces the host std::list walks of cslam::KeyFrameDatabase (S/Database.cpp): add :37-43, erase :45-64, clear :66-70,
// DetectLoopCandidates :72-202, DetectMapMatchCandidates :204-327, DetectRelocalizationCandidates :329-439, and the
// DBoW2 scores they call (D/ScoringObject.cpp:23-311).  DESIGN.md §5 "Keyframe database" has the argument in full.
//
// State.  Every keyframe holds a slot.  Its BowVector (word ids ascending, f64 values) sits in one device pool; the inverted file is
// one segment per word in a second pool (int32 slot per posting, -1 = erased), in insertion order: within a word, the order of the
// reference's list.  Host mirrors of both pools are the truth; add / erase touch the mirrors only (O(|BowVector|) plus the walk of
// each word's list that erase shares with the reference) and record what changed; the next query uploads the changes (a scatter)
// before its first kernel.  A full segment moves to a region twice its size (amortised O(1) per posting); a segment with more
// erased than live postings is compacted in place (order kept); pools that are mostly garbage are repacked and uploaded whole.
// Every call holds the handle's mutex and synchronises before it returns: postings never move under a running query.
//
// Query (B queries at once, blockIdx.y = query):
//   k_prepare   count = 0, first = +inf, hidden = empty slot or client not in the query's mask; then the explicit exclusions
//   k_count     a warp per query word walks that word's postings: atomicAdd of the count, atomicMin of the first-appearance key
//               (rank of the word in the query << 32 | position in the word's list) — the order of lKFsSharingWords
//   k_max       maxCommonWords; minCommonWords = (int)(max * 0.8f) as the reference computes it in float
//   k_compact   slots with count > minCommonWords (the scored ones), unordered
//   k_rank      rank by the first-appearance key -> reference order
//   k_score     a warp per candidate, the query's BowVector in shared memory.  The reference's merge visits the common words in
//               ascending order and adds one term per common word; here 32 lanes look up 32 consecutive words (binary search) and
//               the terms are added in word order by one lane, with __dadd_rn / __dmul_rn / __ddiv_rn / __dsqrt_rn: the f64 score
//               is bit-identical to DBoW2's for L1, L2, ChiSquare, Bhattacharyya and DotProduct.  KL walks the query's words (its
//               sum runs over all of v1) and uses the device log, which is not libm's: |rel. error| <= 1e-12 (DESIGN.md §5).
// Integer work is order independent (atomics on counts and keys), so the candidate list is deterministic.  The covisibility
// accumulation and the 0.75 * bestAccScore retain are order-dependent float work over a few hundred items: ccm_kfdb_select, host.
#include <algorithm>
#include <cmath>
#include <memory>
#include <mutex>
#include <unordered_map>
#include <unordered_set>

#include "common.cuh"

using namespace ccm;

namespace {

enum { S_L1 = 0, S_L2 = 1, S_CHI = 2, S_KL = 3, S_BHAT = 4, S_DOT = 5 };   // DBoW2::ScoringType (D/BowVector.h:45-53)
constexpr int MAX_QUERY_WORDS = 16384;                                     // query BowVector in shared memory: 12 bytes a word
constexpr unsigned long long NO_KEY = ~0ull;
constexpr uint32_t NO_CLIENT = 0xffffffffu;
constexpr int TPB = 256;
constexpr int MAX_BATCH = 65535;                                           // queries per launch: blockIdx.y

// ---- kernels ----------------------------------------------------------------------------------------------------------------

__global__ void k_scatter_i32(int* __restrict__ dst, const long long* __restrict__ pos, const int* __restrict__ val, int n) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) dst[pos[i]] = val[i];
}

__global__ void k_scatter_seg(long long* __restrict__ seg_off, int* __restrict__ seg_len, const int* __restrict__ word,
                              const long long* __restrict__ off, const int* __restrict__ len, int n) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) { seg_off[word[i]] = off[i]; seg_len[word[i]] = len[i]; }
}

__global__ void k_prepare(int S, const uint32_t* __restrict__ slot_client, const unsigned long long* __restrict__ mask,
                          int* __restrict__ count, unsigned long long* __restrict__ first, uint8_t* __restrict__ hidden) {
  const int b = blockIdx.y;
  const unsigned long long m = mask[b];
  for (int s = blockIdx.x * blockDim.x + threadIdx.x; s < S; s += gridDim.x * blockDim.x) {
    const uint32_t c = slot_client[s];
    const size_t i = (size_t)b * S + s;
    count[i] = 0; first[i] = NO_KEY;
    hidden[i] = (c == NO_CLIENT || c >= 64 || !((m >> c) & 1ull)) ? 1 : 0;
  }
}

__global__ void k_exclude(int S, const int* __restrict__ ex_ptr, const int* __restrict__ ex_slot, uint8_t* __restrict__ hidden) {
  const int b = blockIdx.y;
  for (int i = ex_ptr[b] + blockIdx.x * blockDim.x + threadIdx.x; i < ex_ptr[b + 1]; i += gridDim.x * blockDim.x)
    hidden[(size_t)b * S + ex_slot[i]] = 1;
}

// a warp per query word
__global__ void __launch_bounds__(TPB) k_count(int S, const int* __restrict__ q_ptr, const uint32_t* __restrict__ q_word,
                                               const long long* __restrict__ seg_off, const int* __restrict__ seg_len,
                                               const int* __restrict__ post, const uint8_t* __restrict__ hidden, int* __restrict__ count,
                                               unsigned long long* __restrict__ first) {
  const int b = blockIdx.y;
  const int lane = threadIdx.x & 31;
  const int nq = q_ptr[b + 1] - q_ptr[b];
  const size_t base = (size_t)b * S;
  for (int r = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; r < nq; r += (gridDim.x * blockDim.x) >> 5) {
    const uint32_t w = q_word[q_ptr[b] + r];
    const long long off = seg_off[w];
    const int len = seg_len[w];
    for (int p = lane; p < len; p += 32) {
      const int s = post[off + p];
      if (s < 0 || hidden[base + s]) continue;
      atomicAdd(&count[base + s], 1);
      atomicMin(&first[base + s], ((unsigned long long)r << 32) | (unsigned)p);
    }
  }
}

// hdr[b] = {maxCommonWords, number of slots sharing a word, number of scored candidates}
__global__ void k_max(int S, const int* __restrict__ count, int* __restrict__ hdr) {
  const int b = blockIdx.y;
  int m = 0, share = 0;
  for (int s = blockIdx.x * blockDim.x + threadIdx.x; s < S; s += gridDim.x * blockDim.x) {
    const int c = count[(size_t)b * S + s];
    m = max(m, c); share += c > 0;
  }
  for (int o = 16; o > 0; o >>= 1) { m = max(m, __shfl_xor_sync(0xffffffffu, m, o)); share += __shfl_xor_sync(0xffffffffu, share, o); }
  if ((threadIdx.x & 31) == 0) { atomicMax(&hdr[3 * b], m); if (share) atomicAdd(&hdr[3 * b + 1], share); }
}

__device__ __forceinline__ int min_common(int max_common) { return __float2int_rz(__fmul_rn((float)max_common, 0.8f)); }

__global__ void k_compact(int S, const int* __restrict__ count, const unsigned long long* __restrict__ first, int* __restrict__ hdr,
                          int* __restrict__ c_slot, unsigned long long* __restrict__ c_key) {
  const int b = blockIdx.y;
  const int minc = min_common(hdr[3 * b]);
  for (int s = blockIdx.x * blockDim.x + threadIdx.x; s < S; s += gridDim.x * blockDim.x) {
    const size_t i = (size_t)b * S + s;
    if (count[i] > minc) {
      const int k = atomicAdd(&hdr[3 * b + 2], 1);
      c_slot[(size_t)b * S + k] = s; c_key[(size_t)b * S + k] = first[i];
    }
  }
}

// rank = number of smaller keys (keys are distinct: one posting position belongs to one slot)
__global__ void __launch_bounds__(TPB) k_rank(int S, const int* __restrict__ hdr, const int* __restrict__ c_slot,
                                              const unsigned long long* __restrict__ c_key, const int* __restrict__ count,
                                              int* __restrict__ o_slot, int* __restrict__ o_count) {
  __shared__ unsigned long long tile[TPB];
  const int b = blockIdx.y;
  const int n = hdr[3 * b + 2];
  const size_t base = (size_t)b * S;
  for (int i0 = blockIdx.x * blockDim.x; i0 < n; i0 += gridDim.x * blockDim.x) {
    const int i = i0 + threadIdx.x;
    const unsigned long long k = i < n ? c_key[base + i] : NO_KEY;
    int rank = 0;
    for (int j0 = 0; j0 < n; j0 += TPB) {
      __syncthreads();
      tile[threadIdx.x] = j0 + threadIdx.x < n ? c_key[base + j0 + threadIdx.x] : NO_KEY;
      __syncthreads();
      const int m = min(TPB, n - j0);
      for (int j = 0; j < m; j++) rank += tile[j] < k;
    }
    if (i < n) { const int s = c_slot[base + i]; o_slot[base + rank] = s; o_count[base + rank] = count[base + s]; }
  }
}

__device__ __forceinline__ int lower_bound_u32(const uint32_t* a, int n, uint32_t w) {
  int lo = 0, hi = n;
  while (lo < hi) { const int mid = (lo + hi) >> 1; if (a[mid] < w) lo = mid + 1; else hi = mid; }
  return lo;
}

// the term one common word adds (vi: query, wi: candidate), as D/ScoringObject.cpp writes it; `add` is false for a skipped term
__device__ __forceinline__ double term(int scoring, double vi, double wi, bool& add) {
  add = true;
  switch (scoring) {
    case S_L1: return __dsub_rn(__dsub_rn(fabs(__dsub_rn(vi, wi)), fabs(vi)), fabs(wi));   // fabs(vi - wi) - fabs(vi) - fabs(wi)
    case S_CHI: { const double s = __dadd_rn(vi, wi); add = s != 0.0; return __ddiv_rn(__dmul_rn(vi, wi), s); }
    case S_BHAT: return __dsqrt_rn(__dmul_rn(vi, wi));
    default: return __dmul_rn(vi, wi);                                                     // L2, DotProduct
  }
}

// one warp per (query b, candidate i); the query's BowVector in shared memory (dynamic: n * 12 bytes)
__global__ void __launch_bounds__(TPB) k_score(int S, int scoring, double log_eps, const int* __restrict__ q_ptr,
                                               const uint32_t* __restrict__ q_word, const double* __restrict__ q_val,
                                               const int* __restrict__ n_cand /*stride ncs*/, int ncs, const int* __restrict__ cand_slot,
                                               const long long* __restrict__ slot_off, const int* __restrict__ slot_n,
                                               const uint32_t* __restrict__ bow_word, const double* __restrict__ bow_val,
                                               double* __restrict__ score) {
  extern __shared__ double sm[];
  const int b = blockIdx.y;
  const int nq = q_ptr[b + 1] - q_ptr[b];
  double* qv = sm;
  uint32_t* qw = reinterpret_cast<uint32_t*>(sm + nq);
  for (int i = threadIdx.x; i < nq; i += blockDim.x) { qw[i] = q_word[q_ptr[b] + i]; qv[i] = q_val[q_ptr[b] + i]; }
  __syncthreads();
  const int lane = threadIdx.x & 31;
  const int n = n_cand[b * ncs];
  const size_t base = (size_t)b * S;
  for (int c = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; c < n; c += (gridDim.x * blockDim.x) >> 5) {
    const int s = cand_slot[base + c];
    const uint32_t* cw = bow_word + slot_off[s];
    const double* cv = bow_val + slot_off[s];
    const int nc = slot_n[s];
    double acc = 0.0;
    if (scoring != S_KL) {
      // walk the candidate's words; a word is common when the query holds it
      for (int j0 = 0; j0 < nc; j0 += 32) {
        const int j = j0 + lane;
        double t = 0.0; bool add = false;
        if (j < nc) {
          const uint32_t w = cw[j];
          const int k = lower_bound_u32(qw, nq, w);
          if (k < nq && qw[k] == w) t = term(scoring, qv[k], cv[j], add);
        }
        unsigned m = __ballot_sync(0xffffffffu, add);
        while (m) {                                         // in word order, on every lane (the shuffle needs the warp)
          const int src = __ffs(m) - 1; m &= m - 1;
          acc = __dadd_rn(acc, __shfl_sync(0xffffffffu, t, src));
        }
      }
      if (scoring == S_L1) acc = -acc / 2.0;
      else if (scoring == S_L2) acc = acc >= 1 ? 1.0 : __dsub_rn(1.0, __dsqrt_rn(__dsub_rn(1.0, acc)));
      else if (scoring == S_CHI) acc = 2. * acc;
    } else {
      // KL runs over every word of v1 = the query: common -> vi * log(vi / wi) (both non-zero); missing from v2 -> vi * (log(vi) -
      // LOG_EPS), with the != 0 guard only for the words after v2's last word (the loop's tail, D/ScoringObject.cpp:216-218)
      const uint32_t last = nc ? cw[nc - 1] : 0;
      for (int i0 = 0; i0 < nq; i0 += 32) {
        const int i = i0 + lane;
        double t = 0.0; bool add = false;
        if (i < nq) {
          const uint32_t w = qw[i];
          const double vi = qv[i];
          const int k = nc ? lower_bound_u32(cw, nc, w) : 0;
          if (k < nc && cw[k] == w) {
            const double wi = cv[k];
            if (vi != 0 && wi != 0) { t = __dmul_rn(vi, log(__ddiv_rn(vi, wi))); add = true; }
          } else if (nc && w < last) {
            t = __dmul_rn(vi, __dsub_rn(log(vi), log_eps)); add = true;
          } else if (vi != 0) {
            t = __dmul_rn(vi, __dsub_rn(log(vi), log_eps)); add = true;
          }
        }
        unsigned m = __ballot_sync(0xffffffffu, add);
        while (m) {
          const int src = __ffs(m) - 1; m &= m - 1;
          acc = __dadd_rn(acc, __shfl_sync(0xffffffffu, t, src));
        }
      }
    }
    if (lane == 0) score[base + c] = acc;
  }
}

struct Seg { long long off = 0; int len = 0, cap = 0, dead = 0; };

// k_score's dynamic shared memory limit is a process-wide attribute of the function: raised once per device, to the largest query
// any handle accepts, under a process-wide lock (handles of other threads launch k_score concurrently)
void allow_score_smem() {
  static std::mutex mu;
  static std::vector<char> done;
  int dev = 0;
  CCM_CUDA(cudaGetDevice(&dev));                                           // the handle's device, set by the caller
  std::lock_guard<std::mutex> lock(mu);
  if ((int)done.size() <= dev) done.resize(dev + 1, 0);
  if (done[dev]) return;
  CCM_CUDA(cudaFuncSetAttribute((const void*)k_score, cudaFuncAttributeMaxDynamicSharedMemorySize, MAX_QUERY_WORDS * 12));
  done[dev] = 1;
}

int grid_for(const void* fn, size_t smem, long long items_per_query, int per_block) {
  int per_sm = 0;
  CCM_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, fn, TPB, smem));
  CCM_REQUIRE(per_sm >= 1, "ccm_kfdb: kernel does not fit on an SM");
  return (int)std::max<long long>(1, std::min<long long>((long long)sm_count() * per_sm, (items_per_query + per_block - 1) / per_block));
}

}  // namespace

struct ccm_kfdb {
  int n_words = 0, scoring = 0, device = 0;
  cudaStream_t stream = nullptr;
  std::mutex mu;
  struct KF { int slot; uint32_t client; long long off; int n; };
  std::unordered_map<uint64_t, KF> kf;
  // slots
  std::vector<uint64_t> uid_of_slot;
  std::vector<uint32_t> h_slot_client; std::vector<long long> h_slot_off; std::vector<int> h_slot_n;
  std::vector<int> free_slots;
  std::vector<int> dirty_slots;
  DevBuf<uint32_t> d_slot_client; DevBuf<long long> d_slot_off; DevBuf<int> d_slot_n;
  bool slots_full = true;
  // BowVectors
  std::vector<uint32_t> h_bw; std::vector<double> h_bv;
  long long bow_garbage = 0;
  std::vector<std::pair<long long, int>> dirty_bow;   // (offset, n) appended since the last flush
  DevBuf<uint32_t> d_bw; DevBuf<double> d_bv;
  bool bow_full = true;
  // inverted file
  std::vector<Seg> seg;
  std::vector<int> h_post;
  long long post_garbage = 0;
  std::vector<long long> dirty_pos; std::vector<int> dirty_word;
  std::vector<uint8_t> word_dirty;
  DevBuf<int> d_post; DevBuf<long long> d_seg_off; DevBuf<int> d_seg_len;
  bool post_full = true;
  // query scratch
  DevBuf<int> d_count, d_hdr, d_cslot, d_oslot, d_ocount, d_qptr, d_exptr, d_exslot;
  DevBuf<unsigned long long> d_first, d_ckey, d_mask;
  DevBuf<uint8_t> d_hidden;
  DevBuf<uint32_t> d_qword; DevBuf<double> d_qval, d_score;
  DevBuf<long long> d_spos; DevBuf<int> d_sval, d_sword, d_slen; DevBuf<long long> d_soff;
  // CUDA-event kernel timing (bench): count = k_prepare..k_count, score = k_max..k_score
  bool timing = false;
  cudaEvent_t ev[3] = {nullptr, nullptr, nullptr};
  double t_count_ms = 0, t_score_ms = 0;
  long long timed_queries = 0;

  ~ccm_kfdb() {
    for (auto e : ev) if (e) cudaEventDestroy(e);
    if (stream) cudaStreamDestroy(stream);
  }

  int slots() const { return (int)uid_of_slot.size(); }

  void mark_pos(long long p) { if (!post_full) dirty_pos.push_back(p); }
  void mark_word(uint32_t w) { if (!post_full && !word_dirty[w]) { word_dirty[w] = 1; dirty_word.push_back((int)w); } }

  void repack_postings() {
    std::vector<int> np; np.reserve(h_post.size() - post_garbage + 1024);
    for (auto& s : seg) {
      if (!s.cap) continue;
      const long long off = (long long)np.size();
      for (int p = 0; p < s.len; p++) if (h_post[s.off + p] >= 0) np.push_back(h_post[s.off + p]);
      const int len = (int)(np.size() - off);
      int cap = 4; while (cap < len + len / 2) cap *= 2;
      np.resize(off + cap, -1);
      s.off = off; s.len = len; s.cap = cap; s.dead = 0;
    }
    h_post.swap(np); post_garbage = 0; post_full = true;
    dirty_pos.clear(); dirty_word.clear(); std::fill(word_dirty.begin(), word_dirty.end(), 0);
  }

  void repack_bows() {
    std::vector<uint32_t> nw; std::vector<double> nv; nw.reserve(h_bw.size() - bow_garbage); nv.reserve(h_bw.size() - bow_garbage);
    for (auto& kv : kf) {
      KF& e = kv.second;
      const long long off = (long long)nw.size();
      nw.insert(nw.end(), h_bw.begin() + e.off, h_bw.begin() + e.off + e.n); nv.insert(nv.end(), h_bv.begin() + e.off, h_bv.begin() + e.off + e.n);
      e.off = off; h_slot_off[e.slot] = off;
    }
    h_bw.swap(nw); h_bv.swap(nv); bow_garbage = 0; bow_full = true; slots_full = true; dirty_bow.clear();
  }

  void add(uint64_t uid, uint32_t client, int n, const uint32_t* w, const double* v) {
    CCM_REQUIRE(!kf.count(uid), "ccm_kfdb_add: keyframe already in the database (erase it first)");
    CCM_REQUIRE(client < 64, "ccm_kfdb_add: client id >= 64");
    for (int i = 0; i < n; i++) {
      CCM_REQUIRE(w[i] < (uint32_t)n_words, "ccm_kfdb_add: word id out of range");
      CCM_REQUIRE(i == 0 || w[i] > w[i - 1], "ccm_kfdb_add: BowVector words must be strictly ascending (std::map order)");
    }
    int slot;
    if (!free_slots.empty()) { slot = free_slots.back(); free_slots.pop_back(); }
    else { slot = slots(); uid_of_slot.push_back(0); h_slot_client.push_back(NO_CLIENT); h_slot_off.push_back(0); h_slot_n.push_back(0); slots_full = true; }
    const long long off = (long long)h_bw.size();
    h_bw.insert(h_bw.end(), w, w + n); h_bv.insert(h_bv.end(), v, v + n);
    if (!bow_full && n) dirty_bow.push_back({off, n});
    kf[uid] = KF{slot, client, off, n};
    uid_of_slot[slot] = uid; h_slot_client[slot] = client; h_slot_off[slot] = off; h_slot_n[slot] = n;
    if (!slots_full) dirty_slots.push_back(slot);
    for (int i = 0; i < n; i++) {                                  // mvInvertedFile[word].push_back(pKF)
      Seg& s = seg[w[i]];
      if (s.len == s.cap) {                                        // move the segment to a region twice its size
        const int cap = std::max(4, 2 * s.cap);
        const long long noff = (long long)h_post.size();
        h_post.resize(noff + cap, -1);
        for (int p = 0; p < s.len; p++) { h_post[noff + p] = h_post[s.off + p]; mark_pos(noff + p); }
        post_garbage += s.cap;
        s.off = noff; s.cap = cap;
      }
      h_post[s.off + s.len] = slot; mark_pos(s.off + s.len);
      s.len++;
      mark_word(w[i]);
    }
    if (post_garbage > 1024 && 2 * post_garbage > (long long)h_post.size()) repack_postings();
  }

  void erase(uint64_t uid) {
    auto it = kf.find(uid);
    if (it == kf.end()) return;                                     // not in the lists: the reference's loops find nothing
    const KF e = it->second;
    for (int i = 0; i < e.n; i++) {                                 // first occurrence per word (there is one)
      const uint32_t w = h_bw[e.off + i];
      Seg& s = seg[w];
      for (int p = 0; p < s.len; p++)
        if (h_post[s.off + p] == e.slot) { h_post[s.off + p] = -1; mark_pos(s.off + p); s.dead++; break; }
      if (s.len >= 8 && 2 * s.dead > s.len) {                       // compact in place, order kept
        int q = 0;
        for (int p = 0; p < s.len; p++) if (h_post[s.off + p] >= 0) h_post[s.off + q++] = h_post[s.off + p];
        for (int p = q; p < s.len; p++) h_post[s.off + p] = -1;
        for (int p = 0; p < s.len; p++) mark_pos(s.off + p);
        s.len = q; s.dead = 0;
      }
      mark_word(w);
    }
    bow_garbage += e.n;
    uid_of_slot[e.slot] = 0; h_slot_client[e.slot] = NO_CLIENT; h_slot_n[e.slot] = 0;
    if (!slots_full) dirty_slots.push_back(e.slot);
    free_slots.push_back(e.slot);
    kf.erase(it);
    if (bow_garbage > 4096 && 2 * bow_garbage > (long long)h_bw.size()) repack_bows();
  }

  void clear() {
    kf.clear(); uid_of_slot.clear(); h_slot_client.clear(); h_slot_off.clear(); h_slot_n.clear(); free_slots.clear();
    h_bw.clear(); h_bv.clear(); bow_garbage = 0; h_post.clear(); post_garbage = 0;
    std::fill(seg.begin(), seg.end(), Seg{});
    dirty_slots.clear(); dirty_bow.clear(); dirty_pos.clear(); dirty_word.clear(); std::fill(word_dirty.begin(), word_dirty.end(), 0);
    slots_full = bow_full = post_full = true;
  }

  // upload what add / erase changed since the last query
  void flush() {
    cudaStream_t st = stream;
    const int S = slots();
    if (slots_full) {
      d_slot_client.upload(h_slot_client.data(), S, st); d_slot_off.upload(h_slot_off.data(), S, st); d_slot_n.upload(h_slot_n.data(), S, st);
    } else if (!dirty_slots.empty()) {
      for (int s : dirty_slots) {
        CCM_CUDA(cudaMemcpyAsync(d_slot_client.p + s, &h_slot_client[s], 4, cudaMemcpyHostToDevice, st));
        CCM_CUDA(cudaMemcpyAsync(d_slot_off.p + s, &h_slot_off[s], 8, cudaMemcpyHostToDevice, st));
        CCM_CUDA(cudaMemcpyAsync(d_slot_n.p + s, &h_slot_n[s], 4, cudaMemcpyHostToDevice, st));
      }
    }
    if (bow_full || d_bw.n < h_bw.size()) {
      if (d_bw.n < h_bw.size()) { d_bw.alloc(std::max<size_t>(1024, 2 * h_bw.size())); d_bv.alloc(d_bw.n); }
      d_bw.upload(h_bw.data(), h_bw.size(), st); d_bv.upload(h_bv.data(), h_bv.size(), st);
    } else {
      for (auto& r : dirty_bow) {
        CCM_CUDA(cudaMemcpyAsync(d_bw.p + r.first, h_bw.data() + r.first, 4 * (size_t)r.second, cudaMemcpyHostToDevice, st));
        CCM_CUDA(cudaMemcpyAsync(d_bv.p + r.first, h_bv.data() + r.first, 8 * (size_t)r.second, cudaMemcpyHostToDevice, st));
      }
    }
    if (post_full || d_post.n < h_post.size()) {
      if (d_post.n < h_post.size()) d_post.alloc(std::max<size_t>(4096, 2 * h_post.size()));
      d_post.upload(h_post.data(), h_post.size(), st);
      std::vector<long long> so(n_words); std::vector<int> sl(n_words);
      for (int w = 0; w < n_words; w++) { so[w] = seg[w].off; sl[w] = seg[w].len; }
      d_seg_off.upload(so.data(), n_words, st); d_seg_len.upload(sl.data(), n_words, st);
    } else {
      const int np = (int)dirty_pos.size(), nw = (int)dirty_word.size();
      if (np) {
        std::vector<int> val(np);
        for (int i = 0; i < np; i++) val[i] = h_post[dirty_pos[i]];
        d_spos.upload(dirty_pos.data(), np, st); d_sval.upload(val.data(), np, st);
        k_scatter_i32<<<div_up(np, TPB), TPB, 0, st>>>(d_post.p, d_spos.p, d_sval.p, np);
        CCM_LAUNCHED();
      }
      if (nw) {
        std::vector<long long> off(nw); std::vector<int> len(nw);
        for (int i = 0; i < nw; i++) { off[i] = seg[dirty_word[i]].off; len[i] = seg[dirty_word[i]].len; }
        d_sword.upload(dirty_word.data(), nw, st); d_soff.upload(off.data(), nw, st); d_slen.upload(len.data(), nw, st);
        k_scatter_seg<<<div_up(nw, TPB), TPB, 0, st>>>(d_seg_off.p, d_seg_len.p, d_sword.p, d_soff.p, d_slen.p, nw);
        CCM_LAUNCHED();
      }
    }
    for (int w : dirty_word) word_dirty[w] = 0;
    dirty_slots.clear(); dirty_bow.clear(); dirty_pos.clear(); dirty_word.clear();
    slots_full = bow_full = post_full = false;
  }
};

namespace {

int check_bow(const char* what, int n, const uint32_t* w, const double* v) {
  CCM_REQUIRE(n >= 0 && (n == 0 || (w && v)), std::string(what) + ": bad BowVector");
  CCM_REQUIRE(n <= MAX_QUERY_WORDS, std::string(what) + ": query BowVector longer than 16384 words");
  for (int i = 1; i < n; i++) CCM_REQUIRE(w[i] > w[i - 1], std::string(what) + ": BowVector words must be strictly ascending");
  return n;
}

// the query pipeline over B queries; results to the host
void run_queries(ccm_kfdb* h, const ccm_kfdb_request* q, int B, ccm_kfdb_result* r) {
  cudaStream_t st = h->stream;
  const int S = h->slots();
  std::vector<int> qptr(B + 1, 0), exptr(B + 1, 0), exslot;
  std::vector<unsigned long long> mask(B);
  int maxnq = 0;
  for (int b = 0; b < B; b++) {
    const int n = check_bow("ccm_kfdb_query", q[b].n, q[b].word, q[b].value);
    qptr[b + 1] = qptr[b] + n; maxnq = std::max(maxnq, n);
    mask[b] = q[b].client_mask;
    CCM_REQUIRE(q[b].n_exclude >= 0 && (q[b].n_exclude == 0 || q[b].exclude_uid), "ccm_kfdb_query: bad exclusion list");
    for (int i = 0; i < q[b].n_exclude; i++) {
      auto it = h->kf.find(q[b].exclude_uid[i]);
      if (it != h->kf.end()) exslot.push_back(it->second.slot);    // not in the database: nothing to hide
    }
    exptr[b + 1] = (int)exslot.size();
  }
  std::vector<uint32_t> qw(qptr[B]); std::vector<double> qv(qptr[B]);
  for (int b = 0; b < B; b++)
    if (q[b].n) { memcpy(&qw[qptr[b]], q[b].word, 4 * (size_t)q[b].n); memcpy(&qv[qptr[b]], q[b].value, 8 * (size_t)q[b].n); }
  for (int b = 0; b < B; b++) r[b].n = 0, r[b].n_sharing = 0, r[b].max_common = 0, r[b].min_common = 0;
  if (S == 0) return;
  h->flush();
  const size_t BS = (size_t)B * S;
  if (h->d_count.n < BS) {
    h->d_count.alloc(BS); h->d_first.alloc(BS); h->d_hidden.alloc(BS); h->d_cslot.alloc(BS); h->d_ckey.alloc(BS);
    h->d_oslot.alloc(BS); h->d_ocount.alloc(BS); h->d_score.alloc(BS);
  }
  h->d_qptr.upload(qptr.data(), B + 1, st); h->d_exptr.upload(exptr.data(), B + 1, st); h->d_mask.upload(mask.data(), B, st);
  if (!exslot.empty()) h->d_exslot.upload(exslot.data(), exslot.size(), st);
  if (qptr[B]) { h->d_qword.upload(qw.data(), qw.size(), st); h->d_qval.upload(qv.data(), qv.size(), st); }
  if (h->d_hdr.n < (size_t)3 * B) h->d_hdr.alloc((size_t)3 * B);
  CCM_CUDA(cudaMemsetAsync(h->d_hdr.p, 0, sizeof(int) * 3 * B, st));
  if (h->timing) CCM_CUDA(cudaEventRecord(h->ev[0], st));
  const int g_slot = grid_for((const void*)k_prepare, 0, S, TPB);
  k_prepare<<<dim3(g_slot, B), TPB, 0, st>>>(S, h->d_slot_client.p, h->d_mask.p, h->d_count.p, h->d_first.p, h->d_hidden.p);
  CCM_LAUNCHED();
  if (!exslot.empty()) {
    k_exclude<<<dim3(1, B), TPB, 0, st>>>(S, h->d_exptr.p, h->d_exslot.p, h->d_hidden.p);
    CCM_LAUNCHED();
  }
  if (maxnq) {
    const int g_count = grid_for((const void*)k_count, 0, maxnq, TPB / 32);
    k_count<<<dim3(g_count, B), TPB, 0, st>>>(S, h->d_qptr.p, h->d_qword.p, h->d_seg_off.p, h->d_seg_len.p, h->d_post.p, h->d_hidden.p,
                                              h->d_count.p, h->d_first.p);
    CCM_LAUNCHED();
  }
  if (h->timing) CCM_CUDA(cudaEventRecord(h->ev[1], st));
  k_max<<<dim3(g_slot, B), TPB, 0, st>>>(S, h->d_count.p, h->d_hdr.p);
  CCM_LAUNCHED();
  k_compact<<<dim3(g_slot, B), TPB, 0, st>>>(S, h->d_count.p, h->d_first.p, h->d_hdr.p, h->d_cslot.p, h->d_ckey.p);
  CCM_LAUNCHED();
  k_rank<<<dim3(grid_for((const void*)k_rank, 0, S, TPB), B), TPB, 0, st>>>(S, h->d_hdr.p, h->d_cslot.p, h->d_ckey.p, h->d_count.p,
                                                                          h->d_oslot.p, h->d_ocount.p);
  CCM_LAUNCHED();
  const size_t smem = (size_t)maxnq * 12;
  allow_score_smem();
  const double log_eps = log(2.220446049250313e-16);                 // GeneralScoring::LOG_EPS = log(DBL_EPSILON)
  k_score<<<dim3(grid_for((const void*)k_score, smem, S, TPB / 32), B), TPB, smem, st>>>(
      S, h->scoring, log_eps, h->d_qptr.p, h->d_qword.p, h->d_qval.p, h->d_hdr.p + 2, 3, h->d_oslot.p, h->d_slot_off.p, h->d_slot_n.p,
      h->d_bw.p, h->d_bv.p, h->d_score.p);
  CCM_LAUNCHED();
  if (h->timing) CCM_CUDA(cudaEventRecord(h->ev[2], st));
  std::vector<int> hdr(3 * B);
  h->d_hdr.download(hdr.data(), 3 * B, st);
  CCM_CUDA(cudaStreamSynchronize(st));
  if (h->timing) {
    float a = 0, c = 0;
    CCM_CUDA(cudaEventElapsedTime(&a, h->ev[0], h->ev[1])); CCM_CUDA(cudaEventElapsedTime(&c, h->ev[1], h->ev[2]));
    h->t_count_ms += a; h->t_score_ms += c; h->timed_queries += B;
  }
  std::vector<std::vector<int>> os(B), oc(B); std::vector<std::vector<double>> sc(B);
  for (int b = 0; b < B; b++) {
    const int n = hdr[3 * b + 2];
    r[b].max_common = hdr[3 * b]; r[b].n_sharing = hdr[3 * b + 1];
    r[b].min_common = (int)((float)hdr[3 * b] * 0.8f);
    r[b].n = n;
    CCM_REQUIRE(n <= r[b].cap && (n == 0 || r[b].cand), "ccm_kfdb_query: result capacity too small (size it ccm_kfdb_size)");
    os[b].resize(n); oc[b].resize(n); sc[b].resize(n);
    if (n) {
      CCM_CUDA(cudaMemcpyAsync(os[b].data(), h->d_oslot.p + (size_t)b * S, 4 * (size_t)n, cudaMemcpyDeviceToHost, st));
      CCM_CUDA(cudaMemcpyAsync(oc[b].data(), h->d_ocount.p + (size_t)b * S, 4 * (size_t)n, cudaMemcpyDeviceToHost, st));
      CCM_CUDA(cudaMemcpyAsync(sc[b].data(), h->d_score.p + (size_t)b * S, 8 * (size_t)n, cudaMemcpyDeviceToHost, st));
    }
  }
  CCM_CUDA(cudaStreamSynchronize(st));
  for (int b = 0; b < B; b++)
    for (int i = 0; i < r[b].n; i++) {
      ccm_kfdb_candidate& c = r[b].cand[i];
      c.uid = h->uid_of_slot[os[b][i]]; c.n_words = oc[b][i]; c.score_f64 = sc[b][i]; c.score = (float)sc[b][i];
    }
}

}  // namespace

extern "C" {

int ccm_kfdb_create(int32_t n_words, int32_t scoring, ccm_kfdb** out) {
  return guarded([&] {
    CCM_REQUIRE(out, "ccm_kfdb_create: null output");
    *out = nullptr;
    CCM_REQUIRE(n_words > 0 && scoring >= 0 && scoring <= 5, "ccm_kfdb_create: bad vocabulary size or scoring type");
    ensure_device();
    std::unique_ptr<ccm_kfdb> h(new ccm_kfdb);
    h->n_words = n_words; h->scoring = scoring;
    h->device = current_device();
    CCM_CUDA(cudaSetDevice(h->device));
    CCM_CUDA(cudaStreamCreateWithFlags(&h->stream, cudaStreamNonBlocking));
    for (auto& e : h->ev) CCM_CUDA(cudaEventCreate(&e));
    h->seg.assign(n_words, Seg{}); h->word_dirty.assign(n_words, 0);
    *out = h.release();
  });
}

void ccm_kfdb_destroy(ccm_kfdb* h) { delete h; }

int ccm_kfdb_add(ccm_kfdb* h, uint64_t uid, uint32_t client, int32_t n, const uint32_t* word, const double* value) {
  return guarded([&] {
    CCM_REQUIRE(h && n >= 0 && (n == 0 || (word && value)), "ccm_kfdb_add: bad argument");
    std::lock_guard<std::mutex> lock(h->mu);
    h->add(uid, client, n, word, value);
  });
}

int ccm_kfdb_erase(ccm_kfdb* h, uint64_t uid) {
  return guarded([&] {
    CCM_REQUIRE(h, "ccm_kfdb_erase: null handle");
    std::lock_guard<std::mutex> lock(h->mu);
    h->erase(uid);
  });
}

int ccm_kfdb_clear(ccm_kfdb* h) {
  return guarded([&] {
    CCM_REQUIRE(h, "ccm_kfdb_clear: null handle");
    std::lock_guard<std::mutex> lock(h->mu);
    h->clear();
  });
}

int64_t ccm_kfdb_size(ccm_kfdb* h) { if (!h) return -1; std::lock_guard<std::mutex> lock(h->mu); return (int64_t)h->kf.size(); }

int ccm_kfdb_query(ccm_kfdb* h, const ccm_kfdb_request* q, ccm_kfdb_result* r) { return ccm_kfdb_query_batch(h, q, 1, r); }

int ccm_kfdb_query_batch(ccm_kfdb* h, const ccm_kfdb_request* q, int32_t nq, ccm_kfdb_result* r) {
  return guarded([&] {
    CCM_REQUIRE(h && nq >= 0 && (nq == 0 || (q && r)), "ccm_kfdb_query_batch: bad argument");
    std::lock_guard<std::mutex> lock(h->mu);
    CCM_CUDA(cudaSetDevice(h->device));
    for (int b0 = 0; b0 < nq; b0 += MAX_BATCH) run_queries(h, q + b0, std::min(MAX_BATCH, nq - b0), r + b0);   // gridDim.y <= 65535
  });
}

int ccm_kfdb_score_many(ccm_kfdb* h, int32_t n, const uint32_t* word, const double* value, int32_t n_uid, const uint64_t* uid,
                        double* score) {
  return guarded([&] {
    CCM_REQUIRE(h && n_uid >= 0 && (n_uid == 0 || (uid && score)), "ccm_kfdb_score_many: bad argument");
    check_bow("ccm_kfdb_score_many", n, word, value);
    std::lock_guard<std::mutex> lock(h->mu);
    CCM_CUDA(cudaSetDevice(h->device));
    if (!n_uid) return;
    std::vector<int> slot(n_uid);
    for (int i = 0; i < n_uid; i++) {
      auto it = h->kf.find(uid[i]);
      CCM_REQUIRE(it != h->kf.end(), "ccm_kfdb_score_many: keyframe not in the database");
      slot[i] = it->second.slot;
    }
    h->flush();
    cudaStream_t st = h->stream;
    const int qp[2] = {0, n};
    h->d_qptr.upload(qp, 2, st);
    h->d_cslot.upload(slot.data(), n_uid, st);
    if (h->d_hdr.n < 3) h->d_hdr.alloc(3);
    const int hd[3] = {0, 0, n_uid};
    h->d_hdr.upload(hd, 3, st);
    if (n) { h->d_qword.upload(word, n, st); h->d_qval.upload(value, n, st); }
    if (h->d_score.n < (size_t)n_uid) h->d_score.alloc(n_uid);
    const size_t smem = (size_t)n * 12;
    allow_score_smem();
    k_score<<<dim3(grid_for((const void*)k_score, smem, n_uid, TPB / 32), 1), TPB, smem, st>>>(
        n_uid, h->scoring, log(2.220446049250313e-16), h->d_qptr.p, h->d_qword.p, h->d_qval.p, h->d_hdr.p + 2, 3, h->d_cslot.p,
        h->d_slot_off.p, h->d_slot_n.p, h->d_bw.p, h->d_bv.p, h->d_score.p);
    CCM_LAUNCHED();
    h->d_score.download(score, n_uid, st);
    CCM_CUDA(cudaStreamSynchronize(st));
  });
}

int ccm_kfdb_set_timing(ccm_kfdb* h, int32_t on) {
  return guarded([&] {
    CCM_REQUIRE(h, "ccm_kfdb_set_timing: null handle");
    std::lock_guard<std::mutex> lock(h->mu);
    h->timing = on != 0; h->t_count_ms = h->t_score_ms = 0; h->timed_queries = 0;
  });
}

int ccm_kfdb_get_timing(ccm_kfdb* h, double* count_ms, double* score_ms, int64_t* queries) {
  return guarded([&] {
    CCM_REQUIRE(h && count_ms && score_ms && queries, "ccm_kfdb_get_timing: null argument");
    std::lock_guard<std::mutex> lock(h->mu);
    *count_ms = h->t_count_ms; *score_ms = h->t_score_ms; *queries = h->timed_queries;
  });
}

// the covisibility accumulation and the retain of S/Database.cpp:148-201 (loop), :273-326 (map match), :388-438 (relocalisation),
// in the reference's float arithmetic, over the device's scored candidates.  Host only.
int ccm_kfdb_select(const ccm_kfdb_result* r, const int32_t* covis_ptr, const uint64_t* covis_uid, int32_t reloc, float min_score,
                    uint64_t* out_uid, int32_t* n_out) {
  return guarded([&] {
    CCM_REQUIRE(r && n_out && (r->n == 0 || (r->cand && covis_ptr && out_uid)), "ccm_kfdb_select: null argument");
    *n_out = 0;
    std::unordered_map<uint64_t, float> scored;                      // mLoopQuery == id && mnLoopWords > minCommonWords -> mLoopScore
    scored.reserve(2 * (size_t)r->n + 1);
    for (int i = 0; i < r->n; i++) scored[r->cand[i].uid] = r->cand[i].score;
    std::vector<std::pair<float, uint64_t>> acc;
    float bestAccScore = reloc ? 0.f : min_score;
    for (int i = 0; i < r->n; i++) {
      const float si = r->cand[i].score;
      if (!reloc && !(si >= min_score)) continue;                   // lScoreAndMatch holds si >= minScore only
      float bestScore = si, accScore = si;
      uint64_t best = r->cand[i].uid;
      for (int k = covis_ptr[i]; k < covis_ptr[i + 1]; k++) {
        auto it = scored.find(covis_uid[k]);
        if (it == scored.end()) continue;
        accScore += it->second;
        if (it->second > bestScore) { best = covis_uid[k]; bestScore = it->second; }
      }
      acc.push_back({accScore, best});
      if (accScore > bestAccScore) bestAccScore = accScore;
    }
    const float minScoreToRetain = 0.75f * bestAccScore;
    std::unordered_set<uint64_t> added;
    for (auto& a : acc)
      if (a.first > minScoreToRetain && added.insert(a.second).second) out_uid[(*n_out)++] = a.second;
  });
}

}  // extern "C"

// ccm_kfdb_double.cpp — the device entry points of ccm_kfdb_* (include/ccm_b200.h) on the CPU, for running shim/Database_shim.cpp
// without a GPU (TEST INFRASTRUCTURE, NOT PRODUCT).  The inverted file is the reference's (push_back per word, first occurrence erased),
// the scores are the oracle's (orc_bow_score, oracle/kfdb_oracle.cpp); the host selection ccm_kfdb_select is the library's own.
// Linked into oracle/_ref/libkfdb_shim.so with -Bsymbolic, so that the shim's calls bind here.
#include <algorithm>
#include <cstdint>
#include <list>
#include <map>
#include <set>
#include <unordered_map>
#include <vector>

#include "../include/ccm_b200.h"

extern "C" double orc_bow_score(int32_t scoring, int32_t n1, const uint32_t* w1, const double* v1, int32_t n2, const uint32_t* w2,
                                const double* v2);

struct ccm_kfdb {
  int scoring;
  std::vector<std::list<uint64_t>> inv;
  struct KF { uint32_t client; std::vector<uint32_t> w; std::vector<double> v; };
  std::unordered_map<uint64_t, KF> kf;
};

namespace {
void query(ccm_kfdb* h, const ccm_kfdb_request& q, ccm_kfdb_result& r) {
  std::set<uint64_t> hidden(q.exclude_uid, q.exclude_uid + q.n_exclude);
  std::vector<uint64_t> order;
  std::unordered_map<uint64_t, int> cnt;
  for (int i = 0; i < q.n; i++)
    for (uint64_t u : h->inv[q.word[i]]) {
      const uint32_t c = h->kf[u].client;
      if (hidden.count(u) || c >= 64 || !((q.client_mask >> c) & 1ull)) continue;
      if (!cnt.count(u)) order.push_back(u);
      cnt[u]++;
    }
  int mx = 0;
  for (auto& kv : cnt) mx = std::max(mx, kv.second);
  const int mn = mx * 0.8f;
  r.n_sharing = (int32_t)order.size(); r.max_common = mx; r.min_common = mn; r.n = 0;
  for (uint64_t u : order) {
    if (cnt[u] <= mn) continue;
    if (r.n < r.cap) {
      const ccm_kfdb::KF& k = h->kf[u];
      const double s = orc_bow_score(h->scoring, q.n, q.word, q.value, (int32_t)k.w.size(), k.w.data(), k.v.data());
      r.cand[r.n] = ccm_kfdb_candidate{u, cnt[u], (float)s, s};
    }
    r.n++;
  }
}
}  // namespace

extern "C" {

int ccm_kfdb_create(int32_t n_words, int32_t scoring, ccm_kfdb** out) {
  *out = new ccm_kfdb;
  (*out)->scoring = scoring;
  (*out)->inv.resize(n_words);
  return CCM_OK;
}
void ccm_kfdb_destroy(ccm_kfdb* h) { delete h; }

int ccm_kfdb_add(ccm_kfdb* h, uint64_t uid, uint32_t client, int32_t n, const uint32_t* word, const double* value) {
  if (h->kf.count(uid) || client >= 64) return CCM_ERR_INVALID;
  h->kf[uid] = ccm_kfdb::KF{client, std::vector<uint32_t>(word, word + n), std::vector<double>(value, value + n)};
  for (int i = 0; i < n; i++) h->inv[word[i]].push_back(uid);
  return CCM_OK;
}

int ccm_kfdb_erase(ccm_kfdb* h, uint64_t uid) {
  auto it = h->kf.find(uid);
  if (it == h->kf.end()) return CCM_OK;
  for (uint32_t w : it->second.w) {
    std::list<uint64_t>& l = h->inv[w];
    for (auto p = l.begin(); p != l.end(); ++p)
      if (*p == uid) { l.erase(p); break; }
  }
  h->kf.erase(it);
  return CCM_OK;
}

int ccm_kfdb_clear(ccm_kfdb* h) {
  for (auto& l : h->inv) l.clear();
  h->kf.clear();
  return CCM_OK;
}

int64_t ccm_kfdb_size(ccm_kfdb* h) { return h ? (int64_t)h->kf.size() : -1; }

int ccm_kfdb_query_batch(ccm_kfdb* h, const ccm_kfdb_request* q, int32_t nq, ccm_kfdb_result* r) {
  int rc = CCM_OK;
  for (int b = 0; b < nq; b++) {
    query(h, q[b], r[b]);
    if (r[b].n > r[b].cap) rc = CCM_ERR_INVALID;
  }
  return rc;
}

int ccm_kfdb_query(ccm_kfdb* h, const ccm_kfdb_request* q, ccm_kfdb_result* r) { return ccm_kfdb_query_batch(h, q, 1, r); }

int ccm_kfdb_score_many(ccm_kfdb* h, int32_t n, const uint32_t* word, const double* value, int32_t n_uid, const uint64_t* uid,
                        double* score) {
  for (int i = 0; i < n_uid; i++) {
    auto it = h->kf.find(uid[i]);
    if (it == h->kf.end()) return CCM_ERR_INVALID;
    score[i] = orc_bow_score(h->scoring, n, word, value, (int32_t)it->second.w.size(), it->second.w.data(), it->second.v.data());
  }
  return CCM_OK;
}

}  // extern "C"

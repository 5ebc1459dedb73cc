// kfdb_oracle.cpp — CPU oracle for the keyframe database's candidate queries (TEST INFRASTRUCTURE, NOT PRODUCT).
//
// Restates, over flat arrays and stand-in keyframe records:
//   DBoW2 scores (L1, L2, ChiSquare, KL, Bhattacharyya, DotProduct)  D/ScoringObject.cpp:18-311  (the merge-join in ascending word order)
//   KeyFrameDatabase::add / erase / clear                               S/Database.cpp:37-70  (push_back per word; first occurrence)
//   DetectLoopCandidates / DetectMapMatchCandidates                     S/Database.cpp:72-327
//   DetectRelocalizationCandidates                                      S/Database.cpp:329-439
// The marker members the queries use as scratch (mLoopQuery, mMatchQuery, mnLoopWords, mLoopScore, mRelocQuery, mnRelocWords,
// mRelocScore) are kept per keyframe and read back by the tests; they start as the reference's constructor leaves them
// (S/KeyFrame.cpp:39,56: the query ids = defpair, the counts 0) and the two scores, which the reference leaves uninitialised, at 0.
// Built as oracle/libkfdb_oracle.so by oracle/kfdb.mk.
#include <cfloat>
#include <cmath>
#include <cstdint>
#include <list>
#include <map>
#include <set>
#include <unordered_map>
#include <utility>
#include <vector>

namespace {

enum Scoring { L1_NORM = 0, L2_NORM = 1, CHI_SQUARE = 2, KL = 3, BHATTACHARYYA = 4, DOT_PRODUCT = 5 };  // D/BowVector.h:45-53
typedef std::map<uint32_t, double> Bow;
const double LOG_EPS = log(DBL_EPSILON);
const uint64_t NONE = ~0ull;   // defpair

double score(int scoring, const Bow& v1, const Bow& v2) {
  Bow::const_iterator v1_it = v1.begin(), v2_it = v2.begin();
  const Bow::const_iterator v1_end = v1.end(), v2_end = v2.end();
  double s = 0;
  if (scoring == KL) {
    while (v1_it != v1_end && v2_it != v2_end) {
      const double vi = v1_it->second, wi = v2_it->second;
      if (v1_it->first == v2_it->first) {
        if (vi != 0 && wi != 0) s += vi * log(vi / wi);
        ++v1_it; ++v2_it;
      } else if (v1_it->first < v2_it->first) {
        s += vi * (log(vi) - LOG_EPS);
        ++v1_it;
      } else {
        v2_it = v2.lower_bound(v1_it->first);
      }
    }
    for (; v1_it != v1_end; ++v1_it)
      if (v1_it->second != 0) s += v1_it->second * (log(v1_it->second) - LOG_EPS);
    return s;
  }
  while (v1_it != v1_end && v2_it != v2_end) {
    const double vi = v1_it->second, wi = v2_it->second;
    if (v1_it->first == v2_it->first) {
      switch (scoring) {
        case L1_NORM: s += fabs(vi - wi) - fabs(vi) - fabs(wi); break;
        case CHI_SQUARE: if (vi + wi != 0.0) s += vi * wi / (vi + wi); break;
        case BHATTACHARYYA: s += sqrt(vi * wi); break;
        default: s += vi * wi;   // L2, DotProduct
      }
      ++v1_it; ++v2_it;
    } else if (v1_it->first < v2_it->first) {
      v1_it = v1.lower_bound(v2_it->first);
    } else {
      v2_it = v2.lower_bound(v1_it->first);
    }
  }
  if (scoring == L1_NORM) s = -s / 2.0;
  else if (scoring == L2_NORM) s = s >= 1 ? 1.0 : 1.0 - sqrt(1.0 - s);
  else if (scoring == CHI_SQUARE) s = 2. * s;
  return s;
}

Bow make_bow(int32_t n, const uint32_t* w, const double* v) {
  Bow b;
  for (int i = 0; i < n; i++) b[w[i]] = v[i];
  return b;
}

struct KF {
  uint64_t uid = 0;
  uint32_t client = 0;
  Bow bow;
  std::vector<KF*> covis;   // GetBestCovisibilityKeyFrames(10)
  uint64_t mLoopQuery = NONE, mMatchQuery = NONE, mRelocQuery = NONE;
  int mnLoopWords = 0, mnRelocWords = 0;
  float mLoopScore = 0.f, mRelocScore = 0.f;
};

}  // namespace

struct orc_kfdb {
  int scoring;
  std::vector<std::list<KF*>> inv;
  std::unordered_map<uint64_t, KF*> kfs;   // every keyframe record, in the database or not
  // the scored list of the last query (for comparison with the device): uid, words, f64 score; max / min common words
  std::vector<uint64_t> s_uid; std::vector<int> s_words; std::vector<double> s_score;
  int max_common = 0, min_common = 0, n_sharing = 0;
  ~orc_kfdb() { for (auto& kv : kfs) delete kv.second; }
  KF* get(uint64_t uid) {
    KF*& p = kfs[uid];
    if (!p) { p = new KF; p->uid = uid; }
    return p;
  }
};

namespace {

// the part of the three queries after lKFsSharingWords: mark = the query-id marker of the kind, words / sc = the count / score
template <class Mark, class Words, class Sc>
int finish(orc_kfdb* db, const Bow& q, uint64_t qid, const std::list<KF*>& lKFsSharingWords, float minScore, bool reloc, Mark mark,
           Words words, Sc sc, uint64_t* out) {
  db->s_uid.clear(); db->s_words.clear(); db->s_score.clear();
  db->n_sharing = (int)lKFsSharingWords.size(); db->max_common = db->min_common = 0;
  if (lKFsSharingWords.empty()) return 0;
  int maxCommonWords = 0;
  for (KF* k : lKFsSharingWords) if (words(k) > maxCommonWords) maxCommonWords = words(k);
  int minCommonWords = maxCommonWords * 0.8f;
  db->max_common = maxCommonWords; db->min_common = minCommonWords;
  std::list<std::pair<float, KF*>> lScoreAndMatch;
  for (KF* k : lKFsSharingWords) {
    if (words(k) > minCommonWords) {
      const double sd = score(db->scoring, q, k->bow);
      float si = sd;
      sc(k) = si;
      db->s_uid.push_back(k->uid); db->s_words.push_back(words(k)); db->s_score.push_back(sd);
      if (reloc || si >= minScore) lScoreAndMatch.push_back(std::make_pair(si, k));
    }
  }
  if (lScoreAndMatch.empty()) return 0;
  std::list<std::pair<float, KF*>> lAccScoreAndMatch;
  float bestAccScore = reloc ? 0 : minScore;
  for (auto& it : lScoreAndMatch) {
    KF* pKFi = it.second;
    float bestScore = it.first, accScore = it.first;
    KF* pBestKF = pKFi;
    for (KF* pKF2 : pKFi->covis) {
      if (reloc) {
        if (mark(pKF2) != qid) continue;
      } else if (!(mark(pKF2) == qid && words(pKF2) > minCommonWords)) {
        continue;
      }
      accScore += sc(pKF2);
      if (sc(pKF2) > bestScore) { pBestKF = pKF2; bestScore = sc(pKF2); }
    }
    lAccScoreAndMatch.push_back(std::make_pair(accScore, pBestKF));
    if (accScore > bestAccScore) bestAccScore = accScore;
  }
  float minScoreToRetain = 0.75f * bestAccScore;
  std::set<KF*> spAlreadyAddedKF;
  int n = 0;
  for (auto& it : lAccScoreAndMatch)
    if (it.first > minScoreToRetain && !spAlreadyAddedKF.count(it.second)) { out[n++] = it.second->uid; spAlreadyAddedKF.insert(it.second); }
  return n;
}

}  // namespace

extern "C" {

double orc_bow_score(int32_t scoring, int32_t n1, const uint32_t* w1, const double* v1, int32_t n2, const uint32_t* w2, const double* v2) {
  return score(scoring, make_bow(n1, w1, v1), make_bow(n2, w2, v2));
}

orc_kfdb* orc_kfdb_create(int32_t n_words, int32_t scoring) {
  orc_kfdb* db = new orc_kfdb;
  db->scoring = scoring;
  db->inv.resize(n_words);
  return db;
}
void orc_kfdb_destroy(orc_kfdb* db) { delete db; }

// a keyframe record (mUniqueId, client = mId.second, mBowVec); it is not in the database until orc_kfdb_add
void orc_kfdb_keyframe(orc_kfdb* db, uint64_t uid, uint32_t client, int32_t n, const uint32_t* w, const double* v) {
  KF* k = db->get(uid);
  k->client = client; k->bow = make_bow(n, w, v);
}
void orc_kfdb_set_covis(orc_kfdb* db, uint64_t uid, int32_t n, const uint64_t* nb) {
  KF* k = db->get(uid);
  k->covis.clear();
  for (int i = 0; i < n; i++) k->covis.push_back(db->get(nb[i]));
}

void orc_kfdb_add(orc_kfdb* db, uint64_t uid) {
  KF* k = db->get(uid);
  for (auto& kv : k->bow) db->inv[kv.first].push_back(k);
}
void orc_kfdb_erase(orc_kfdb* db, uint64_t uid) {
  KF* k = db->get(uid);
  for (auto& kv : k->bow) {
    std::list<KF*>& l = db->inv[kv.first];
    for (auto it = l.begin(); it != l.end(); ++it)
      if (*it == k) { l.erase(it); break; }
  }
}
void orc_kfdb_clear(orc_kfdb* db) {
  const size_t n = db->inv.size();
  db->inv.clear(); db->inv.resize(n);
}

// DetectLoopCandidates(pKF = record q_uid, minScore): connected = GetConnectedKeyFrames(), in_map = the uids of GetMmpKeyFrames()
int32_t orc_kfdb_detect_loop(orc_kfdb* db, uint64_t q_uid, float minScore, int32_t n_conn, const uint64_t* conn, int32_t n_map,
                             const uint64_t* in_map, uint64_t* out) {
  KF* pKF = db->get(q_uid);
  std::set<uint64_t> spConnected(conn, conn + n_conn), mpAllKfsInMap(in_map, in_map + n_map);
  std::list<KF*> lKFsSharingWords;
  for (auto& kv : pKF->bow)
    for (KF* pKFi : db->inv[kv.first]) {
      if (pKFi->uid == pKF->uid) continue;
      if (!mpAllKfsInMap.count(pKFi->uid)) continue;
      if (!(pKFi->mLoopQuery == q_uid)) {
        pKFi->mnLoopWords = 0;
        if (!spConnected.count(pKFi->uid)) { pKFi->mLoopQuery = q_uid; lKFsSharingWords.push_back(pKFi); }
      }
      pKFi->mnLoopWords++;
    }
  return finish(db, pKF->bow, q_uid, lKFsSharingWords, minScore, false, [](KF* k) -> uint64_t& { return k->mLoopQuery; },
                [](KF* k) -> int& { return k->mnLoopWords; }, [](KF* k) -> float& { return k->mLoopScore; }, out);
}

// DetectMapMatchCandidates(pKF = record q_uid, minScore, pMap): assoc = pMap->msuAssClients
int32_t orc_kfdb_detect_map_match(orc_kfdb* db, uint64_t q_uid, float minScore, int32_t n_assoc, const uint32_t* assoc, uint64_t* out) {
  KF* pKF = db->get(q_uid);
  std::set<uint32_t> msuAssClients(assoc, assoc + n_assoc);
  std::list<KF*> lKFsSharingWords;
  for (auto& kv : pKF->bow)
    for (KF* pKFi : db->inv[kv.first]) {
      if (!(pKFi->mMatchQuery == q_uid)) {
        pKFi->mnLoopWords = 0;
        if (!msuAssClients.count(pKFi->client)) { pKFi->mMatchQuery = q_uid; lKFsSharingWords.push_back(pKFi); }
      }
      pKFi->mnLoopWords++;
    }
  return finish(db, pKF->bow, q_uid, lKFsSharingWords, minScore, false, [](KF* k) -> uint64_t& { return k->mMatchQuery; },
                [](KF* k) -> int& { return k->mnLoopWords; }, [](KF* k) -> float& { return k->mLoopScore; }, out);
}

// DetectRelocalizationCandidates(F): F.mId = frame_id, F.mBowVec = (n, w, v)
int32_t orc_kfdb_detect_reloc(orc_kfdb* db, uint64_t frame_id, int32_t n, const uint32_t* w, const double* v, uint64_t* out) {
  const Bow q = make_bow(n, w, v);
  std::list<KF*> lKFsSharingWords;
  for (auto& kv : q)
    for (KF* pKFi : db->inv[kv.first]) {
      if (pKFi->mRelocQuery != frame_id) { pKFi->mnRelocWords = 0; pKFi->mRelocQuery = frame_id; lKFsSharingWords.push_back(pKFi); }
      pKFi->mnRelocWords++;
    }
  return finish(db, q, frame_id, lKFsSharingWords, 0.f, true, [](KF* k) -> uint64_t& { return k->mRelocQuery; },
                [](KF* k) -> int& { return k->mnRelocWords; }, [](KF* k) -> float& { return k->mRelocScore; }, out);
}

// the scored list of the last query: n, then uid / shared words / f64 score per candidate in order; hdr = max, min, sharing
int32_t orc_kfdb_last_scored(const orc_kfdb* db, uint64_t* uid, int32_t* words, double* sc, int32_t* hdr) {
  const int n = (int)db->s_uid.size();
  for (int i = 0; i < n; i++) { uid[i] = db->s_uid[i]; words[i] = db->s_words[i]; sc[i] = db->s_score[i]; }
  hdr[0] = db->max_common; hdr[1] = db->min_common; hdr[2] = db->n_sharing;
  return n;
}

// markers of a record: q[0..2] = mLoopQuery, mMatchQuery, mRelocQuery (~0 = defpair); i[0..1] = mnLoopWords, mnRelocWords;
// f[0..1] = mLoopScore, mRelocScore
void orc_kfdb_markers(orc_kfdb* db, uint64_t uid, uint64_t* q, int32_t* i, float* f) {
  KF* k = db->get(uid);
  q[0] = k->mLoopQuery; q[1] = k->mMatchQuery; q[2] = k->mRelocQuery;
  i[0] = k->mnLoopWords; i[1] = k->mnRelocWords; f[0] = k->mLoopScore; f[1] = k->mRelocScore;
}

}  // extern "C"

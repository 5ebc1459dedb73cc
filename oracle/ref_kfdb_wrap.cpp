// ref_kfdb_wrap.cpp — drives the reference's own cslam::KeyFrameDatabase (cslam/src/Database.cpp, compiled in place) over the
// stand-in records of ref_stub_db/ through the C interface of kfdb_oracle.cpp (ref_ instead of orc_).  TEST INFRASTRUCTURE, NOT PRODUCT.
#include <cslam/Database.h>

#include <cstdint>
#include <unordered_map>

using namespace cslam;

namespace {
typedef boost::shared_ptr<KeyFrame> kfptr;

// a vocabulary of n words with the given scoring object: mvInvertedFile is sized by size() (Database.cpp:32) and score() is the
// reference's ScoringObject.cpp; nothing else of the vocabulary is used by the database
struct SizedVocabulary : public ORBVocabulary {
  SizedVocabulary(int n, DBoW2::ScoringType s) : ORBVocabulary(10, 6, DBoW2::TF_IDF, s) { m_words.resize(n, 0); }
};

struct Db {
  vocptr voc;
  KeyFrameDatabase* db;
  std::unordered_map<uint64_t, kfptr> kfs;
  kfptr get(uint64_t uid) {
    kfptr& p = kfs[uid];
    if (!p) { p.reset(new KeyFrame); p->mUniqueId = uid; p->mId = std::make_pair((size_t)uid, (size_t)0); }
    return p;
  }
  ~Db() {
    for (auto& kv : kfs) { kv.second->mvpCovis.clear(); kv.second->mspConnected.clear(); }   // break the shared_ptr cycles
    delete db;
  }
};

DBoW2::BowVector make_bow(int32_t n, const uint32_t* w, const double* v) {
  DBoW2::BowVector b;
  for (int i = 0; i < n; i++) b[w[i]] = v[i];
  return b;
}

uint64_t first_or_none(const idpair& p) { return p == idpair(defpair) ? ~0ull : (uint64_t)p.first; }

int32_t out_uids(const std::vector<kfptr>& v, uint64_t* out) {
  for (size_t i = 0; i < v.size(); i++) out[i] = v[i]->mUniqueId;
  return (int32_t)v.size();
}
}  // namespace

extern "C" {

void* ref_kfdb_create(int32_t n_words, int32_t scoring) {
  Db* d = new Db;
  d->voc.reset(new SizedVocabulary(n_words, (DBoW2::ScoringType)scoring));
  d->db = new KeyFrameDatabase(d->voc);
  return d;
}
void ref_kfdb_destroy(void* d) { delete static_cast<Db*>(d); }

void ref_kfdb_keyframe(void* d, uint64_t uid, uint32_t client, int32_t n, const uint32_t* w, const double* v) {
  kfptr k = static_cast<Db*>(d)->get(uid);
  k->mId = std::make_pair((size_t)uid, (size_t)client);
  k->mBowVec = make_bow(n, w, v);
}
void ref_kfdb_set_covis(void* d, uint64_t uid, int32_t n, const uint64_t* nb) {
  Db* D = static_cast<Db*>(d);
  kfptr k = D->get(uid);
  k->mvpCovis.clear();
  for (int i = 0; i < n; i++) k->mvpCovis.push_back(D->get(nb[i]));
}
void ref_kfdb_add(void* d, uint64_t uid) { Db* D = static_cast<Db*>(d); D->db->add(D->get(uid)); }
void ref_kfdb_erase(void* d, uint64_t uid) { Db* D = static_cast<Db*>(d); D->db->erase(D->get(uid)); }
void ref_kfdb_clear(void* d) { static_cast<Db*>(d)->db->clear(); }

int32_t ref_kfdb_detect_loop(void* d, uint64_t q_uid, float minScore, int32_t n_conn, const uint64_t* conn, int32_t n_map,
                             const uint64_t* in_map, uint64_t* out) {
  Db* D = static_cast<Db*>(d);
  kfptr q = D->get(q_uid);
  q->mspConnected.clear();
  for (int i = 0; i < n_conn; i++) q->mspConnected.insert(D->get(conn[i]));
  q->mpMap.reset(new Map);
  for (int i = 0; i < n_map; i++) { kfptr k = D->get(in_map[i]); q->mpMap->mmpKeyFrames[k->mId] = k; }
  std::vector<kfptr> r = D->db->DetectLoopCandidates(q, minScore);
  q->mpMap.reset(); q->mspConnected.clear();
  return out_uids(r, out);
}

int32_t ref_kfdb_detect_map_match(void* d, uint64_t q_uid, float minScore, int32_t n_assoc, const uint32_t* assoc, uint64_t* out) {
  Db* D = static_cast<Db*>(d);
  boost::shared_ptr<Map> m(new Map);
  for (int i = 0; i < n_assoc; i++) m->msuAssClients.insert(assoc[i]);
  return out_uids(D->db->DetectMapMatchCandidates(D->get(q_uid), minScore, m), out);
}

int32_t ref_kfdb_detect_reloc(void* d, uint64_t frame_id, int32_t n, const uint32_t* w, const double* v, uint64_t* out) {
  Frame F;
  F.mId = std::make_pair((size_t)frame_id, (size_t)0);
  F.mBowVec = make_bow(n, w, v);
  return out_uids(static_cast<Db*>(d)->db->DetectRelocalizationCandidates(F), out);
}

void ref_kfdb_markers(void* d, uint64_t uid, uint64_t* q, int32_t* i, float* f) {
  kfptr k = static_cast<Db*>(d)->get(uid);
  q[0] = first_or_none(k->mLoopQuery); q[1] = first_or_none(k->mMatchQuery); q[2] = first_or_none(k->mRelocQuery);
  i[0] = k->mnLoopWords; i[1] = k->mnRelocWords; f[0] = k->mLoopScore; f[1] = k->mRelocScore;
}

}  // extern "C"

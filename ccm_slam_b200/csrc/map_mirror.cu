// map_mirror.cu — a persistent flat mirror of the map for the global BA, behind ccm_mirror_* (include/ccm_b200.h); SURVEY.md §8(f)
// rank 1.  Host code only (no kernel in this file): it exists so that a GBA does not re-walk the pointer graph.
//
// The reference flattens the whole map inside every MapFusionGBA call (S/Optimizer.cpp:658-787): GetAllKeyFrames / GetAllMapPoints,
// a GetObservations() std::map copy per point under its mutex, Converter::toSE3Quat per keyframe.  That walk is serial, outside the
// reference's own optimise timer, and becomes the wall-clock of a GBA once optimize() is fast.  The mirror is told about changes
// where they happen (KeyFrame::SetPose, MapPoint::SetWorldPos, AddObservation / EraseObservation, SetBadFlag — INTEGRATION.md) and
// hands ccm_ba_solve a ccm_ba_problem whose arrays it owns:
//   * a value change (pose, position) is O(1) and also patches the problem last handed out;
//   * a structural change (insert / erase / bad flag / observation) marks the problem stale; the next ccm_mirror_ba_problem runs
//     ONE pass over flat arrays (no pointers, no locks, no map copies) that applies the reference's selection rules:
//       keyframes  alive, not bad, uid <= max_kf_uid                       (S/Optimizer.cpp:693-706, :733)
//       edges      both ends selected                                       (S/Optimizer.cpp:727-771; dangling observations are dropped)
//       points     alive, not bad, >= min_edges observations in all and >= min_edges selected edges; min_edges = 2 is MapFusionGBA's
//                  rule (S/Optimizer.cpp:722-740: observations.size() < 2 || nEdges < 2 skips the point), 1 is
//                  BundleAdjustmentClient's (:117-160: nEdges == 0 removes the vertex); ccm_mirror_set_min_edges, default 2
//     edges are emitted grouped by point row (counting sort), the order ccm_ba_create takes without grouping on the host;
//     rows keep first-insertion order (erase + insert again moves to the end), so the result is deterministic — unlike the
//     reference's, whose edge order follows pointer values (SURVEY.md §7 "hard parts"); BA parity is tolerance-based for that reason.
// Poses are converted once per SetPose with ccm_pose_from_Tcw_f32 (Converter::toSE3Quat), points widened f32 -> f64 as
// Converter::toVector3d does.
#include <unordered_map>
#include <vector>

#include "common.cuh"

using namespace ccm;

struct ccm_map_mirror {
  struct KF { uint64_t uid; double pose[7]; double intr[4]; uint8_t bad, alive; int row; };
  struct MP { uint64_t uid; double pos[3]; uint8_t bad, alive; int row; };
  struct Obs { int kf, mp; float u, v, w; uint8_t alive; };     // kf / mp are slots
  std::vector<KF> kfs;
  std::vector<MP> mps;
  std::vector<Obs> obs;
  std::unordered_map<uint64_t, int> kf_slot, mp_slot;
  struct PairHash { size_t operator()(const std::pair<int, int>& p) const { return std::hash<uint64_t>()(((uint64_t)(uint32_t)p.first << 32) | (uint32_t)p.second); } };
  std::unordered_map<std::pair<int, int>, int, PairHash> obs_slot;   // (mp slot, kf slot) -> obs slot
  size_t dead = 0;
  // the problem last handed out
  bool stale = true;
  uint64_t built_max_uid = 0;
  std::vector<uint64_t> built_fixed;
  std::vector<double> poses, intr, points;
  std::vector<uint8_t> fixed;
  std::vector<int32_t> obs_kf, obs_mp;
  std::vector<float> obs_uv, obs_w;
  std::vector<uint64_t> kf_uid_of_row, mp_uid_of_row;
  long long rebuilds = 0;
  int min_edges = 2;

  void compact() {   // drop dead slots once they outnumber the living; slot numbers change, maps are rebuilt
    if (dead * 2 < kfs.size() + mps.size() + obs.size() + 64) return;
    std::vector<int> kmap(kfs.size(), -1), mmap(mps.size(), -1);
    std::vector<KF> nk; std::vector<MP> nm; std::vector<Obs> no;
    for (size_t i = 0; i < kfs.size(); i++) if (kfs[i].alive) { kmap[i] = (int)nk.size(); nk.push_back(kfs[i]); }
    for (size_t i = 0; i < mps.size(); i++) if (mps[i].alive) { mmap[i] = (int)nm.size(); nm.push_back(mps[i]); }
    for (const Obs& o : obs) if (o.alive && kmap[o.kf] >= 0 && mmap[o.mp] >= 0) { Obs c = o; c.kf = kmap[o.kf]; c.mp = mmap[o.mp]; no.push_back(c); }
    kfs.swap(nk); mps.swap(nm); obs.swap(no);
    kf_slot.clear(); mp_slot.clear(); obs_slot.clear();
    for (size_t i = 0; i < kfs.size(); i++) kf_slot[kfs[i].uid] = (int)i;
    for (size_t i = 0; i < mps.size(); i++) mp_slot[mps[i].uid] = (int)i;
    for (size_t i = 0; i < obs.size(); i++) obs_slot[{obs[i].mp, obs[i].kf}] = (int)i;
    dead = 0;
  }

  void build(uint64_t max_kf_uid, const uint64_t* fixed_uid, int n_fixed) {
    compact();
    poses.clear(); intr.clear(); points.clear(); fixed.clear(); obs_kf.clear(); obs_mp.clear(); obs_uv.clear(); obs_w.clear();
    kf_uid_of_row.clear(); mp_uid_of_row.clear();
    for (KF& k : kfs) {
      k.row = -1;
      if (!k.alive || k.bad || k.uid > max_kf_uid) continue;
      k.row = (int)fixed.size();
      poses.insert(poses.end(), k.pose, k.pose + 7); intr.insert(intr.end(), k.intr, k.intr + 4);
      uint8_t fx = 0;
      for (int i = 0; i < n_fixed; i++) fx |= fixed_uid[i] == k.uid;
      fixed.push_back(fx); kf_uid_of_row.push_back(k.uid);
    }
    int nedges_prev = 0;
    std::vector<int> nedges(mps.size(), 0), nobs(mps.size(), 0);
    for (const Obs& o : obs) {
      if (!o.alive || !kfs[o.kf].alive || !mps[o.mp].alive || mps[o.mp].bad) continue;
      nobs[o.mp]++;                                              // observations.size(): every observation the point still holds
      if (kfs[o.kf].row >= 0) nedges[o.mp]++;                    // nEdges: those whose keyframe is in the problem
    }
    std::vector<int> start;                                       // first edge of every point row (counting sort by point row)
    for (size_t i = 0; i < mps.size(); i++) {
      MP& m = mps[i];
      m.row = -1;
      if (!m.alive || m.bad || nobs[i] < min_edges || nedges[i] < min_edges || nedges[i] == 0) continue;
      m.row = (int)mp_uid_of_row.size();
      points.insert(points.end(), m.pos, m.pos + 3); mp_uid_of_row.push_back(m.uid);
      start.push_back(start.empty() ? 0 : start.back() + nedges_prev);
      nedges_prev = nedges[i];
    }
    const size_t E = start.empty() ? 0 : (size_t)start.back() + nedges_prev;
    obs_kf.resize(E); obs_mp.resize(E); obs_uv.resize(2 * E); obs_w.resize(E);
    for (const Obs& o : obs) {                                    // insertion order is kept inside every point's group
      if (!o.alive || !kfs[o.kf].alive || kfs[o.kf].row < 0 || !mps[o.mp].alive || mps[o.mp].row < 0) continue;
      const size_t e = (size_t)start[mps[o.mp].row]++;
      obs_kf[e] = kfs[o.kf].row; obs_mp[e] = mps[o.mp].row;
      obs_uv[2 * e] = o.u; obs_uv[2 * e + 1] = o.v; obs_w[e] = o.w;
    }
    built_max_uid = max_kf_uid; built_fixed.assign(fixed_uid, fixed_uid + n_fixed);
    stale = false; rebuilds++;
  }
};

extern "C" {

int ccm_mirror_create(ccm_map_mirror** out) {
  return guarded([&] { CCM_REQUIRE(out, "ccm_mirror_create: null output"); *out = new ccm_map_mirror(); });
}
void ccm_mirror_destroy(ccm_map_mirror* m) { delete m; }

int ccm_mirror_set_keyframe(ccm_map_mirror* m, uint64_t uid, const float* Tcw, const float* intr4, int32_t bad) {
  return guarded([&] {
    CCM_REQUIRE(m && Tcw, "ccm_mirror_set_keyframe: null argument");
    auto it = m->kf_slot.find(uid);
    if (it == m->kf_slot.end()) {
      CCM_REQUIRE(intr4, "ccm_mirror_set_keyframe: a new keyframe needs its intrinsics");
      ccm_map_mirror::KF k{};
      k.uid = uid; k.alive = 1; k.bad = bad != 0; k.row = -1;
      ccm_pose_from_Tcw_f32(Tcw, 1, k.pose);
      for (int i = 0; i < 4; i++) k.intr[i] = intr4[i];
      m->kf_slot[uid] = (int)m->kfs.size(); m->kfs.push_back(k);
      m->stale = true;
      return;
    }
    ccm_map_mirror::KF& k = m->kfs[it->second];
    ccm_pose_from_Tcw_f32(Tcw, 1, k.pose);
    if (intr4) for (int i = 0; i < 4; i++) {
      if (k.intr[i] != (double)intr4[i]) { k.intr[i] = intr4[i]; if (k.row >= 0 && !m->stale) m->intr[4 * (size_t)k.row + i] = intr4[i]; }
    }
    if ((bad != 0) != (k.bad != 0)) { k.bad = bad != 0; m->stale = true; }
    if (!m->stale && k.row >= 0) for (int i = 0; i < 7; i++) m->poses[7 * (size_t)k.row + i] = k.pose[i];   // value change: patch in place
  });
}

int ccm_mirror_erase_keyframe(ccm_map_mirror* m, uint64_t uid) {
  return guarded([&] {
    CCM_REQUIRE(m, "ccm_mirror_erase_keyframe: null mirror");
    auto it = m->kf_slot.find(uid);
    if (it == m->kf_slot.end()) return;
    m->kfs[it->second].alive = 0; m->kf_slot.erase(it); m->dead++; m->stale = true;   // its observations die with it at the next build / compaction
  });
}

int ccm_mirror_set_point(ccm_map_mirror* m, uint64_t uid, const float* pos3, int32_t bad) {
  return guarded([&] {
    CCM_REQUIRE(m && pos3, "ccm_mirror_set_point: null argument");
    auto it = m->mp_slot.find(uid);
    if (it == m->mp_slot.end()) {
      ccm_map_mirror::MP p{};
      p.uid = uid; p.alive = 1; p.bad = bad != 0; p.row = -1;
      for (int i = 0; i < 3; i++) p.pos[i] = pos3[i];
      m->mp_slot[uid] = (int)m->mps.size(); m->mps.push_back(p);
      return;   // a point without observations does not enter the problem: nothing to rebuild yet
    }
    ccm_map_mirror::MP& p = m->mps[it->second];
    for (int i = 0; i < 3; i++) p.pos[i] = pos3[i];
    if ((bad != 0) != (p.bad != 0)) { p.bad = bad != 0; m->stale = true; }
    if (!m->stale && p.row >= 0) for (int i = 0; i < 3; i++) m->points[3 * (size_t)p.row + i] = p.pos[i];
  });
}

int ccm_mirror_erase_point(ccm_map_mirror* m, uint64_t uid) {
  return guarded([&] {
    CCM_REQUIRE(m, "ccm_mirror_erase_point: null mirror");
    auto it = m->mp_slot.find(uid);
    if (it == m->mp_slot.end()) return;
    m->mps[it->second].alive = 0; m->mp_slot.erase(it); m->dead++; m->stale = true;
  });
}

int ccm_mirror_set_observation(ccm_map_mirror* m, uint64_t kf_uid, uint64_t mp_uid, float u, float v, float inv_sigma2) {
  return guarded([&] {
    CCM_REQUIRE(m, "ccm_mirror_set_observation: null mirror");
    auto k = m->kf_slot.find(kf_uid); auto p = m->mp_slot.find(mp_uid);
    CCM_REQUIRE(k != m->kf_slot.end() && p != m->mp_slot.end(), "ccm_mirror_set_observation: unknown keyframe or point");
    const std::pair<int, int> key(p->second, k->second);
    auto o = m->obs_slot.find(key);
    if (o != m->obs_slot.end() && m->obs[o->second].alive) {       // the same pair again: new measurement, same place
      ccm_map_mirror::Obs& e = m->obs[o->second];
      e.u = u; e.v = v; e.w = inv_sigma2;
      m->stale = true;                                             // edge rows are not tracked per slot: rebuild
      return;
    }
    m->obs_slot[key] = (int)m->obs.size();
    m->obs.push_back(ccm_map_mirror::Obs{k->second, p->second, u, v, inv_sigma2, 1});
    m->stale = true;
  });
}

int ccm_mirror_erase_observation(ccm_map_mirror* m, uint64_t kf_uid, uint64_t mp_uid) {
  return guarded([&] {
    CCM_REQUIRE(m, "ccm_mirror_erase_observation: null mirror");
    auto k = m->kf_slot.find(kf_uid); auto p = m->mp_slot.find(mp_uid);
    if (k == m->kf_slot.end() || p == m->mp_slot.end()) return;
    auto o = m->obs_slot.find({p->second, k->second});
    if (o == m->obs_slot.end()) return;
    m->obs[o->second].alive = 0; m->obs_slot.erase(o); m->dead++; m->stale = true;
  });
}

int ccm_mirror_ba_problem(ccm_map_mirror* m, uint64_t max_kf_uid, const uint64_t* fixed_uid, int32_t n_fixed, ccm_ba_problem* out,
                          const uint64_t** kf_uid_of_row, const uint64_t** mp_uid_of_row) {
  return guarded([&] {
    CCM_REQUIRE(m && out && n_fixed >= 0 && (n_fixed == 0 || fixed_uid), "ccm_mirror_ba_problem: bad argument");
    const bool same_query = !m->stale && m->built_max_uid == max_kf_uid && (int)m->built_fixed.size() == n_fixed &&
                            std::equal(m->built_fixed.begin(), m->built_fixed.end(), fixed_uid);
    if (!same_query) m->build(max_kf_uid, fixed_uid, n_fixed);
    out->K = (int32_t)m->fixed.size(); out->P = (int32_t)m->mp_uid_of_row.size(); out->E = (int32_t)m->obs_kf.size();
    out->poses = m->poses.data(); out->intr = m->intr.data(); out->fixed = m->fixed.data(); out->points = m->points.data();
    out->obs_kf = m->obs_kf.data(); out->obs_mp = m->obs_mp.data(); out->obs_uv = m->obs_uv.data(); out->obs_w = m->obs_w.data();
    out->edge_flags = nullptr;
    if (kf_uid_of_row) *kf_uid_of_row = m->kf_uid_of_row.data();
    if (mp_uid_of_row) *mp_uid_of_row = m->mp_uid_of_row.data();
  });
}

long long ccm_mirror_rebuilds(const ccm_map_mirror* m) { return m ? m->rebuilds : -1; }

int ccm_mirror_set_min_edges(ccm_map_mirror* m, int32_t min_edges) {
  return guarded([&] {
    CCM_REQUIRE(m && (min_edges == 1 || min_edges == 2), "ccm_mirror_set_min_edges: 1 (BundleAdjustmentClient) or 2 (MapFusionGBA)");
    if (m->min_edges != min_edges) { m->min_edges = min_edges; m->stale = true; }
  });
}

}  // extern "C"

// Optimizer_shim.cpp — reference-side translation unit: keeps cslam/include/cslam/Optimizer.h byte-identical and replaces
// cslam/src/Optimizer.cpp for the entry points on the BA hot path.  Everything g2o did between "graph built" and "results
// read back" is one call into libccm_b200.so; graph selection and write-back keep the reference's rules.
//
// It is the binding a maintainer adds to cslam/CMakeLists.txt in place of src/Optimizer.cpp (see INTEGRATION.md).  In this repository
// it is compiled against the reference's own Optimizer.h / Converter.h and stand-in Map / KeyFrame / MapPoint / Frame classes and run
// through the class interface by tests/test_shim_optimizer.py (oracle/Makefile: _ref/liboptimizer_shim.so).
// g2o is only needed for the g2o::Sim3 value type that appears in Optimizer.h.
#include <cslam/Optimizer.h>

#include <unistd.h>

#include <list>
#include <mutex>
#include <unordered_map>

#include "MapPoint_shim.h"
#include "ccm_b200.h"

namespace cslam {

// shim/MapPoint_shim.cpp defines these.  A build that keeps the reference's own MapPoint.cpp links the no-ops below instead: the
// write-back loops then leave every UpdateNormalAndDepth() to the reference body, point by point.
__attribute__((weak)) void ccm_b200_prepare_normals(const vector<boost::shared_ptr<MapPoint> >&, const float*) {}
__attribute__((weak)) void ccm_b200_clear_normals() {}

namespace {

struct FlatBA {
  std::vector<double> poses, intr, points;
  std::vector<uint8_t> fixed;
  std::vector<int32_t> obs_kf, obs_mp;
  std::vector<float> obs_uv, obs_w;
  std::vector<KeyFrame*> kf_of_row;   // raw pointers only for index lookup during flattening
  std::unordered_map<KeyFrame*, int> row_of_kf;

  int add_kf(const boost::shared_ptr<KeyFrame>& pKF, bool fix) {
    const int row = (int)kf_of_row.size();
    row_of_kf[pKF.get()] = row;
    kf_of_row.push_back(pKF.get());
    cv::Mat T = pKF->GetPose();                       // 4x4 CV_32F, Converter::toSE3Quat(pKF->GetPose())
    double qt[7];
    ccm_pose_from_Tcw_f32(T.ptr<float>(0), 1, qt);     // same R->q branches + normalisation as g2o::SE3Quat(R, t)
    poses.insert(poses.end(), qt, qt + 7);
    intr.push_back(pKF->fx); intr.push_back(pKF->fy); intr.push_back(pKF->cx); intr.push_back(pKF->cy);
    fixed.push_back(fix ? 1 : 0);
    return row;
  }
  int add_mp(const boost::shared_ptr<MapPoint>& pMP) {
    cv::Mat X = pMP->GetWorldPos();
    for (int i = 0; i < 3; i++) points.push_back(X.at<float>(i));
    return (int)points.size() / 3 - 1;
  }
  void add_obs(int kf_row, int mp_row, const boost::shared_ptr<KeyFrame>& pKF, size_t idx) {
    const cv::KeyPoint& kpUn = pKF->mvKeysUn[idx];
    obs_kf.push_back(kf_row); obs_mp.push_back(mp_row);
    obs_uv.push_back(kpUn.pt.x); obs_uv.push_back(kpUn.pt.y);
    obs_w.push_back(pKF->mvInvLevelSigma2[kpUn.octave]);
  }
  ccm_ba_problem problem(const uint8_t* flags = nullptr) const {
    ccm_ba_problem p;
    p.K = (int32_t)fixed.size(); p.P = (int32_t)points.size() / 3; p.E = (int32_t)obs_kf.size();
    p.poses = poses.data(); p.intr = intr.data(); p.fixed = fixed.data(); p.points = points.data();
    p.obs_kf = obs_kf.data(); p.obs_mp = obs_mp.data(); p.obs_uv = obs_uv.data(); p.obs_w = obs_w.data();
    p.edge_flags = flags;
    return p;
  }
};

cv::Mat pose_to_cv(const double* qt) {
  cv::Mat T(4, 4, CV_32F);
  ccm_pose_to_Tcw_f32(qt, 1, T.ptr<float>(0));          // Converter::toCvMat(SE3Quat): homogeneous matrix rounded to f32
  return T;
}
cv::Mat point_to_cv(const double* x) {
  cv::Mat X(3, 1, CV_32F);
  for (int i = 0; i < 3; i++) X.at<float>(i) = (float)x[i];
  return X;
}
// the points a write-back loop is about to SetWorldPos + UpdateNormalAndDepth, with the f32 positions they will take
struct NormalBatch {
  vector<boost::shared_ptr<MapPoint> > mps;
  vector<float> pos;
  void add(const boost::shared_ptr<MapPoint>& pMP, const double* x) { mps.push_back(pMP); for (int i = 0; i < 3; i++) pos.push_back((float)x[i]); }
  void prepare() const { ccm_b200_prepare_normals(mps, pos.data()); }
};
void check(int rc) { if (rc != CCM_OK) { std::cerr << "libccm_b200: " << ccm_last_error() << std::endl; throw estd::infrastructure_ex(); } }

// Optional persistent mirrors (INTEGRATION.md 4a, SURVEY.md 8(f) rank 1): a server that keeps a ccm_map_mirror up to date for a Map
// registers it here; MapFusionGBA then takes the flat problem from the mirror instead of walking the pointer graph.
// With the mirror comes a cached solver handle: as long as the mirror did not have to rebuild its flat arrays (values changed, the
// structure did not), the next global BA keeps the device-resident structure and uploads the estimate only (ccm_ba_set_estimate).
struct MirrorEntry {
  ccm_map_mirror* mirror = nullptr;
  ccm_ba_handle* handle = nullptr;
  long long rebuilds = -1;                 // ccm_mirror_rebuilds() when the handle was created
  uint64_t max_uid = 0, fixed_uid = 0;
};
std::mutex g_mirror_mu;
std::unordered_map<const Map*, MirrorEntry> g_mirrors;
MirrorEntry* mirror_of(const Map* m) {
  std::lock_guard<std::mutex> lock(g_mirror_mu);
  auto it = g_mirrors.find(m);
  return it == g_mirrors.end() ? nullptr : &it->second;   // (entries are stable: unordered_map never moves its nodes)
}

}  // namespace

void ccm_b200_register_mirror(const Map* map, ccm_map_mirror* mirror) {   // cslam::ccm_b200_register_mirror; mirror == nullptr: forget the map
  std::lock_guard<std::mutex> lock(g_mirror_mu);
  auto it = g_mirrors.find(map);
  if (it != g_mirrors.end()) {
    if (it->second.handle) ccm_ba_destroy(it->second.handle);   // the cached solver state goes with the registration
    g_mirrors.erase(it);
  }
  if (mirror) g_mirrors[map].mirror = mirror;
}

// ---- MapFusionGBA (S/Optimizer.cpp:646-859) ---------------------------------------------------------------------------
void Optimizer::MapFusionGBA(mapptr pMap, size_t ClientId, int nIterations, bool* pbStopFlag, idpair nLoopKF, const bool bRobust) {
  (void)ClientId;
  vector<kfptr> vpKFs = pMap->GetAllKeyFrames();
  vector<mpptr> vpMP = pMap->GetAllMapPoints();
  const idpair zeropair = make_pair(0, pMap->mMapId);
  if (pMap->mvpKeyFrameOrigins.empty()) throw infrastructure_ex();
  const idpair FixedId = (*(pMap->mvpKeyFrameOrigins.begin()))->mId;

  if (MirrorEntry* ent = mirror_of(pMap.get())) {
    ccm_map_mirror* mir = ent->mirror;
    // The mirror already holds the flat arrays (same selection rules, tests/test_map_mirror.py): no GetObservations() copies, no
    // Converter::toSE3Quat per keyframe.  Only the id -> object tables of the write-back are built here: O(K + P), no observation walk.
    std::unordered_map<uint64_t, kfptr> kf_of_uid;
    std::unordered_map<uint64_t, mpptr> mp_of_uid;
    size_t maxKFid = 0;
    uint64_t fixed_uid = 0;
    for (kfptr pKF : vpKFs) {
      if (pKF->isBad()) continue;
      kf_of_uid[(uint64_t)pKF->mUniqueId] = pKF;
      maxKFid = std::max(maxKFid, (size_t)pKF->mUniqueId);
      if (pKF->mId == FixedId) fixed_uid = (uint64_t)pKF->mUniqueId;
    }
    for (mpptr pMP : vpMP) if (!pMP->isBad()) mp_of_uid[(uint64_t)pMP->mUniqueId] = pMP;
    ccm_ba_problem prob;
    const uint64_t *kf_uid = nullptr, *mp_uid = nullptr;
    check(ccm_mirror_ba_problem(mir, (uint64_t)maxKFid, &fixed_uid, 1, &prob, &kf_uid, &mp_uid));
    ccm_ba_options opt = {};
    opt.iterations = nIterations; opt.robust = bRobust;
    opt.huber_delta = (double)(float)sqrt(5.99);
    opt.stop = reinterpret_cast<const volatile uint8_t*>(pbStopFlag);
    vector<double> poses((size_t)prob.K * 7), points((size_t)prob.P * 3);
    ccm_ba_result res = {};
    res.poses = poses.data(); res.points = points.data();
    const long long gen = ccm_mirror_rebuilds(mir);
    if (ent->handle && ent->rebuilds == gen && ent->max_uid == (uint64_t)maxKFid && ent->fixed_uid == fixed_uid) {
      check(ccm_ba_set_estimate(ent->handle, prob.poses, prob.points));   // same structure: the device keeps it, only the values travel
    } else {
      if (ent->handle) { ccm_ba_destroy(ent->handle); ent->handle = nullptr; }
      check(ccm_ba_create(&prob, &ent->handle));
      ent->rebuilds = gen; ent->max_uid = (uint64_t)maxKFid; ent->fixed_uid = fixed_uid;
    }
    const int rc = ccm_ba_optimize(ent->handle, &opt, &res);
    if (rc != CCM_OK) { ccm_ba_destroy(ent->handle); ent->handle = nullptr; check(rc); }
    for (int r = 0; r < prob.K; r++) {                        // write-back by id, as the reference does (:803-823)
      auto it = kf_of_uid.find(kf_uid[r]);
      if (it == kf_of_uid.end() || it->second->isBad()) continue;
      cv::Mat T = pose_to_cv(&poses[7 * (size_t)r]);
      if (nLoopKF == zeropair) it->second->SetPose(T, true);
      else { it->second->mTcwGBA.create(4, 4, CV_32F); T.copyTo(it->second->mTcwGBA); it->second->mBAGlobalForKF = nLoopKF; }
    }
    ParkedNormalsGuard parked_normals;
    if (nLoopKF == zeropair) {                                // every UpdateNormalAndDepth() below in one device call
      NormalBatch nb;
      for (int r = 0; r < prob.P; r++) {
        auto it = mp_of_uid.find(mp_uid[r]);
        if (it != mp_of_uid.end() && !it->second->isBad()) nb.add(it->second, &points[3 * (size_t)r]);
      }
      nb.prepare();
    }
    for (int r = 0; r < prob.P; r++) {                        // :827-857
      auto it = mp_of_uid.find(mp_uid[r]);
      if (it == mp_of_uid.end() || it->second->isBad()) continue;
      cv::Mat X = point_to_cv(&points[3 * (size_t)r]);
      if (nLoopKF == zeropair) { it->second->SetWorldPos(X, true); it->second->UpdateNormalAndDepth(); }
      else { it->second->mPosGBA.create(3, 1, CV_32F); X.copyTo(it->second->mPosGBA); it->second->mBAGlobalForKF = nLoopKF; }
    }
    return;
  }

  FlatBA f;
  size_t maxKFid = 0;
  // kf_row[i]: row of vpKFs[i] in the flat problem, -1 if skipped.  The write-back looks rows up here (the reference looks every
  // vertex up by id, :805): GBA runs in its own thread while culling continues, so a keyframe may turn bad between flatten and
  // write-back, and a running row counter would then hand every later keyframe its neighbour's pose.
  vector<int> kf_row(vpKFs.size(), -1);
  for (size_t i = 0; i < vpKFs.size(); i++) {                 // keyframe vertices, :695-709
    kfptr pKF = vpKFs[i];
    if (pKF->isBad()) continue;
    kf_row[i] = f.add_kf(pKF, pKF->mId == FixedId);
    maxKFid = std::max(maxKFid, (size_t)pKF->mUniqueId);
  }
  vector<int> mp_row(vpMP.size(), -1);
  for (size_t i = 0; i < vpMP.size(); i++) {                  // landmark vertices + edges, :715-787
    mpptr pMP = vpMP[i];
    if (pMP->isBad()) continue;
    const map<kfptr, size_t> observations = pMP->GetObservations();
    int nEdges = 0;
    for (auto& ob : observations) {
      kfptr pKF = ob.first;
      if (!pKF || pKF->isBad() || pKF->mUniqueId > maxKFid || !f.row_of_kf.count(pKF.get())) continue;  // dangling edges dropped
      nEdges++;
    }
    if (observations.size() < 2 || nEdges < 2) continue;
    mp_row[i] = f.add_mp(pMP);
    for (auto& ob : observations) {
      kfptr pKF = ob.first;
      if (!pKF || pKF->isBad() || pKF->mUniqueId > maxKFid || !f.row_of_kf.count(pKF.get())) continue;
      f.add_obs(f.row_of_kf[pKF.get()], mp_row[i], pKF, ob.second);
    }
  }

  ccm_ba_problem prob = f.problem();
  ccm_ba_options opt = {};
  opt.iterations = nIterations; opt.robust = bRobust;
  opt.huber_delta = (double)(float)sqrt(5.99);               // const float thHuber2D = sqrt(5.99), :712
  opt.stop = reinterpret_cast<const volatile uint8_t*>(pbStopFlag);   // optimizer.setForceStopFlag(pbStopFlag)
  vector<double> poses(f.poses.size()), points(f.points.size());
  ccm_ba_result res = {};
  res.poses = poses.data(); res.points = points.data();
  check(ccm_ba_solve(&prob, &opt, &res));                     // == initializeOptimization(); optimize(nIterations)

  for (size_t i = 0; i < vpKFs.size(); i++) {                 // write-back, :803-823
    kfptr pKF = vpKFs[i];
    if (kf_row[i] < 0 || pKF->isBad()) continue;
    cv::Mat T = pose_to_cv(&poses[7 * (size_t)kf_row[i]]);
    if (nLoopKF == zeropair) pKF->SetPose(T, true);
    else { pKF->mTcwGBA.create(4, 4, CV_32F); T.copyTo(pKF->mTcwGBA); pKF->mBAGlobalForKF = nLoopKF; }
  }
  ParkedNormalsGuard parked_normals;
  if (nLoopKF == zeropair) {
    NormalBatch nb;
    for (size_t i = 0; i < vpMP.size(); i++)
      if (mp_row[i] >= 0 && !vpMP[i]->isBad()) nb.add(vpMP[i], &points[3 * (size_t)mp_row[i]]);
    nb.prepare();
  }
  for (size_t i = 0; i < vpMP.size(); i++) {                  // :827-857
    if (mp_row[i] < 0) continue;
    mpptr pMP = vpMP[i];
    if (pMP->isBad()) continue;
    cv::Mat X = point_to_cv(&points[3 * (size_t)mp_row[i]]);
    if (nLoopKF == zeropair) { pMP->SetWorldPos(X, true); pMP->UpdateNormalAndDepth(); }
    else { pMP->mPosGBA.create(3, 1, CV_32F); X.copyTo(pMP->mPosGBA); pMP->mBAGlobalForKF = nLoopKF; }
  }
}

// ---- BundleAdjustmentClient / GlobalBundleAdjustemntClient (S/Optimizer.cpp:32-212) -------------------------------------
void Optimizer::GlobalBundleAdjustemntClient(mapptr pMap, size_t ClientId, int nIterations, bool* pbStopFlag, const idpair nLoopKF, const bool bRobust) {
  BundleAdjustmentClient(pMap->GetAllKeyFrames(), pMap->GetAllMapPoints(), ClientId, nIterations, pbStopFlag, nLoopKF, bRobust);
}

void Optimizer::BundleAdjustmentClient(const vector<kfptr>& vpKFs, const vector<mpptr>& vpMP, size_t ClientId, int nIterations,
                                       bool* pbStopFlag, const idpair nLoopKF, const bool bRobust) {
  const idpair zeropair = make_pair(0, ClientId);
  FlatBA f;
  vector<int> kf_row(vpKFs.size(), -1);                       // as in MapFusionGBA: rows by table, not by a running counter
  for (size_t i = 0; i < vpKFs.size(); i++) {
    kfptr pKF = vpKFs[i];
    if (pKF->isBad()) continue;
    if (pKF->mId.first >= IDRANGE) throw infrastructure_ex();
    kf_row[i] = f.add_kf(pKF, pKF->mId == zeropair);
  }
  vector<int> mp_row(vpMP.size(), -1);
  for (size_t i = 0; i < vpMP.size(); i++) {
    mpptr pMP = vpMP[i];
    if (pMP->isBad()) continue;
    if (pMP->mId.first >= IDRANGE) throw infrastructure_ex();
    const map<kfptr, size_t> observations = pMP->GetObservations();
    int row = -1;
    for (auto& ob : observations) {
      kfptr pKF = ob.first;
      if (pKF->isBad() || !f.row_of_kf.count(pKF.get())) continue;
      if (row < 0) row = f.add_mp(pMP);
      f.add_obs(f.row_of_kf[pKF.get()], row, pKF, ob.second);
    }
    mp_row[i] = row;                                          // vbNotIncludedMP[i] == (row < 0)
  }
  ccm_ba_problem prob = f.problem();
  ccm_ba_options opt = {};
  opt.iterations = nIterations; opt.robust = bRobust; opt.huber_delta = (double)(float)sqrt(5.99);
  opt.stop = reinterpret_cast<const volatile uint8_t*>(pbStopFlag);
  vector<double> poses(f.poses.size()), points(f.points.size());
  ccm_ba_result res = {};
  res.poses = poses.data(); res.points = points.data();
  check(ccm_ba_solve(&prob, &opt, &res));
  for (size_t i = 0; i < vpKFs.size(); i++) {
    kfptr pKF = vpKFs[i];
    if (kf_row[i] < 0 || pKF->isBad()) continue;
    cv::Mat T = pose_to_cv(&poses[7 * (size_t)kf_row[i]]);
    if (nLoopKF == zeropair) pKF->SetPose(T, false);
    else { pKF->mTcwGBA.create(4, 4, CV_32F); T.copyTo(pKF->mTcwGBA); pKF->mBAGlobalForKF = nLoopKF; }
  }
  ParkedNormalsGuard parked_normals;
  if (nLoopKF == zeropair) {
    NormalBatch nb;
    for (size_t i = 0; i < vpMP.size(); i++)
      if (mp_row[i] >= 0 && !vpMP[i]->isBad()) nb.add(vpMP[i], &points[3 * (size_t)mp_row[i]]);
    nb.prepare();
  }
  for (size_t i = 0; i < vpMP.size(); i++) {
    if (mp_row[i] < 0 || vpMP[i]->isBad()) continue;
    cv::Mat X = point_to_cv(&points[3 * (size_t)mp_row[i]]);
    if (nLoopKF == zeropair) { vpMP[i]->SetWorldPos(X, false); vpMP[i]->UpdateNormalAndDepth(); }
    else { vpMP[i]->mPosGBA.create(3, 1, CV_32F); X.copyTo(vpMP[i]->mPosGBA); vpMP[i]->mBAGlobalForKF = nLoopKF; }
  }
}

// ---- LocalBundleAdjustmentClient (S/Optimizer.cpp:349-644) --------------------------------------------------------------
void Optimizer::LocalBundleAdjustmentClient(kfptr pKF, bool* pbStopFlag, mapptr pMap, size_t ClientId, eSystemState SysState) {
  // window selection exactly as the reference (:351-404): current KF + covisibles are local, their points are local,
  // other observers of those points are fixed
  list<kfptr> lLocalKeyFrames; lLocalKeyFrames.push_back(pKF); pKF->mBALocalForKF = pKF->mId;
  for (kfptr pKFi : pKF->GetVectorCovisibleKeyFrames()) { pKFi->mBALocalForKF = pKF->mId; if (!pKFi->isBad()) lLocalKeyFrames.push_back(pKFi); }
  list<mpptr> lLocalMapPoints;
  for (kfptr k : lLocalKeyFrames)
    for (mpptr pMP : k->GetMapPointMatches())
      if (pMP && !pMP->isBad() && pMP->mBALocalForKF != pKF->mId) { lLocalMapPoints.push_back(pMP); pMP->mBALocalForKF = pKF->mId; }
  list<kfptr> lFixedCameras;
  for (mpptr pMP : lLocalMapPoints)
    for (auto& ob : pMP->GetObservations()) {
      kfptr pKFi = ob.first;
      if (pKFi->mBALocalForKF != pKF->mId && pKFi->mBAFixedForKF != pKF->mId) { pKFi->mBAFixedForKF = pKF->mId; if (!pKFi->isBad()) lFixedCameras.push_back(pKFi); }
    }

  FlatBA f;
  for (kfptr k : lLocalKeyFrames) { if (k->mId.first >= IDRANGE) throw infrastructure_ex(); f.add_kf(k, k->mId.first == 0 && k->mId.second == ClientId); }
  for (kfptr k : lFixedCameras) { if (k->mId.first >= IDRANGE) throw infrastructure_ex(); f.add_kf(k, true); }
  vector<kfptr> vpEdgeKF; vector<mpptr> vpEdgeMP;
  vector<mpptr> mp_rows;
  for (mpptr pMP : lLocalMapPoints) {
    if (pMP->mId.first >= IDRANGE) throw infrastructure_ex();
    const int row = f.add_mp(pMP); mp_rows.push_back(pMP);
    for (auto& ob : pMP->GetObservations()) {
      kfptr pKFi = ob.first;
      if (pKFi->isBad() || !f.row_of_kf.count(pKFi.get())) continue;
      f.add_obs(f.row_of_kf[pKFi.get()], row, pKFi, ob.second);
      vpEdgeKF.push_back(pKFi); vpEdgeMP.push_back(pMP);
    }
  }
  if (pbStopFlag && *pbStopFlag) return;                        // :530-532

  const size_t E = f.obs_kf.size();
  ccm_ba_problem prob = f.problem();
  ccm_ba_handle* h = nullptr;
  check(ccm_ba_create(&prob, &h));
  struct HandleGuard {                                          // every exit path (check() throws on OOM / CUDA errors) destroys the handle
    ccm_ba_handle* h;
    ~HandleGuard() { if (h) ccm_ba_destroy(h); }
  } guard{h};
  ccm_ba_options opt = {};
  opt.robust = 1; opt.huber_delta = (double)(float)sqrt(5.991);  // const float thHuberMono = sqrt(5.991), :468
  opt.stop = reinterpret_cast<const volatile uint8_t*>(pbStopFlag);
  vector<double> poses(f.poses.size()), points(f.points.size()), chi2(E, 0.0);
  vector<uint8_t> depth(E, 1), flags(E, 0);
  ccm_ba_result res = {};
  res.poses = poses.data(); res.points = points.data(); res.chi2 = chi2.data(); res.depth_pos = depth.data();
  opt.iterations = 5;
  check(ccm_ba_optimize(h, &opt, &res));                        // optimizer.optimize(5), :537
  const bool bDoMore = !(pbStopFlag && *pbStopFlag);
  if (bDoMore) {
    for (size_t i = 0; i < E; i++) {                            // :548-562
      if (vpEdgeMP[i]->isBad()) continue;                       // such edges keep level 0 and their kernel
      if (chi2[i] > 5.991 || !depth[i]) flags[i] |= 1;          // e->setLevel(1)
      flags[i] |= 2;                                            // e->setRobustKernel(0)
    }
    check(ccm_ba_set_edge_flags(h, flags.data()));              // initializeOptimization(0)
    opt.iterations = 10;
    check(ccm_ba_optimize(h, &opt, &res));                      // chi2 of level-1 edges keeps its round-1 value (res.chi2 untouched there)
  }
  ccm_ba_destroy(h); guard.h = nullptr;

  vector<pair<kfptr, mpptr>> vToErase;
  for (size_t i = 0; i < E; i++) {                              // :573-587
    if (vpEdgeMP[i]->isBad()) continue;
    if (chi2[i] > 5.991 || !depth[i]) vToErase.push_back(make_pair(vpEdgeKF[i], vpEdgeMP[i]));
  }
  if (SysState != eSystemState::SERVER) while (!pMap->LockMapUpdate()) { usleep(params::timings::miLockSleep); }
  for (auto& e : vToErase) { e.first->EraseMapPointMatch(e.second); e.second->EraseObservation(e.first); }
  size_t row = 0;
  for (kfptr k : lLocalKeyFrames) { k->SetPose(pose_to_cv(&poses[7 * row++]), false); k->mbUpdatedByServer = false; }
  ParkedNormalsGuard parked_normals;
  {
    NormalBatch nb;
    for (size_t i = 0; i < mp_rows.size(); i++)
      if (!mp_rows[i]->isBad()) nb.add(mp_rows[i], &points[3 * i]);
    nb.prepare();
  }
  for (size_t i = 0; i < mp_rows.size(); i++) {
    mpptr pMP = mp_rows[i];
    if (pMP->isBad()) { if (pMap->GetMpPtr(pMP->mId)) throw estd::infrastructure_ex(); continue; }
    pMP->SetWorldPos(point_to_cv(&points[3 * i]), false);
    pMP->UpdateNormalAndDepth();
  }
  if (SysState != eSystemState::SERVER) pMap->UnLockMapUpdate();
}

// ---- OptimizeEssentialGraph* (S/Optimizer.cpp:1058-1566) ----------------------------------------------------------------
// Both variants build the same kind of graph — one Sim3 vertex per keyframe (fixed: the loop keyframe), identity-information edges
// Sji = Sjw * Swi for the new loop connections, the spanning tree, earlier loop edges and strong covisibility — and differ in where
// the poses come from (the loop-closure variant looks keyframes up in CorrectedSim3 / NonCorrectedSim3 first) and in which
// "corrected by" tag of a map point names its reference.  Graph collection and recovery follow the reference's loops; the
// optimisation between them is one ccm_pgo_solve.
namespace {

void sim3_flat(const g2o::Sim3& S, double* o) {
  o[0] = S.rotation().x(); o[1] = S.rotation().y(); o[2] = S.rotation().z(); o[3] = S.rotation().w();
  o[4] = S.translation()[0]; o[5] = S.translation()[1]; o[6] = S.translation()[2]; o[7] = S.scale();
}

void optimize_essential_graph(Optimizer::mapptr pMap, Optimizer::kfptr pLoopKF, Optimizer::kfptr pCurKF,
                              const Optimizer::KeyFrameAndPose* NonCorrectedSim3, const Optimizer::KeyFrameAndPose* CorrectedSim3,
                              const map<Optimizer::kfptr, set<Optimizer::kfptr> >& LoopConnections, bool bFixScale) {
  typedef Optimizer::kfptr kfptr;
  typedef Optimizer::mpptr mpptr;
  typedef Optimizer::KeyFrameAndPose KeyFrameAndPose;
  const vector<kfptr> kfs = pMap->GetAllKeyFrames();
  const vector<mpptr> mps = pMap->GetAllMapPoints();
  const int min_weight = params::opt::miEssGraphMinFeats;

  // vertices, :1086-1118 / :1360-1384.  Rows in ascending mUniqueId = the order of g2o's index mapping.
  map<size_t, g2o::Sim3> S_cw;
  map<size_t, int> row_of_id;
  for (size_t i = 0; i < kfs.size(); i++) {
    kfptr pKF = kfs[i];
    if (pKF->isBad()) continue;
    const size_t id_i = pKF->mUniqueId;
    KeyFrameAndPose::const_iterator it;
    if (CorrectedSim3 && (it = CorrectedSim3->find(pKF)) != CorrectedSim3->end()) S_cw[id_i] = it->second;
    else S_cw[id_i] = g2o::Sim3(Converter::toMatrix3d(pKF->GetRotation()), Converter::toVector3d(pKF->GetTranslation()), 1.0);
  }
  std::vector<double> sim3(8 * S_cw.size());
  std::vector<uint8_t> fixed(S_cw.size(), 0);
  {
    int row = 0;
    for (map<size_t, g2o::Sim3>::const_iterator it = S_cw.begin(); it != S_cw.end(); ++it, ++row) {
      row_of_id[it->first] = row;
      sim3_flat(it->second, &sim3[8 * (size_t)row]);
    }
  }
  if (row_of_id.count(pLoopKF->mUniqueId)) fixed[row_of_id[pLoopKF->mUniqueId]] = 1;

  std::vector<int32_t> ei, ej;
  std::vector<double> meas;
  auto in_graph = [&](const kfptr& k) { return row_of_id.count(k->mUniqueId) != 0; };
  auto add_edge = [&](const kfptr& kfi, const kfptr& pKFj, const g2o::Sim3& Sji) {   // vertex 0 = i, vertex 1 = j
    ei.push_back(row_of_id[kfi->mUniqueId]); ej.push_back(row_of_id[pKFj->mUniqueId]);
    meas.resize(meas.size() + 8);
    sim3_flat(Sji, &meas[meas.size() - 8]);
  };
  auto uncorrected = [&](const kfptr& pKF) -> g2o::Sim3 {                  // Sjw of a neighbour: NonCorrectedSim3 first (loop closure only)
    KeyFrameAndPose::const_iterator it;
    if (NonCorrectedSim3 && (it = NonCorrectedSim3->find(pKF)) != NonCorrectedSim3->end()) return it->second;
    return S_cw.find(pKF->mUniqueId)->second;                              // only called for keyframes in the graph
  };

  // new loop connections, :1124-1155 / :1390-1421
  set<pair<long unsigned int, long unsigned int> > linked;
  for (map<kfptr, set<kfptr> >::const_iterator mit = LoopConnections.begin(); mit != LoopConnections.end(); ++mit) {
    kfptr pKF = mit->first;
    if (pKF->isBad() || !in_graph(pKF)) continue;
    const size_t id_i = pKF->mUniqueId;
    const g2o::Sim3 S_wi = S_cw.find(id_i)->second.inverse();
    for (set<kfptr>::const_iterator sit = mit->second.begin(); sit != mit->second.end(); ++sit) {
      if ((*sit)->isBad() || !in_graph(*sit)) continue;
      const size_t id_j = (*sit)->mUniqueId;
      if ((id_i != pCurKF->mUniqueId || id_j != pLoopKF->mUniqueId) && pKF->GetWeight(*sit) < min_weight) continue;
      add_edge(pKF, *sit, S_cw.find(id_j)->second * S_wi);
      linked.insert(make_pair(min(id_i, id_j), max(id_i, id_j)));
    }
  }
  // spanning tree, earlier loop edges, covisibility, :1158-1268 / :1424-1504.  An edge to a keyframe that is not a vertex (bad) is not
  // added, as g2o refuses an edge with a missing vertex.
  for (size_t i = 0; i < kfs.size(); i++) {
    kfptr pKF = kfs[i];
    if (pKF->isBad()) continue;
    const size_t id_i = pKF->mUniqueId;
    const g2o::Sim3 S_wi = uncorrected(pKF).inverse();
    kfptr parent = pKF->GetParent();
    if (parent && in_graph(parent)) add_edge(pKF, parent, uncorrected(parent) * S_wi);
    const set<kfptr> old_loops = pKF->GetLoopEdges();
    for (set<kfptr>::const_iterator sit = old_loops.begin(); sit != old_loops.end(); ++sit) {
      kfptr lk = *sit;
      if (lk->mUniqueId < id_i && in_graph(lk)) add_edge(pKF, lk, uncorrected(lk) * S_wi);
    }
    const vector<kfptr> strong = pKF->GetCovisiblesByWeight(min_weight);
    for (vector<kfptr>::const_iterator vit = strong.begin(); vit != strong.end(); ++vit) {
      kfptr nb = *vit;
      if (!nb || nb->isBad() || !in_graph(nb)) continue;
      if (nb != parent && !pKF->hasChild(nb) && !old_loops.count(nb)) {
        const size_t id_j = nb->mUniqueId;
        if (id_j < id_i) {
          if (linked.count(make_pair(min(id_i, id_j), max(id_i, id_j)))) continue;
          add_edge(pKF, nb, uncorrected(nb) * S_wi);
        }
      }
    }
  }

  // solver->setUserLambdaInit(1e-16); optimizer.initializeOptimization(); optimizer.optimize(20)
  ccm_pgo_problem p = {(int32_t)fixed.size(), (int32_t)ei.size(), sim3.data(), fixed.data(), ei.data(), ej.data(), meas.data(), bFixScale ? 1 : 0};
  ccm_pgo_options o = {};
  o.iterations = 20; o.lambda_init = 1e-16;
  std::vector<double> out(sim3.size());
  ccm_pgo_result r = {};
  r.sim3 = out.data();
  check(ccm_pgo_solve(&p, &o, &r));

  // recovery, :1280-1330 / :1517-1565: [sR t; 0 1] -> [R t/s; 0 1] per keyframe, every map point moved through its reference keyframe
  map<size_t, g2o::Sim3> S_wc_new;
  for (size_t i = 0; i < kfs.size(); i++) {
    kfptr kfi = kfs[i];
    if (kfi->isBad()) continue;
    const size_t id_i = kfi->mUniqueId;
    const double* q = &out[8 * (size_t)row_of_id[id_i]];
    g2o::Sim3 S_iw_new(Eigen::Quaterniond(q[3], q[0], q[1], q[2]), Eigen::Vector3d(q[4], q[5], q[6]), q[7]);
    S_wc_new[id_i] = S_iw_new.inverse();
    Eigen::Matrix3d Rm = S_iw_new.rotation().toRotationMatrix();
    Eigen::Vector3d tv = S_iw_new.translation();
    double s = S_iw_new.scale();
    tv *= (1. / s);
    kfi->SetPose(Converter::toCvSE3(Rm, tv), true);
  }
  // every x_new first, then one device call for the normals, then the write-back in the same order as before
  vector<size_t> moved;
  vector<Eigen::Matrix<double, 3, 1> > x_news;
  NormalBatch nb;
  for (size_t i = 0; i < mps.size(); i++) {
    mpptr mp = mps[i];
    if (mp->isBad()) continue;
    size_t id_ref;
    const bool tagged = NonCorrectedSim3 ? mp->mCorrectedByKF_LC == pCurKF->mId : mp->mCorrectedByKF_MM == pCurKF->mId;
    if (tagged) id_ref = NonCorrectedSim3 ? mp->mCorrectedReference_LC : mp->mCorrectedReference_MM;
    else id_ref = mp->GetReferenceKeyFrame()->mUniqueId;
    if (!S_cw.count(id_ref)) continue;                           // reference keyframe not in the graph
    Eigen::Matrix<double, 3, 1> x_old = Converter::toVector3d(mp->GetWorldPos());
    Eigen::Matrix<double, 3, 1> x_new = S_wc_new.find(id_ref)->second.map(S_cw.find(id_ref)->second.map(x_old));
    moved.push_back(i); x_news.push_back(x_new);
    const double x[3] = {x_new[0], x_new[1], x_new[2]};
    nb.add(mp, x);                                               // Converter::toCvMat(x_new): each component rounded to float
  }
  ParkedNormalsGuard parked_normals;
  nb.prepare();
  for (size_t j = 0; j < moved.size(); j++) {
    mpptr mp = mps[moved[j]];
    mp->SetWorldPos(Converter::toCvMat(x_news[j]), true);
    mp->UpdateNormalAndDepth();
  }
}

}  // namespace

void Optimizer::OptimizeEssentialGraphLoopClosure(mapptr pMap, kfptr pLoopKF, kfptr pCurKF, const KeyFrameAndPose& NonCorrectedSim3,
                                                  const KeyFrameAndPose& CorrectedSim3, const map<kfptr, set<kfptr> >& LoopConnections,
                                                  const bool& bFixScale) {
  optimize_essential_graph(pMap, pLoopKF, pCurKF, &NonCorrectedSim3, &CorrectedSim3, LoopConnections, bFixScale);
}

void Optimizer::OptimizeEssentialGraphMapFusion(mapptr pMap, kfptr pLoopKF, kfptr pCurKF, const map<kfptr, set<kfptr> >& LoopConnections,
                                                const bool& bFixScale) {
  optimize_essential_graph(pMap, pLoopKF, pCurKF, nullptr, nullptr, LoopConnections, bFixScale);
}

// ---- PoseOptimizationClient (S/Optimizer.cpp:215-347) ---------------------------------------------------------------------
int Optimizer::PoseOptimizationClient(Frame& Frame) {
  std::vector<float> Xw, uv, w;
  std::vector<size_t> index;                                   // vnIndexEdgeMono
  {
    unique_lock<mutex> lock(MapPoint::mGlobalMutex);
    for (int i = 0; i < Frame.N; i++) {
      mpptr pMP = Frame.mvpMapPoints[i];
      if (!pMP) continue;
      Frame.mvbOutlier[i] = false;
      const cv::KeyPoint& kpUn = Frame.mvKeysUn[i];
      cv::Mat X = pMP->GetWorldPos();
      for (int k = 0; k < 3; k++) Xw.push_back(X.at<float>(k));
      uv.push_back(kpUn.pt.x); uv.push_back(kpUn.pt.y);
      w.push_back(Frame.mvInvLevelSigma2[kpUn.octave]);
      index.push_back(i);
    }
  }
  const int n = (int)index.size();
  if (n < 3) return 0;
  double Tcw[7];
  ccm_pose_from_Tcw_f32(Frame.mTcw.ptr<float>(0), 1, Tcw);   // Converter::toSE3Quat(Frame.mTcw)
  ccm_pose_opt_problem prob = {n, Tcw, Xw.data(), uv.data(), w.data(), Frame.fx, Frame.fy, Frame.cx, Frame.cy};
  std::vector<uint8_t> outlier(n);
  ccm_pose_opt_result res = {};
  res.outlier = outlier.data();
  check(ccm_pose_optimize(&prob, 1, &res));                    // 4 x { setEstimate, optimize(10), classify } in one launch
  for (int e = 0; e < n; e++) Frame.mvbOutlier[index[e]] = outlier[e] != 0;
  Frame.SetPose(pose_to_cv(res.Tcw));
  return res.n_inliers;                                        // nInitialCorrespondences - nBad
}

// ---- OptimizeSim3 (S/Optimizer.cpp:861-1056) --------------------------------------------------------------------------------
int Optimizer::OptimizeSim3(kfptr pKF1, kfptr pKF2, std::vector<mpptr>& vpMatches1, g2o::Sim3& g2oS12, const float th2, bool bFixScale) {
  const cv::Mat R1w = pKF1->GetRotation(), t1w = pKF1->GetTranslation(), R2w = pKF2->GetRotation(), t2w = pKF2->GetTranslation();
  const vector<mpptr> vpMapPoints1 = pKF1->GetMapPointMatches();
  std::vector<float> P1c, P2c, uv1, uv2, w1, w2;
  std::vector<size_t> index;                                   // vnIndexEdge
  for (size_t i = 0; i < vpMatches1.size(); i++) {
    if (!vpMatches1[i]) continue;
    mpptr pMP1 = vpMapPoints1[i], pMP2 = vpMatches1[i];
    if (!pMP1 || !pMP2) continue;
    const int i2 = pMP2->GetIndexInKeyFrame(pKF2);
    if (pMP1->isBad() || pMP2->isBad() || i2 < 0) continue;    // the reference's pair filter (:917-931)
    cv::Mat X1 = R1w * pMP1->GetWorldPos() + t1w, X2 = R2w * pMP2->GetWorldPos() + t2w;   // f32, as the reference
    for (int k = 0; k < 3; k++) { P1c.push_back(X1.at<float>(k)); P2c.push_back(X2.at<float>(k)); }
    const cv::KeyPoint &kp1 = pKF1->mvKeysUn[i], &kp2 = pKF2->mvKeysUn[i2];
    uv1.push_back(kp1.pt.x); uv1.push_back(kp1.pt.y); uv2.push_back(kp2.pt.x); uv2.push_back(kp2.pt.y);
    w1.push_back(pKF1->mvInvLevelSigma2[kp1.octave]); w2.push_back(pKF2->mvInvLevelSigma2[kp2.octave]);
    index.push_back(i);
  }
  const Eigen::Quaterniond q = g2oS12.rotation();
  const Eigen::Vector3d t = g2oS12.translation();
  double S12[8] = {q.x(), q.y(), q.z(), q.w(), t[0], t[1], t[2], g2oS12.scale()};
  ccm_sim3_opt_problem prob = {};
  prob.n = (int32_t)index.size(); prob.S12 = S12;
  prob.P1c = P1c.data(); prob.P2c = P2c.data(); prob.uv1 = uv1.data(); prob.uv2 = uv2.data();
  prob.inv_sigma2_1 = w1.data(); prob.inv_sigma2_2 = w2.data();
  const cv::Mat &K1 = pKF1->mK, &K2 = pKF2->mK;
  prob.K1[0] = K1.at<float>(0, 0); prob.K1[1] = K1.at<float>(1, 1); prob.K1[2] = K1.at<float>(0, 2); prob.K1[3] = K1.at<float>(1, 2);
  prob.K2[0] = K2.at<float>(0, 0); prob.K2[1] = K2.at<float>(1, 1); prob.K2[2] = K2.at<float>(0, 2); prob.K2[3] = K2.at<float>(1, 2);
  prob.th2 = th2; prob.fix_scale = bFixScale ? 1 : 0;
  std::vector<uint8_t> inlier(index.size() + 1);
  ccm_sim3_opt_result res = {};
  res.inlier = inlier.data();
  check(ccm_sim3_optimize(&prob, 1, &res));
  for (size_t e = 0; e < index.size(); e++)
    if (!inlier[e]) vpMatches1[index[e]] = static_cast<mpptr>(NULL);
  if (memcmp(res.S12, S12, sizeof S12) != 0)                    // untouched when < 10 pairs survive the first pass (the reference returns before writing g2oS12)
    g2oS12 = g2o::Sim3(Eigen::Quaterniond(res.S12[3], res.S12[0], res.S12[1], res.S12[2]),
                       Eigen::Vector3d(res.S12[4], res.S12[5], res.S12[6]), res.S12[7]);
  return res.n_inliers;
}

}  // namespace cslam

// Sim3Correction_shim.cpp — reference-side translation unit for the Sim3 correction pass of LoopFinder::CorrectLoop
// (cslam/src/LoopFinder.cpp:568-613) and MapMerger::MergeMaps (cslam/src/MapMerger.cpp:349-395); INTEGRATION.md §4h replaces each
// loop by one call of ccm_b200_correct_sim3.
//
//   flatten   one walk of the map: each entry's keyframe and GetMapPointMatches() in map order, each distinct point once (position,
//             isBad() or already tagged with the current mId, observers in mObservations order, mpRefKF and its scale factors as
//             shim/MapPoint_shim.cpp flattens them), each keyframe row's GetCameraCenter() and isBad() once
//   prepare   ccm_b200_prepare_connections on the entries (shim/KeyFrameConnections_shim.cpp, INTEGRATION.md §4e)
//   compute   one ccm_sim3_correction call: poses, centres, which entry moves which point, the moved positions and their normals with
//             the reference's mix of corrected and pre-loop centres; the normals are parked (ccm_b200_park_normals)
//   apply     the reference's loop, in its order, with its live checks; the values come from the call
// In this repository it is compiled against the stand-ins of oracle/ref_stub_sc and run next to a literal restatement of both loop
// bodies by tests/test_shim_sim3_correction.py.
#include <cslam/KeyFrame.h>
#include <cslam/MapPoint.h>
#include <cslam/estd.h>

#include <atomic>
#include <iostream>
#include <unordered_map>
#include <vector>

#include "KeyFrameConnections_shim.h"
#include "MapPoint_shim.h"
#include "Sim3Correction_shim.h"
#include "ccm_b200.h"

namespace cslam {

namespace {

typedef boost::shared_ptr<KeyFrame> kfptr;
typedef boost::shared_ptr<MapPoint> mpptr;
typedef std::pair<size_t, size_t> idpair_t;

void check(int rc, const char* fn) {
  if (rc != CCM_OK) { std::cerr << "libccm_b200: " << fn << ": " << ccm_last_error() << std::endl; throw estd::infrastructure_ex(); }
}

void sim3_flat(const g2o::Sim3& S, double* out) {
  out[0] = S.rotation().x(); out[1] = S.rotation().y(); out[2] = S.rotation().z(); out[3] = S.rotation().w();
  for (int i = 0; i < 3; i++) out[4 + i] = S.translation()[i];
  out[7] = S.scale();
}

idpair_t& tag_of(MapPoint& m, bool merge) { return merge ? m.mCorrectedByKF_MM : m.mCorrectedByKF_LC; }

// the arrays of include/ccm_b200.h's ccm_sim3_correction
struct Flat {
  std::vector<float> centre, pos, scale_ref, scale_last;
  std::vector<uint8_t> kf_bad, skip;
  std::vector<int32_t> entry_kf, slot_mp, obs, ref;
  std::vector<double> siw_new, siw_old;
  std::vector<int64_t> slot_ptr{0}, obs_ptr{0};
  std::vector<kfptr> kfs;
  std::vector<mpptr> mps;
  std::unordered_map<const KeyFrame*, int32_t> kf_row;
  std::unordered_map<const MapPoint*, int32_t> mp_row;

  int32_t add_kf(const kfptr& pKF) {
    std::unordered_map<const KeyFrame*, int32_t>::const_iterator it = kf_row.find(pKF.get());
    if (it != kf_row.end()) return it->second;
    const int32_t r = (int32_t)kfs.size();
    kf_row[pKF.get()] = r;
    kfs.push_back(pKF);
    return r;
  }
  int32_t add_mp(const mpptr& pMP) {
    std::unordered_map<const MapPoint*, int32_t>::const_iterator it = mp_row.find(pMP.get());
    if (it != mp_row.end()) return it->second;
    const int32_t r = (int32_t)mps.size();
    mp_row[pMP.get()] = r;
    mps.push_back(pMP);
    return r;
  }
};

std::atomic<unsigned long long> g_calls(0), g_moved(0), g_fallbacks(0);

// a point the flattened state did not predict: the reference's own arithmetic through the host entry point, one point, no observers
void correct_on_host(const double* siw_new, const double* siw_old, const cv::Mat& P3Dw, float out[3]) {
  const float centre[3] = {0.f, 0.f, 0.f}, X[3] = {P3Dw.at<float>(0), P3Dw.at<float>(1), P3Dw.at<float>(2)}, one = 1.f;
  const uint8_t bad = 0, skip = 0;
  const int32_t kf = 0, slot = 0, no_ref = -1;
  const int64_t slot_ptr[2] = {0, 1}, obs_ptr[2] = {0, 0};
  float Tcw[16], Ow[3], normal[3], dmax, dmin;
  int32_t entry;
  uint8_t status;
  check(ccm_sim3_correction_host(1, centre, &bad, 1, &kf, siw_new, siw_old, slot_ptr, &slot, 1, X, &skip, obs_ptr, nullptr, &no_ref, &one,
                                 &one, Tcw, Ow, &entry, out, normal, &dmax, &dmin, &status),
        "ccm_sim3_correction_host");
}

}  // namespace

void ccm_b200_sim3_correction_stats(unsigned long long* calls, unsigned long long* moved, unsigned long long* fallbacks) {
  if (calls) *calls = g_calls.load();
  if (moved) *moved = g_moved.load();
  if (fallbacks) *fallbacks = g_fallbacks.load();
}

void ccm_b200_correct_sim3(const Sim3CorrectionMap& corrected, const Sim3CorrectionMap& noncorrected, kfptr pCurKF, bool merge,
                           std::set<idpair_t>* changed) {
  g_calls++;
  const idpair_t mId = pCurKF->mId;
  const size_t uid = pCurKF->mUniqueId;
  // flatten
  Flat f;
  std::vector<kfptr> entries;
  for (Sim3CorrectionMap::const_iterator mit = corrected.begin(); mit != corrected.end(); ++mit) {
    const kfptr pKFi = mit->first;
    entries.push_back(pKFi);
    f.entry_kf.push_back(f.add_kf(pKFi));
    double s[8];
    sim3_flat(mit->second, s);
    f.siw_new.insert(f.siw_new.end(), s, s + 8);
    Sim3CorrectionMap::const_iterator nit = noncorrected.find(pKFi);
    sim3_flat(nit == noncorrected.end() ? g2o::Sim3() : nit->second, s);       // NonCorrectedSim3[pKFi]: operator[] inserts the identity
    f.siw_old.insert(f.siw_old.end(), s, s + 8);
    const std::vector<mpptr> vpMPsi = pKFi->GetMapPointMatches();
    for (size_t i = 0; i < vpMPsi.size(); i++) f.slot_mp.push_back(vpMPsi[i] ? f.add_mp(vpMPsi[i]) : -1);
    f.slot_ptr.push_back((int64_t)f.slot_mp.size());
  }
  for (size_t i = 0; i < f.mps.size(); i++) {
    MapPoint& m = *f.mps[i];
    const cv::Mat X = m.GetWorldPos();
    for (int j = 0; j < 3; j++) f.pos.push_back(X.at<float>(j));
    f.skip.push_back(m.isBad() || tag_of(m, merge) == mId ? 1 : 0);
    const std::map<kfptr, size_t> observations = m.GetObservations();
    const kfptr pRefKF = m.GetReferenceKeyFrame();
    if (observations.empty() || !pRefKF) {                                       // UpdateNormalAndDepth returns before writing
      f.obs_ptr.push_back((int64_t)f.obs.size());
      f.ref.push_back(-1); f.scale_ref.push_back(1.f); f.scale_last.push_back(1.f);
      continue;
    }
    for (std::map<kfptr, size_t>::const_iterator it = observations.begin(); it != observations.end(); ++it) f.obs.push_back(f.add_kf(it->first));
    f.obs_ptr.push_back((int64_t)f.obs.size());
    f.ref.push_back(f.add_kf(pRefKF));
    std::map<kfptr, size_t>::const_iterator r = observations.find(pRefKF);
    const size_t idx = r == observations.end() ? 0 : r->second;                 // observations[pRefKF] inserts 0 (MapPoint.cpp:813)
    f.scale_ref.push_back(pRefKF->mvScaleFactors[pRefKF->mvKeysUn[idx].octave]);
    f.scale_last.push_back(pRefKF->mvScaleFactors[pRefKF->mnScaleLevels - 1]);
  }
  for (size_t k = 0; k < f.kfs.size(); k++) {
    const cv::Mat O = f.kfs[k]->GetCameraCenter();
    for (int j = 0; j < 3; j++) f.centre.push_back(O.at<float>(j));
    f.kf_bad.push_back(f.kfs[k]->isBad() ? 1 : 0);
  }
  ParkedConnectionsGuard connections_guard;
  ccm_b200_prepare_connections(entries);
  // compute
  const int32_t E = (int32_t)entries.size(), P = (int32_t)f.mps.size();
  std::vector<float> Tcw((size_t)E * 16), Ow((size_t)E * 3), pos((size_t)P * 3), normal((size_t)P * 3), dmax(P), dmin(P);
  std::vector<int32_t> mp_entry(P);
  std::vector<uint8_t> status(P);
  if (E) {
    check(ccm_sim3_correction((int32_t)f.kfs.size(), f.centre.data(), f.kf_bad.data(), E, f.entry_kf.data(), f.siw_new.data(), f.siw_old.data(),
                              f.slot_ptr.data(), f.slot_mp.data(), P, f.pos.data(), f.skip.data(), f.obs_ptr.data(), f.obs.data(), f.ref.data(),
                              f.scale_ref.data(), f.scale_last.data(), Tcw.data(), Ow.data(), mp_entry.data(), pos.data(), normal.data(),
                              dmax.data(), dmin.data(), status.data()),
          "ccm_sim3_correction");
  }
  ParkedNormalsGuard normals_guard;
  ccm_b200_park_normals(f.mps, pos.data(), normal.data(), dmax.data(), dmin.data(), status.data());
  // apply, in the reference's order
  for (int32_t e = 0; e < E; e++) {
    const kfptr pKFi = entries[e];
    const std::vector<mpptr> vpMPsi = pKFi->GetMapPointMatches();
    for (size_t iMP = 0, endMPi = vpMPsi.size(); iMP < endMPi; iMP++) {
      const mpptr pMPi = vpMPsi[iMP];
      if (!pMPi) continue;
      if (pMPi->isBad()) continue;
      idpair_t& tag = tag_of(*pMPi, merge);
      if (tag == mId) continue;
      std::unordered_map<const MapPoint*, int32_t>::const_iterator row = f.mp_row.find(pMPi.get());
      cv::Mat cvCorrectedP3Dw(3, 1, CV_32F);
      if (row != f.mp_row.end() && mp_entry[row->second] == e) {
        for (int j = 0; j < 3; j++) cvCorrectedP3Dw.at<float>(j) = pos[3 * (size_t)row->second + j];
        g_moved++;
      } else {                                                                   // the flattened state did not predict this point
        float X[3];
        correct_on_host(&f.siw_new[8 * (size_t)e], &f.siw_old[8 * (size_t)e], pMPi->GetWorldPos(), X);
        for (int j = 0; j < 3; j++) cvCorrectedP3Dw.at<float>(j) = X[j];
        g_fallbacks++;
      }
      pMPi->SetWorldPos(cvCorrectedP3Dw, true);
      tag = mId;
      (merge ? pMPi->mCorrectedReference_MM : pMPi->mCorrectedReference_LC) = uid;
      pMPi->UpdateNormalAndDepth();
    }
    cv::Mat correctedTiw(4, 4, CV_32F);
    for (int j = 0; j < 16; j++) correctedTiw.at<float>(j / 4, j % 4) = Tcw[16 * (size_t)e + j];
    pKFi->SetPose(correctedTiw, true);
    if (!merge) changed->insert(pKFi->mId);
    pKFi->UpdateConnections();
    if (merge) pKFi->mCorrected_MM = mId;
  }
}

}  // namespace cslam

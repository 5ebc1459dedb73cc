// ref_sim3_correction_wrap.cpp — TEST INFRASTRUCTURE: stand-in KeyFrame / MapPoint scenes (oracle/ref_stub_sc) built from the flat
// arrays of synth.make_sim3_correction, a real KeyFrameAndPose of real shared_ptr keyframes, and two ways to run the correction:
//   sc_literal   the loop bodies of LoopFinder::CorrectLoop (cslam/src/LoopFinder.cpp:568-613) and MapMerger::MergeMaps
//                (cslam/src/MapMerger.cpp:349-395) restated statement by statement (_LC tags and sChangedKFs, or _MM tags and
//                mCorrected_MM), with Converter's conversions and the reference's UpdateNormalAndDepth body (MapPoint.cpp:779-823)
//                restated as in ref_normal_depth_wrap.cpp
//   sc_shim      shim/Sim3Correction_shim.cpp's ccm_b200_correct_sim3
// Keyframes live in one array in the order of their address rank, so std::less<kfptr> walks them in the scene's rank order.
// KeyFrame::UpdateConnections is a stand-in: it logs the call and counts the keyframe's weights from mvpMapPoints (the counting itself
// is shim/KeyFrameConnections_shim.cpp's, checked by tests/test_shim_covisibility.py); ccm_b200_prepare_connections only logs.
#include <cslam/KeyFrame.h>
#include <cslam/MapPoint.h>

#include <cstdint>
#include <map>
#include <set>
#include <vector>

#include "../shim/KeyFrameConnections_shim.h"
#include "../shim/MapPoint_shim.h"
#include "../shim/Sim3Correction_shim.h"
#include "ref_stub_mp/opencv_matexpr.h"

using namespace cslam;
using std::map;
typedef boost::shared_ptr<KeyFrame> kfptr;
typedef boost::shared_ptr<MapPoint> mpptr;
typedef Sim3CorrectionMap KeyFrameAndPose;

struct Scene {
  std::vector<KeyFrame> kf_store;   // in address-rank order
  std::vector<kfptr> kfs;           // by row
  std::vector<mpptr> mps;
  KeyFrameAndPose corrected, noncorrected;
  kfptr cur;
  std::vector<int32_t> connect_log;
  std::set<idpair> changed;
};

static Scene* g_scene = nullptr;   // the scene whose UpdateConnections calls are logged
static unsigned long long g_prepared = 0;

namespace cslam {
struct Sim3CorrectionProbe {
  static bool written(MapPoint& m) { return !m.mNormalVector.empty(); }
  static void read(MapPoint& m, float* pos, float* normal, float* dmax, float* dmin) {
    for (int j = 0; j < 3; j++) pos[j] = m.mWorldPos.at<float>(j);
    if (written(m)) for (int j = 0; j < 3; j++) normal[j] = m.mNormalVector.at<float>(j);
    *dmax = m.mfMaxDistance; *dmin = m.mfMinDistance;
  }
  // MapPoint::UpdateNormalAndDepth, MapPoint.cpp:779-823, restated on the stand-in
  static void update_normal_and_depth(MapPoint& self) {
    map<kfptr, size_t> observations;
    kfptr pRefKF;
    cv::Mat Pos;
    {
      std::unique_lock<std::mutex> lock1(self.mMutexFeatures);
      std::unique_lock<std::mutex> lock2(self.mMutexPos);
      if (self.mbBad) return;
      observations = self.mObservations;
      pRefKF = self.mpRefKF;
      Pos = self.mWorldPos.clone();
    }
    if (observations.empty()) return;
    cv::Mat normal = cv::Mat::zeros(3, 1, CV_32F);
    int n = 0;
    for (map<kfptr, size_t>::iterator mit = observations.begin(), mend = observations.end(); mit != mend; mit++) {
      kfptr pKF = mit->first;
      if (pKF->isBad()) continue;
      cv::Mat Owi = pKF->GetCameraCenter();
      cv::Mat normali = self.mWorldPos - Owi;
      cv::scaleAdd(normali, 1.0 / cv::norm(normali), normal, normal);   // normal = normal + normali/cv::norm(normali);
      n++;
    }
    cv::Mat PC = Pos - pRefKF->GetCameraCenter();
    const float dist = cv::norm(PC);
    const int level = pRefKF->mvKeysUn[observations[pRefKF]].octave;
    const float levelScaleFactor = pRefKF->mvScaleFactors[level];
    const int nLevels = pRefKF->mnScaleLevels;
    {
      std::unique_lock<std::mutex> lock3(self.mMutexPos);
      self.mfMaxDistance = dist * levelScaleFactor;
      self.mfMinDistance = self.mfMaxDistance / pRefKF->mvScaleFactors[nLevels - 1];
      cv::convertTo(normal, self.mNormalVector, CV_32F, 1.0 / n);        // mNormalVector = normal/n;
    }
  }
};

void KeyFrame::UpdateConnections(bool bIgnoreMutex) {
  (void)bIgnoreMutex;
  if (g_scene) g_scene->connect_log.push_back(mnRowForTest);
  std::map<kfptr, int> KFcounter;
  for (size_t i = 0; i < mvpMapPoints.size(); i++) {
    const mpptr& pMP = mvpMapPoints[i];
    if (!pMP || pMP->isBad()) continue;
    const std::map<kfptr, size_t> obs = pMP->GetObservations();
    for (std::map<kfptr, size_t>::const_iterator it = obs.begin(); it != obs.end(); ++it)
      if (it->first.get() != this) KFcounter[it->first]++;
  }
  mConnectedKeyFrameWeights = KFcounter;
}

void ccm_b200_prepare_connections(const std::vector<kfptr>& keyframes) { g_prepared += keyframes.size(); }
void ccm_b200_clear_connections() {}
}  // namespace cslam

static void noop(KeyFrame*) {}

// Converter::toVector3d / toCvMat / toCvSE3 (cslam/src/Converter.cc)
static g2o::Vector3d toVector3d(const cv::Mat& c) { return g2o::Vector3d(c.at<float>(0), c.at<float>(1), c.at<float>(2)); }
static cv::Mat toCvMat(const g2o::Vector3d& m) {
  cv::Mat cvMat(3, 1, CV_32F);
  for (int i = 0; i < 3; i++) cvMat.at<float>(i) = m(i);
  return cvMat.clone();
}
static cv::Mat toCvSE3(const double R[3][3], const g2o::Vector3d& t) {
  cv::Mat cvMat = cv::Mat::eye(4, 4, CV_32F);
  for (int i = 0; i < 3; i++) {
    for (int j = 0; j < 3; j++) cvMat.at<float>(i, j) = R[i][j];
  }
  for (int i = 0; i < 3; i++) cvMat.at<float>(i, 3) = t(i);
  return cvMat.clone();
}

extern "C" void* sc_scene_create(int32_t K, const float* Tcw, const uint8_t* kf_bad, const uint32_t* kf_rank, int32_t cur, int32_t E,
                                 const int32_t* entry_kf, const double* siw_new, const double* siw_old, const int64_t* slot_ptr,
                                 const int32_t* slot_mp, int32_t P, const float* pos, const uint8_t* mp_bad, const uint8_t* mp_tagged,
                                 const int64_t* obs_ptr, const int32_t* obs_kf, const int32_t* mp_ref) {
  Scene* s = new Scene();
  s->kf_store = std::vector<KeyFrame>(K);
  s->kfs.resize(K);
  std::vector<float> sf(8, 1.f);
  for (int l = 1; l < 8; l++) sf[l] = sf[l - 1] * 1.2f;
  for (int k = 0; k < K; k++) {
    KeyFrame& kf = s->kf_store[kf_rank[k]];
    cv::Mat T(4, 4, CV_32F);
    for (int j = 0; j < 16; j++) T.at<float>(j / 4, j % 4) = Tcw[16 * (size_t)k + j];
    kf.SetPose(T, true);
    kf.mbBad = kf_bad[k] != 0;
    kf.mId = idpair((size_t)k, 3);
    kf.mUniqueId = 1000 + (size_t)k;
    kf.mvScaleFactors = sf;
    kf.mvKeysUn.push_back(cv::KeyPoint(0.f, 0.f, 7.f, -1.f, 0.f, k % 8));
    kf.mnRowForTest = k;
    s->kfs[k] = kfptr(&kf, noop);
  }
  s->cur = s->kfs[cur];
  for (int i = 0; i < P; i++) {
    mpptr m(new MapPoint());
    cv::Mat X(3, 1, CV_32F);
    for (int j = 0; j < 3; j++) X.at<float>(j) = pos[3 * i + j];
    m->SetWorldPos(X, true);
    for (int64_t e = obs_ptr[i]; e < obs_ptr[i + 1]; e++) {
      KeyFrame& kf = *s->kfs[obs_kf[e]];
      kf.mvKeysUn.push_back(cv::KeyPoint(0.f, 0.f, 7.f, -1.f, 0.f, (int)((i + e) % 8)));
      m->AddObservationForTest(s->kfs[obs_kf[e]], kf.mvKeysUn.size() - 1);
    }
    if (mp_ref[i] >= 0) m->SetReferenceForTest(s->kfs[mp_ref[i]]);
    m->SetBadForTest(mp_bad[i] != 0);
    if (mp_tagged[i]) { m->mCorrectedByKF_LC = s->cur->mId; m->mCorrectedByKF_MM = s->cur->mId; }
    s->mps.push_back(m);
  }
  for (int e = 0; e < E; e++) {
    const kfptr& pKF = s->kfs[entry_kf[e]];
    for (int64_t j = slot_ptr[e]; j < slot_ptr[e + 1]; j++) pKF->mvpMapPoints.push_back(slot_mp[j] >= 0 ? s->mps[slot_mp[j]] : mpptr());
    const double* a = siw_new + 8 * (size_t)e;
    const double* b = siw_old + 8 * (size_t)e;
    s->corrected[pKF] = g2o::Sim3(g2o::Quaterniond(a[3], a[0], a[1], a[2]), g2o::Vector3d(a[4], a[5], a[6]), a[7]);
    s->noncorrected[pKF] = g2o::Sim3(g2o::Quaterniond(b[3], b[0], b[1], b[2]), g2o::Vector3d(b[4], b[5], b[6]), b[7]);
  }
  return s;
}

extern "C" void sc_scene_destroy(void* h) { delete static_cast<Scene*>(h); }

// the entry order std::less<kfptr> gives, as keyframe rows
extern "C" void sc_map_order(void* h, int32_t* rows) {
  Scene* s = static_cast<Scene*>(h);
  int i = 0;
  for (KeyFrameAndPose::iterator it = s->corrected.begin(); it != s->corrected.end(); ++it) rows[i++] = it->first->mnRowForTest;
}

// LoopFinder.cpp:568-613 (merge = 0) or MapMerger.cpp:349-395 (merge = 1), on the stand-ins
extern "C" void sc_literal(void* h, int merge) {
  Scene* s = static_cast<Scene*>(h);
  g_scene = s;
  KeyFrameAndPose& CorrectedSim3 = s->corrected;
  KeyFrameAndPose& NonCorrectedSim3 = s->noncorrected;
  kfptr mpCurrentKF = s->cur;
  for (KeyFrameAndPose::iterator mit = CorrectedSim3.begin(), mend = CorrectedSim3.end(); mit != mend; mit++) {
    kfptr pKFi = mit->first;
    g2o::Sim3 g2oCorrectedSiw = mit->second;
    g2o::Sim3 g2oCorrectedSwi = g2oCorrectedSiw.inverse();
    g2o::Sim3 g2oSiw = NonCorrectedSim3[pKFi];
    std::vector<mpptr> vpMPsi = pKFi->GetMapPointMatches();
    for (size_t iMP = 0, endMPi = vpMPsi.size(); iMP < endMPi; iMP++) {
      mpptr pMPi = vpMPsi[iMP];
      if (!pMPi) continue;
      if (pMPi->isBad()) continue;
      if ((merge ? pMPi->mCorrectedByKF_MM : pMPi->mCorrectedByKF_LC) == mpCurrentKF->mId) continue;
      cv::Mat P3Dw = pMPi->GetWorldPos();
      g2o::Vector3d eigP3Dw = toVector3d(P3Dw);
      g2o::Vector3d eigCorrectedP3Dw = g2oCorrectedSwi.map(g2oSiw.map(eigP3Dw));
      cv::Mat cvCorrectedP3Dw = toCvMat(eigCorrectedP3Dw);
      pMPi->SetWorldPos(cvCorrectedP3Dw, true);
      if (merge) {
        pMPi->mCorrectedByKF_MM = mpCurrentKF->mId;
        pMPi->mCorrectedReference_MM = mpCurrentKF->mUniqueId;
      } else {
        pMPi->mCorrectedByKF_LC = mpCurrentKF->mId;
        pMPi->mCorrectedReference_LC = mpCurrentKF->mUniqueId;
      }
      Sim3CorrectionProbe::update_normal_and_depth(*pMPi);
    }
    double eigR[3][3];
    g2oCorrectedSiw.rotation().toRotationMatrix(eigR);
    g2o::Vector3d eigt = g2oCorrectedSiw.translation();
    double sc = g2oCorrectedSiw.scale();
    const double inv = 1. / sc;                                          // eigt *=(1./s);
    for (int i = 0; i < 3; i++) eigt[i] *= inv;
    cv::Mat correctedTiw = toCvSE3(eigR, eigt);
    pKFi->SetPose(correctedTiw, true);
    if (merge) {
      pKFi->UpdateConnections();
      pKFi->mCorrected_MM = mpCurrentKF->mId;
    } else {
      s->changed.insert(pKFi->mId);
      pKFi->UpdateConnections();
    }
  }
  g_scene = nullptr;
}

extern "C" int sc_shim(void* h, int merge) {
  Scene* s = static_cast<Scene*>(h);
  g_scene = s;
  try {
    ccm_b200_correct_sim3(s->corrected, s->noncorrected, s->cur, merge != 0, merge ? nullptr : &s->changed);
  } catch (...) {
    g_scene = nullptr;
    return 1;
  }
  g_scene = nullptr;
  return 0;
}

// what the pass left.  Keyframes by row: Tcw [K][16], Twc [K][16], Ow [K][3], corrected_mm [K][2], conn [K][2] (number of connected
// keyframes, sum of weights), changed [K] (1: mId in sChangedKFs).  Points by row: pos, normal [P][3], max, min, written [P],
// tag_lc, tag_mm [P][2], ref_lc, ref_mm [P].  log [E]: the rows UpdateConnections ran on, in order; returns its length.
extern "C" int32_t sc_read(void* h, float* Tcw, float* Twc, float* Ow, uint64_t* corrected_mm, int32_t* conn, uint8_t* changed, float* pos,
                           float* normal, float* dmax, float* dmin, uint8_t* written, uint64_t* tag_lc, uint64_t* tag_mm, uint64_t* ref_lc,
                           uint64_t* ref_mm, int32_t* log) {
  Scene* s = static_cast<Scene*>(h);
  for (size_t k = 0; k < s->kfs.size(); k++) {
    KeyFrame& kf = *s->kfs[k];
    for (int j = 0; j < 16; j++) { Tcw[16 * k + j] = kf.Tcw.at<float>(j / 4, j % 4); Twc[16 * k + j] = kf.Twc.at<float>(j / 4, j % 4); }
    for (int j = 0; j < 3; j++) Ow[3 * k + j] = kf.Ow.at<float>(j);
    corrected_mm[2 * k] = kf.mCorrected_MM.first; corrected_mm[2 * k + 1] = kf.mCorrected_MM.second;
    int sum = 0;
    for (std::map<kfptr, int>::iterator it = kf.mConnectedKeyFrameWeights.begin(); it != kf.mConnectedKeyFrameWeights.end(); ++it) sum += it->second;
    conn[2 * k] = (int32_t)kf.mConnectedKeyFrameWeights.size(); conn[2 * k + 1] = sum;
    changed[k] = s->changed.count(kf.mId) ? 1 : 0;
  }
  for (size_t i = 0; i < s->mps.size(); i++) {
    MapPoint& m = *s->mps[i];
    normal[3 * i] = normal[3 * i + 1] = normal[3 * i + 2] = 0.f;
    Sim3CorrectionProbe::read(m, pos + 3 * i, normal + 3 * i, dmax + i, dmin + i);
    written[i] = Sim3CorrectionProbe::written(m) ? 1 : 0;
    tag_lc[2 * i] = m.mCorrectedByKF_LC.first; tag_lc[2 * i + 1] = m.mCorrectedByKF_LC.second;
    tag_mm[2 * i] = m.mCorrectedByKF_MM.first; tag_mm[2 * i + 1] = m.mCorrectedByKF_MM.second;
    ref_lc[i] = m.mCorrectedReference_LC; ref_mm[i] = m.mCorrectedReference_MM;
  }
  for (size_t e = 0; e < s->connect_log.size(); e++) log[e] = s->connect_log[e];
  return (int32_t)s->connect_log.size();
}

// outcome counters, process-wide: Sim3 shim (calls, moved, fallbacks), normals (hits, stale, host), keyframes prepared for connections
extern "C" void sc_stats(unsigned long long* c) {
  ccm_b200_sim3_correction_stats(&c[0], &c[1], &c[2]);
  ccm_b200_normals_stats(&c[3], &c[4], &c[5]);
  c[6] = g_prepared;
}

// ref_normal_depth_wrap.cpp — TEST INFRASTRUCTURE: stand-in MapPoint / KeyFrame scenes (oracle/ref_stub_mp) built from the flat arrays
// of synth.make_normal_depth, and three ways to fill their normals and depth limits:
//   nd_literal   the reference body (cslam/src/MapPoint.cpp:779-823) restated line by line on the stand-ins, each cv::Mat expression
//                evaluated the way OpenCV evaluates it (opencv_matexpr.h); results go to arrays, the objects are not touched
//   nd_shim      shim/MapPoint_shim.cpp's member UpdateNormalAndDepth() on every point, optionally after ccm_b200_prepare_normals
//   nd_shim_stale  prepare, then change the scene (observation added / pRefKF changed / position changed) before the members run
// Keyframes live in one array in row order, so every std::map<kfptr> iterates its observers in ascending row (map_order scenes).
#include <cslam/KeyFrame.h>
#include <cslam/MapPoint.h>

#include <cstdint>
#include <map>
#include <vector>

#include "../shim/MapPoint_shim.h"
#include "ref_stub_mp/opencv_matexpr.h"

using namespace cslam;
using std::map;
typedef boost::shared_ptr<KeyFrame> kfptr;
typedef boost::shared_ptr<MapPoint> mpptr;

namespace cslam {
struct NormalDepthProbe {
  static bool written(MapPoint& m) { return !m.mNormalVector.empty(); }
  static void read(MapPoint& m, float* normal, float* dmax, float* dmin) {
    for (int j = 0; j < 3; j++) normal[j] = m.mNormalVector.at<float>(j);
    *dmax = m.mfMaxDistance; *dmin = m.mfMinDistance;
  }
};
}  // namespace cslam

struct Scene {
  std::vector<KeyFrame> kf_store;
  std::vector<kfptr> kfs;
  std::vector<mpptr> mps;
};

static void noop(KeyFrame*) {}

extern "C" void* nd_scene_create(int32_t K, const float* centre, const uint8_t* kf_bad, const int32_t* kf_oct0, int32_t P, const float* pos,
                                 const uint8_t* mp_bad, const int64_t* obs_ptr, const int32_t* obs_kf, const int32_t* obs_octave,
                                 const int32_t* mp_ref) {
  Scene* s = new Scene();
  s->kf_store = std::vector<KeyFrame>(K);
  std::vector<float> sf(8, 1.f);
  for (int l = 1; l < 8; l++) sf[l] = sf[l - 1] * 1.2f;
  for (int k = 0; k < K; k++) {
    KeyFrame& kf = s->kf_store[k];
    kf.Ow = cv::Mat(3, 1, CV_32F);
    for (int j = 0; j < 3; j++) kf.Ow.at<float>(j) = centre[3 * k + j];
    kf.mbBad = kf_bad[k] != 0;
    kf.mvScaleFactors = sf;
    kf.mvKeysUn.push_back(cv::KeyPoint(0.f, 0.f, 7.f, -1.f, 0.f, kf_oct0[k]));
    s->kfs.push_back(kfptr(&kf, noop));
  }
  for (int i = 0; i < P; i++) {
    mpptr m(new MapPoint());
    cv::Mat X(3, 1, CV_32F);
    for (int j = 0; j < 3; j++) X.at<float>(j) = pos[3 * i + j];
    m->SetWorldPos(X, true);
    for (int64_t e = obs_ptr[i]; e < obs_ptr[i + 1]; e++) {
      KeyFrame& kf = s->kf_store[obs_kf[e]];
      kf.mvKeysUn.push_back(cv::KeyPoint(0.f, 0.f, 7.f, -1.f, 0.f, obs_octave[e]));
      m->AddObservationForTest(s->kfs[obs_kf[e]], kf.mvKeysUn.size() - 1);
    }
    if (mp_ref[i] >= 0) m->SetReferenceForTest(s->kfs[mp_ref[i]]);
    m->SetBadForTest(mp_bad[i] != 0);
    s->mps.push_back(m);
  }
  return s;
}

extern "C" void nd_scene_destroy(void* h) { delete static_cast<Scene*>(h); }

// the member's outcome counters (hits, stale, host), process-wide
extern "C" void nd_stats(unsigned long long* counts) { ccm_b200_normals_stats(&counts[0], &counts[1], &counts[2]); }

// MapPoint.cpp:779-823, on the stand-ins; status 0 where the body returns before writing
extern "C" void nd_literal(void* h, float* out_normal, float* out_max, float* out_min, uint8_t* status) {
  Scene* s = static_cast<Scene*>(h);
  for (size_t i = 0; i < s->mps.size(); i++) {
    MapPoint* self = s->mps[i].get();
    status[i] = 0;
    out_normal[3 * i] = out_normal[3 * i + 1] = out_normal[3 * i + 2] = 0.f; out_max[i] = out_min[i] = 0.f;
    map<kfptr, size_t> observations;
    kfptr pRefKF;
    cv::Mat Pos;
    {
      if (self->isBad()) continue;
      observations = self->GetObservations();
      pRefKF = self->GetReferenceKeyFrame();
      Pos = self->GetWorldPos();
    }
    if (observations.empty()) continue;
    cv::Mat mWorldPos = Pos;
    cv::Mat normal = cv::Mat::zeros(3, 1, CV_32F);
    int n = 0;
    for (map<kfptr, size_t>::iterator mit = observations.begin(), mend = observations.end(); mit != mend; mit++) {
      kfptr pKF = mit->first;
      if (pKF->isBad()) continue;
      cv::Mat Owi = pKF->GetCameraCenter();
      cv::Mat normali = mWorldPos - Owi;
      cv::scaleAdd(normali, 1.0 / cv::norm(normali), normal, normal);   // normal = normal + normali/cv::norm(normali);
      n++;
    }
    cv::Mat PC = Pos - pRefKF->GetCameraCenter();
    const float dist = cv::norm(PC);
    const int level = pRefKF->mvKeysUn[observations[pRefKF]].octave;
    const float levelScaleFactor = pRefKF->mvScaleFactors[level];
    const int nLevels = pRefKF->mnScaleLevels;
    const float mfMaxDistance = dist * levelScaleFactor;
    const float mfMinDistance = mfMaxDistance / pRefKF->mvScaleFactors[nLevels - 1];
    cv::Mat mNormalVector;
    cv::convertTo(normal, mNormalVector, CV_32F, 1.0 / n);           // mNormalVector = normal/n;
    for (int j = 0; j < 3; j++) out_normal[3 * i + j] = mNormalVector.at<float>(j);
    out_max[i] = mfMaxDistance; out_min[i] = mfMinDistance; status[i] = 1;
  }
}

static void run_members(Scene* s, float* out_normal, float* out_max, float* out_min, uint8_t* status) {
  for (size_t i = 0; i < s->mps.size(); i++) {
    MapPoint& m = *s->mps[i];
    m.UpdateNormalAndDepth();
    status[i] = NormalDepthProbe::written(m) ? 1 : 0;
    out_normal[3 * i] = out_normal[3 * i + 1] = out_normal[3 * i + 2] = 0.f; out_max[i] = out_min[i] = 0.f;
    if (status[i]) NormalDepthProbe::read(m, out_normal + 3 * i, out_max + i, out_min + i);
  }
}

// prepare: 0 member only (host path), 1 ccm_b200_prepare_normals first (parked path); returns 0 or -1 on an exception
extern "C" int nd_shim(void* h, int prepare, float* out_normal, float* out_max, float* out_min, uint8_t* status) {
  Scene* s = static_cast<Scene*>(h);
  try {
    ParkedNormalsGuard guard;
    if (prepare) ccm_b200_prepare_normals(s->mps, nullptr);
    run_members(s, out_normal, out_max, out_min, status);
  } catch (...) {
    return -1;
  }
  return 0;
}

// prepare, then on every other point: kind 1 add an observation from keyframe `kf`, kind 2 make `kf` the reference keyframe, kind 3
// move the point by `shift` along x.  Then the members, as nd_shim.
extern "C" int nd_shim_stale(void* h, int kind, int32_t kf, float shift, float* out_normal, float* out_max, float* out_min, uint8_t* status) {
  Scene* s = static_cast<Scene*>(h);
  try {
    ParkedNormalsGuard guard;
    ccm_b200_prepare_normals(s->mps, nullptr);
    for (size_t i = 0; i < s->mps.size(); i += 2) {
      MapPoint& m = *s->mps[i];
      if (kind == 1) {
        KeyFrame& k = s->kf_store[kf];
        k.mvKeysUn.push_back(cv::KeyPoint(0.f, 0.f, 7.f, -1.f, 0.f, 3));
        m.AddObservationForTest(s->kfs[kf], k.mvKeysUn.size() - 1);
      } else if (kind == 2) {
        m.SetReferenceForTest(s->kfs[kf]);
      } else {
        cv::Mat X = m.GetWorldPos();
        X.at<float>(0) += shift;
        m.SetWorldPos(X, true);
      }
    }
    run_members(s, out_normal, out_max, out_min, status);
  } catch (...) {
    return -1;
  }
  return 0;
}

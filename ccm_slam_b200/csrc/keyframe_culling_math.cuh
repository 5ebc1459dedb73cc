// keyframe_culling_math.cuh — the redundancy test of LocalMapping::KeyFrameCullingV3 (cslam/src/Mapping.cpp:771-863) and the effects
// of a cull on the map points it reaches, shared by the kernel (keyframe_culling.cu), the host entry point ccm_keyframe_culling_host
// and the host settle that both entry points end with.
//
//   slot_redundant   one slot of candidate `kf` at octave `level`: the point's nObs > th and at least th of its observers are not the
//                    candidate, not bad and at octave <= level + 1 (Mapping.cpp:812-838; the walk stops at th as the reference's break)
//   culled           nRedundant > mfRedundancyThres * nMPs with fptype = double (config.h:37, :234): the product and the comparison f64
//   erase_observation  MapPoint::EraseObservation(pKF, false, true) (MapPoint.cpp:442-509) on the server, for the culled row `kf`, which
//                    the caller has already marked bad: that stands for its erased entry in mObservations, since every keyframe this
//                    member erases from a point is bad from then on.  A point turned bad stays counted nowhere, which is also what
//                    MapPoint::SetBadFlag's nulling of its observers' slots amounts to.
#pragma once
#include <stdint.h>

#if defined(__CUDACC__)
#define CCM_KC_HD __host__ __device__ __forceinline__
#else
#define CCM_KC_HD inline
#endif

namespace ccm {
namespace kc {

CCM_KC_HD bool slot_redundant(int32_t kf, int32_t level, int32_t nobs, const int32_t* obs_kf, const int32_t* obs_octave, int64_t b, int64_t e,
                              const uint8_t* kf_bad, int32_t th) {
  if (nobs <= th) return false;
  const int64_t top = (int64_t)level + 1;   // the reference's int sum; octaves are small, the widening only avoids overflow
  int32_t n = 0;
  for (int64_t j = b; j < e && n < th; j++) {
    const int32_t k = obs_kf[j];
    if (kf_bad[k] || k == kf) continue;
    if ((int64_t)obs_octave[j] <= top) n++;
  }
  return n >= th;
}

CCM_KC_HD bool culled(int32_t n_red, int32_t n_mps, double red_thres) { return (double)n_red > red_thres * (double)n_mps; }

// Effects of erasing the observation of the culled row kf (already marked bad in kf_bad) from point p, once per distinct point of its
// slots (a second slot of the same point changes nothing: the first left it bad or with a reference keyframe).
CCM_KC_HD void erase_observation(int32_t kf, int32_t p, const int64_t* obs_ptr, const int32_t* obs_kf, const uint8_t* kf_bad, uint8_t* mp_bad,
                                 int32_t* mp_nobs, int32_t* mp_ref) {
  if (mp_bad[p]) return;                  // mObservations is empty and mbBad set: nothing changes
  bool observes = false;
  for (int64_t j = obs_ptr[p]; j < obs_ptr[p + 1]; j++)
    if (obs_kf[j] == kf) { observes = true; break; }
  bool bad = false;
  if (observes) {
    mp_nobs[p]--;
    if (mp_ref[p] == kf) {
      mp_ref[p] = -1;
      if (mp_nobs[p] > 0)
        for (int64_t j = obs_ptr[p]; j < obs_ptr[p + 1]; j++)
          if (!kf_bad[obs_kf[j]]) { mp_ref[p] = obs_kf[j]; break; }
    }
    if (mp_nobs[p] <= 2) bad = true;
  }
  if (bad || mp_ref[p] < 0) mp_bad[p] = 1;   // SetBadFlag, and the !mpRefKF check outside the count(pKF) block
}

}  // namespace kc
}  // namespace ccm

// keyframe_culling_oracle.cpp — TEST INFRASTRUCTURE: the checker's flat restatement of LocalMapping::KeyFrameCullingV3
// (cslam/src/Mapping.cpp:771-863) over the arrays of ccm_keyframe_culling (include/ccm_b200.h).  Written from the reference member, not
// from the product's keyframe_culling_math.cuh: it walks the candidates in order over live state — keyframe bad flags, each point's
// bad flag, nObs, mpRefKF and its observer list, from which EraseObservation removes entries — and runs KeyFrame::SetBadFlag
// (KeyFrame.cpp:936-990), MapPoint::EraseObservation (MapPoint.cpp:442-509) and MapPoint::SetBadFlag (which clears the observer list)
// the moment a verdict is reached.  There is no first pass and no settle: each candidate is counted once, over the state as it stands.
//
// orc_keyframe_culling takes the product's arguments (without n_settled) and `slip`, a deliberately wrong reading the tests must tell
// apart from the real one: 0 none, 1 `>=` for `>`, 2 the threshold product and comparison in f32, 3 no cull takes effect (no
// cascade), 4 the candidate's own observation counted, 5 `<` for `<=` on the octave.  Returns 0, or -1 on a row out of range.
#include <cstdint>
#include <utility>
#include <vector>

namespace {

struct Point {
  bool bad;
  int32_t nobs, ref;
  std::vector<std::pair<int32_t, int32_t> > obs;   // (keyframe row, octave) in mObservations order
};

struct Walk {
  std::vector<uint8_t> kf_bad;
  std::vector<Point> pts;

  void point_set_bad(Point& P) {   // MapPoint::SetBadFlag: mbBad, mObservations cleared (the observers' slots lose it)
    if (P.bad) return;
    P.bad = true;
    P.obs.clear();
  }

  void erase_observation(Point& P, int32_t kf) {   // MapPoint::EraseObservation(pKF, false, true), server
    bool bBad = false;
    for (size_t j = 0; j < P.obs.size(); j++) {
      if (P.obs[j].first != kf) continue;
      P.nobs--;
      P.obs.erase(P.obs.begin() + (long)j);
      if (P.ref == kf) {
        if (P.nobs > 0) {
          P.ref = -1;
          for (size_t r = 0; r < P.obs.size() && P.ref < 0; r++)
            if (!kf_bad[P.obs[r].first]) P.ref = P.obs[r].first;
        } else {
          P.ref = -1;
        }
      }
      if (P.nobs <= 2) bBad = true;
      break;
    }
    if (bBad) point_set_bad(P);
    if (P.ref < 0 && !P.bad) point_set_bad(P);
  }
};

}  // namespace

extern "C" int orc_keyframe_culling(int32_t n_kf, const uint8_t* kf_bad, int32_t n_c, const int32_t* cand_kf, const uint8_t* cand_not_erase,
                                    const int64_t* slot_ptr, const int32_t* slot_mp, const int32_t* slot_octave, int32_t n_mp,
                                    const uint8_t* mp_bad, const int32_t* mp_nobs, const int32_t* mp_ref, const int64_t* obs_ptr,
                                    const int32_t* obs_kf, const int32_t* obs_octave, int32_t th_obs, double red_thres, uint8_t* cull,
                                    int32_t* n_mps, int32_t* n_red, int slip) {
  Walk w;
  w.kf_bad.assign(kf_bad, kf_bad + n_kf);
  w.pts.resize((size_t)n_mp);
  for (int32_t i = 0; i < n_mp; i++) {
    Point& P = w.pts[i];
    P.bad = mp_bad[i] != 0; P.nobs = mp_nobs[i]; P.ref = mp_ref[i];
    if (P.ref < -1 || P.ref >= n_kf) return -1;
    for (int64_t j = obs_ptr[i]; j < obs_ptr[i + 1]; j++) {
      if (obs_kf[j] < 0 || obs_kf[j] >= n_kf) return -1;
      P.obs.emplace_back(obs_kf[j], obs_octave[j]);
    }
  }
  for (int32_t c = 0; c < n_c; c++) {
    const int32_t pKF = cand_kf[c];
    if (pKF < 0 || pKF >= n_kf) return -1;
    const int thObs = th_obs;
    int nRedundantObservations = 0;
    int nMPs = 0;
    for (int64_t i = slot_ptr[c]; i < slot_ptr[c + 1]; i++) {
      const int32_t p = slot_mp[i];
      if (p < -1 || p >= n_mp) return -1;
      if (p < 0) continue;
      Point& P = w.pts[p];
      if (P.bad) continue;
      nMPs++;
      if (P.nobs > thObs) {
        const int scaleLevel = slot_octave[i];
        int nObs = 0;
        for (size_t m = 0; m < P.obs.size(); m++) {
          const int32_t pKFi = P.obs[m].first;
          if (w.kf_bad[pKFi]) continue;
          if (pKFi == pKF && slip != 4) continue;
          const int scaleLeveli = P.obs[m].second;
          if (slip == 5 ? scaleLeveli < scaleLevel + 1 : scaleLeveli <= scaleLevel + 1) {
            nObs++;
            if (nObs >= thObs) break;
          }
        }
        if (nObs >= thObs) nRedundantObservations++;
      }
    }
    bool culled;
    if (slip == 1) culled = nRedundantObservations >= red_thres * nMPs;
    else if (slip == 2) culled = (float)nRedundantObservations > (float)red_thres * (float)nMPs;
    else culled = nRedundantObservations > red_thres * nMPs;
    cull[c] = culled;
    n_mps[c] = nMPs;
    n_red[c] = nRedundantObservations;
    if (!culled || slip == 3) continue;
    // KeyFrame::SetBadFlag: nothing when already bad or mbNotErase (mbToBeErased only); mId.first 0 never reaches here
    if (w.kf_bad[pKF] || cand_not_erase[c]) continue;
    for (int64_t i = slot_ptr[c]; i < slot_ptr[c + 1]; i++)
      if (slot_mp[i] >= 0) w.erase_observation(w.pts[slot_mp[i]], pKF);
    w.kf_bad[pKF] = 1;   // mbBad = true at the end of SetBadFlag
  }
  return 0;
}

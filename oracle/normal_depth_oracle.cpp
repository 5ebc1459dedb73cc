// normal_depth_oracle.cpp — TEST INFRASTRUCTURE: the checker's own restatement of MapPoint::UpdateNormalAndDepth
// (cslam/src/MapPoint.cpp:779-823) over the flat arrays of ccm_normal_depth (include/ccm_b200.h).  Written from the reference body and
// OpenCV's evaluation of each expression, not from the product's normal_depth_math.cuh:
//   normali = mWorldPos - Owi            f32 subtraction
//   cv::norm(normali)                    sqrt of the f64 sum, in index order, of the f64 squares of the f32 components
//   normal + normali / norm              cv::scaleAdd(normali, 1.0 / norm, normal): fmaf with the scale rounded to float
//   normal / n                           Mat::convertTo(CV_32F, 1.0 / n, 0): x * (float)(1.0 / n) + 0.f
// Compiled by oracle/normal_depth.mk with -ffp-contract=off.
#include <cmath>
#include <cstdint>

static double cv_norm3(float a, float b, float c) {
  double s = 0.0;
  const double v[3] = {(double)a, (double)b, (double)c};
  for (int i = 0; i < 3; i++) s += v[i] * v[i];
  return std::sqrt(s);
}

extern "C" int orc_normal_depth(int32_t n_kf, const float* kf_centre, const uint8_t* kf_bad, int32_t n_mp, const float* mp_pos,
                                const int64_t* obs_ptr, const int32_t* obs_kf, const int32_t* mp_ref, const float* mp_scale_ref,
                                const float* mp_scale_last, float* normal, float* max_dist, float* min_dist, uint8_t* status) {
  if (n_kf < 0 || n_mp < 0) return -1;
  for (int32_t i = 0; i < n_mp; i++) {
    float* out = normal + 3 * (size_t)i;
    out[0] = out[1] = out[2] = 0.f; max_dist[i] = min_dist[i] = 0.f; status[i] = 0;
    if (obs_ptr[i] == obs_ptr[i + 1] || mp_ref[i] < 0) continue;             // empty observations: return before writing
    const float* X = mp_pos + 3 * (size_t)i;
    float acc[3] = {0.f, 0.f, 0.f};
    int n = 0;
    for (int64_t j = obs_ptr[i]; j < obs_ptr[i + 1]; j++) {
      const int32_t k = obs_kf[j];
      if (k < 0 || k >= n_kf) return -1;
      if (kf_bad[k]) continue;                                               // if(pKF->isBad()) continue;
      const float* O = kf_centre + 3 * (size_t)k;
      const float d0 = X[0] - O[0], d1 = X[1] - O[1], d2 = X[2] - O[2];
      const float alpha = (float)(1.0 / cv_norm3(d0, d1, d2));
      acc[0] = std::fmaf(d0, alpha, acc[0]);
      acc[1] = std::fmaf(d1, alpha, acc[1]);
      acc[2] = std::fmaf(d2, alpha, acc[2]);
      n++;
    }
    const int32_t r = mp_ref[i];
    if (r >= n_kf) return -1;
    const float* O = kf_centre + 3 * (size_t)r;
    const float dist = (float)cv_norm3(X[0] - O[0], X[1] - O[1], X[2] - O[2]);
    max_dist[i] = dist * mp_scale_ref[i];
    min_dist[i] = max_dist[i] / mp_scale_last[i];
    const float a = (float)(1.0 / (double)n);
    for (int c = 0; c < 3; c++) out[c] = acc[c] * a + 0.f;
    status[i] = 1;
  }
  return 0;
}

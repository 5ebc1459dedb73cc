// Sim3Split_shim.h — Fuse(Scw)'s and SearchByProjection(Scw)'s split of a Sim3 into a camera (cslam/src/ORBmatcher.cpp:316-321,
// :1003-1008), in the reference's own cv::Mat expressions so that its float rounding is OpenCV's.  Shared by
// shim/ORBmatcher_proj_shim.cpp and shim/SearchAndFuse_shim.cpp.
#ifndef CCM_SIM3_SPLIT_SHIM_H
#define CCM_SIM3_SPLIT_SHIM_H
#include <cmath>

#include <opencv2/core/core.hpp>

namespace cslam {

struct Sim3Split { cv::Mat Rcw, tcw, Ow; };

inline Sim3Split split_sim3(const cv::Mat& Scw) {
  cv::Mat sRcw = Scw.rowRange(0, 3).colRange(0, 3);
  const float scw = sqrt(sRcw.row(0).dot(sRcw.row(0)));
  Sim3Split s;
  s.Rcw = sRcw / scw;
  s.tcw = Scw.rowRange(0, 3).col(3) / scw;
  s.Ow = -s.Rcw.t() * s.tcw;
  return s;
}

}  // namespace cslam
#endif

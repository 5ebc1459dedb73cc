// Stand-in for cslam::Converter::toCvMat(const g2o::Sim3&) (cslam/src/Converter.cc:58-64, toCvSE3 :95-112) over the g2o::Sim3 stand-in
// of oracle/ref_stub_sc (TEST INFRASTRUCTURE): the 4x4 CV_32F matrix [s*R t; 0 0 0 1], each f64 entry rounded to f32.
#ifndef CCM_REF_STUB_SF_CONVERTER_H
#define CCM_REF_STUB_SF_CONVERTER_H
#include <opencv2/core/core.hpp>

#include "thirdparty/g2o/g2o/types/sim3.h"

namespace cslam {
class Converter {
 public:
  static cv::Mat toCvMat(const g2o::Sim3& Sim3) {
    double eigR[3][3];
    Sim3.rotation().toRotationMatrix(eigR);
    const g2o::Vector3d eigt = Sim3.translation();
    const double s = Sim3.scale();
    cv::Mat cvMat = cv::Mat::eye(4, 4, CV_32F);
    for (int i = 0; i < 3; i++)
      for (int j = 0; j < 3; j++) cvMat.at<float>(i, j) = s * eigR[i][j];
    for (int i = 0; i < 3; i++) cvMat.at<float>(i, 3) = eigt(i);
    return cvMat;
  }
};
}  // namespace cslam
#endif

// Two OpenCV evaluation steps the stand-in cv::Mat (ref_stub/opencv2/core/core.hpp) does not model (TEST INFRASTRUCTURE).  Its
// operators round as plain f32 / f64 arithmetic and stay as they are; the literal restatement of MapPoint::UpdateNormalAndDepth
// (ref_normal_depth_wrap.cpp) calls these explicitly where OpenCV's MatExpr machinery would:
//   `a + b / s` with Mat a, b  ->  cv::scaleAdd(b, 1.0 / s, a, dst)   (f32: fmaf with the scale rounded to float)
//   `a / s`                    ->  a.convertTo(dst, CV_32F, 1.0 / s)  (f32: x * (float)scale + 0.f, convert_scale.simd.hpp cvt_32f)
#ifndef CCM_REF_STUB_MP_OPENCV_MATEXPR_H
#define CCM_REF_STUB_MP_OPENCV_MATEXPR_H
#include <cmath>

#include <opencv2/core/core.hpp>

namespace cv {

inline void scaleAdd(const Mat& src1, double alpha, const Mat& src2, Mat& dst) {
  Mat out(src1.rows, src1.cols, CV_32F);
  const float a = (float)alpha;
  for (int r = 0; r < src1.rows; r++)
    for (int c = 0; c < src1.cols; c++) out.at<float>(r, c) = std::fmaf(src1.at<float>(r, c), a, src2.at<float>(r, c));
  dst = out;
}

inline void convertTo(const Mat& src, Mat& dst, int type, double alpha, double beta = 0.0) {
  (void)type;
  Mat out(src.rows, src.cols, CV_32F);
  const float a = (float)alpha, b = (float)beta;
  for (int r = 0; r < src.rows; r++)
    for (int c = 0; c < src.cols; c++) out.at<float>(r, c) = src.at<float>(r, c) * a + b;
  dst = out;
}

}  // namespace cv
#endif

// ORBextractor_shim.cpp — replaces cslam/src/ORBextractor.cpp; cslam/include/cslam/ORBextractor.h stays byte-identical
// (constructor, operator(), mvImagePyramid, the six inline getters).  Compiled against the reference's own
// cslam/ORBextractor.h and run next to the reference's ORBextractor.cpp by tests/test_shim_extractor.py.
#include <cslam/ORBextractor.h>

#include <map>
#include <mutex>

#include "ccm_b200.h"

namespace cslam {

namespace {
// the header has no room for a handle member: keep one GPU handle per (extractor, image size) in a side table
std::mutex g_mu;
std::map<std::pair<const ORBextractor*, std::pair<int, int>>, ccm_orb_handle*> g_handles;
}

ORBextractor::ORBextractor(int _nfeatures, float _scaleFactor, int _nlevels, int _iniThFAST, int _minThFAST)
    : nfeatures(_nfeatures), scaleFactor(_scaleFactor), nlevels(_nlevels), iniThFAST(_iniThFAST), minThFAST(_minThFAST) {
  // scale tables exactly as the reference builds them (S/ORBextractor.cpp:584-600); the getters return these vectors
  mvScaleFactor.resize(nlevels); mvLevelSigma2.resize(nlevels);
  mvScaleFactor[0] = 1.0f; mvLevelSigma2[0] = 1.0f;
  for (int i = 1; i < nlevels; i++) { mvScaleFactor[i] = mvScaleFactor[i - 1] * scaleFactor; mvLevelSigma2[i] = mvScaleFactor[i] * mvScaleFactor[i]; }
  mvInvScaleFactor.resize(nlevels); mvInvLevelSigma2.resize(nlevels);
  for (int i = 0; i < nlevels; i++) { mvInvScaleFactor[i] = 1.0f / mvScaleFactor[i]; mvInvLevelSigma2[i] = 1.0f / mvLevelSigma2[i]; }
  mvImagePyramid.resize(nlevels);
  // per-level quotas, pattern and umax live inside the library (ccm_orb_create)
}

void ORBextractor::operator()(cv::InputArray _image, cv::InputArray /*_mask*/, std::vector<cv::KeyPoint>& _keypoints, cv::OutputArray _descriptors) {
  if (_image.empty()) return;
  cv::Mat image = _image.getMat();
  assert(image.type() == CV_8UC1);
  ccm_orb_handle* h;
  {
    std::lock_guard<std::mutex> lk(g_mu);
    auto key = std::make_pair((const ORBextractor*)this, std::make_pair(image.cols, image.rows));
    auto it = g_handles.find(key);
    if (it == g_handles.end()) {
      ccm_orb_config cfg = {nfeatures, (float)scaleFactor, nlevels, iniThFAST, minThFAST, /*blur_2413=*/CV_MAJOR_VERSION < 3};
      ccm_orb_handle* nh = nullptr;
      if (ccm_orb_create(&cfg, image.cols, image.rows, &nh) != CCM_OK) throw estd::infrastructure_ex();
      it = g_handles.insert(std::make_pair(key, nh)).first;
    }
    h = it->second;
  }
  int cap = 0;
  if (ccm_orb_max_keypoints(h, &cap) != CCM_OK) throw estd::infrastructure_ex();
  std::vector<ccm_keypoint> kps(cap);
  cv::Mat desc(cap, 32, CV_8U);
  int n = 0;
  if (ccm_orb_extract(h, image.ptr<uchar>(0), (int)image.step, kps.data(), cap, &n, desc.ptr<uchar>(0)) != CCM_OK) throw estd::infrastructure_ex();
  _keypoints.clear(); _keypoints.reserve(n);
  for (int i = 0; i < n; i++) _keypoints.push_back(cv::KeyPoint(kps[i].x, kps[i].y, kps[i].size, kps[i].angle, kps[i].response, kps[i].octave));
  if (n == 0) _descriptors.release(); else desc.rowRange(0, n).copyTo(_descriptors);
  for (int l = 0; l < nlevels; l++) {                          // mvImagePyramid is a public member read by Frame/Tracking
    int w = 0, hh = 0;
    ccm_orb_get_level(h, l, nullptr, &w, &hh);
    mvImagePyramid[l].create(hh, w, CV_8U);
    ccm_orb_get_level(h, l, mvImagePyramid[l].ptr<uchar>(0), &w, &hh);
  }
}

}  // namespace cslam

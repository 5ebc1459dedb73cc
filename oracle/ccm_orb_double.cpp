// ccm_orb_double.cpp — link-time stand-in for the device ORB extractor behind shim/ORBextractor_shim.cpp (TEST INFRASTRUCTURE, NOT PRODUCT).
// ccm_orb_create / max_keypoints / extract / get_level on top of the CPU oracle, so that the shim's own code (scale tables, handle cache, keypoint and
// descriptor marshalling, the public mvImagePyramid) can run without a GPU.  Linked only into oracle/_ref/libextractor_shim.so.
#include <algorithm>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <vector>

#include "ccm_b200.h"

extern "C" {
struct orc_orb_config { int32_t nfeatures; float scale_factor; int32_t nlevels, ini_th_fast, min_th_fast, blur_2413; };
struct orc_keypoint { float x, y, size, angle, response; int32_t octave; };
int orc_orb_extract(const uint8_t* img, int w, int h, int stride, const orc_orb_config* c, orc_keypoint* kps, int max_kp, int* n, uint8_t* desc);
void orc_orb_tables(const orc_orb_config* c, int w, int h, int* n_per_level, int* umax16, int* level_wh);
void orc_resize_linear_u8(const uint8_t* src, int sw, int sh, uint8_t* dst, int dw, int dh);
}

struct ccm_orb_handle {
  orc_orb_config cfg; int w, h;
  std::vector<std::vector<uint8_t> > level; std::vector<int> wh;
};

extern "C" {
int ccm_orb_create(const ccm_orb_config* c, int32_t width, int32_t height, ccm_orb_handle** out) {
  ccm_orb_handle* h = new ccm_orb_handle;
  h->cfg = orc_orb_config{c->nfeatures, c->scale_factor, c->nlevels, c->ini_th_fast, c->min_th_fast, c->blur_2413};
  h->w = width; h->h = height;
  *out = h;
  return CCM_OK;
}
// the device library's bound (orb.cu): per level max(4 * nIni, quota + 3), nIni = root nodes of the level's quadtree
int ccm_orb_max_keypoints(const ccm_orb_handle* h, int32_t* n) {
  const int L = h->cfg.nlevels;
  std::vector<int> npl(L), umax(16), wh(2 * L);
  orc_orb_tables(&h->cfg, h->w, h->h, npl.data(), umax.data(), wh.data());
  int cap = 0;
  for (int l = 0; l < L; l++) {
    const int border = 2 * (19 - 3);             // the quadtree spans the level less EDGE_THRESHOLD - 3 on each side
    const int nIni = (int)std::round(static_cast<float>(wh[2 * l] - border) / (wh[2 * l + 1] - border));
    cap += std::max(4 * nIni, npl[l] + 3);
  }
  *n = cap;
  return CCM_OK;
}
int ccm_orb_extract(ccm_orb_handle* h, const uint8_t* img, int32_t stride, ccm_keypoint* kps, int32_t max_kp, int32_t* n, uint8_t* desc) {
  int cap = 0;
  ccm_orb_max_keypoints(h, &cap);
  std::vector<orc_keypoint> k(cap);
  std::vector<uint8_t> d((size_t)cap * 32);
  int cnt = 0;
  orc_orb_extract(img, h->w, h->h, stride, &h->cfg, k.data(), cap, &cnt, d.data());
  *n = cnt;
  if (cnt > max_kp) return CCM_ERR_INVALID;   // as the device library: refuse, write nothing
  for (int i = 0; i < cnt; i++) kps[i] = ccm_keypoint{k[i].x, k[i].y, k[i].size, k[i].angle, k[i].response, k[i].octave};
  if (desc) std::memcpy(desc, d.data(), (size_t)cnt * 32);
  // ComputePyramid (S/ORBextractor.cpp:1280-1304): level l is level l-1 resized, INTER_LINEAR
  const int L = h->cfg.nlevels;
  std::vector<int> npl(L), umax(16);
  h->wh.assign(2 * L, 0);
  orc_orb_tables(&h->cfg, h->w, h->h, npl.data(), umax.data(), h->wh.data());
  h->level.assign(L, std::vector<uint8_t>());
  h->level[0].resize((size_t)h->w * h->h);
  for (int r = 0; r < h->h; r++) std::memcpy(&h->level[0][(size_t)r * h->w], img + (size_t)r * stride, h->w);
  for (int l = 1; l < L; l++) {
    h->level[l].resize((size_t)h->wh[2 * l] * h->wh[2 * l + 1]);
    orc_resize_linear_u8(h->level[l - 1].data(), h->wh[2 * l - 2], h->wh[2 * l - 1], h->level[l].data(), h->wh[2 * l], h->wh[2 * l + 1]);
  }
  return CCM_OK;
}
int ccm_orb_get_level(ccm_orb_handle* h, int32_t level, uint8_t* out, int32_t* w, int32_t* hgt) {
  *w = h->wh[2 * level]; *hgt = h->wh[2 * level + 1];
  if (out) std::memcpy(out, h->level[level].data(), h->level[level].size());
  return CCM_OK;
}
void ccm_orb_destroy(ccm_orb_handle* h) { delete h; }
}

// orb.cu — ORB front end behind ccm_orb_* (include/ccm_b200.h).
//
// Replaces cslam::ORBextractor::operator() (S/ORBextractor.cpp:1216-1278).  Integer-exact stages run on the GPU:
//   k_resize        ComputePyramid: chained cv::resize INTER_LINEAR u8, fixed point, coefficient tables built on the host
//                   exactly like OpenCV builds them (S/ORBextractor.cpp:1280-1304, OCV/imgproc/src/imgwarp.cpp)
//   k_fast_cells    ComputeKeyPointsOctTree's per-cell cv::FAST(20) -> cv::FAST(7) fallback with 3x3 NMS restricted to
//                   the cell (S/ORBextractor.cpp:957-997, OCV/features2d/src/fast.cpp, fast_score.cpp): one CTA per cell,
//                   ROI staged in shared memory, candidates emitted in the reference's row-major order
//   k_gather        orders the candidates (level, cell row, cell col, y, x) and computes the IC_Angle integer moments
//                   m01, m10 over the radius-15 disc (S/ORBextractor.cpp:68-95)
//   k_blur          cv::GaussianBlur 7x7 sigma 2 u8, fixed point 8.8 -> 16.16 (S/ORBextractor.cpp:1258-1259)
//   k_descriptors   computeOrbDescriptor: 256 steered brightness tests, one warp per keypoint, one byte per lane
//                   (S/ORBextractor.cpp:100-316)
// The order-dependent quadtree (DistributeOctTree, S/ORBextractor.cpp:707-931) and the three float transcendental
// evaluations per keypoint (fastAtan2, cosf, sinf) stay on the host so that they are bit-identical to a CPU build of
// the reference (SURVEY.md §7 hard parts); they touch O(10^4) items per frame.
#include <algorithm>
#include <cfloat>
#include <cmath>
#include <list>

#include "common.cuh"
#include "orb_pattern.h"

using namespace ccm;

namespace {

constexpr int kEdge = 19;       // EDGE_THRESHOLD
constexpr int kHalfPatch = 15;  // HALF_PATCH_SIZE
constexpr int kPatch = 31;

__constant__ signed char c_pattern[1024];
__constant__ int c_umax[16];

struct BlurTaps { int k[7]; };  // per handle (ccm_orb_config::blur_2413), so handles of both tap sets can coexist

struct Cell {            // one FAST cell of one pyramid level
  int level, img_off, img_w;
  int x0, y0, x1, y1;    // ROI [x0,x1) x [y0,y1) in level pixels
  int out_off;           // first slot in the per-cell candidate array
};

struct Cand {            // candidate keypoint, coordinates relative to (minBorderX, minBorderY) like the reference
  float x, y;
  int score, level, m01, m10;
};

struct KpIn {            // keypoint handed to the descriptor kernel
  int level, cx, cy;
  float a, b;            // cos / sin of the orientation, evaluated on the host
};

// ---- pyramid --------------------------------------------------------------------------------------------------
__global__ void k_resize(const uint8_t* __restrict__ src, int sw, int sh, uint8_t* __restrict__ dst, int dw, int dh,
                         const int* __restrict__ xofs, const short* __restrict__ xa, const int* __restrict__ yofs,
                         const short* __restrict__ ya) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
  if (x >= dw || y >= dh) return;
  const int x0 = xofs[x], x1 = min(x0 + 1, sw - 1);
  const int y0 = yofs[y], y1 = min(y0 + 1, sh - 1);
  const int a0 = xa[2 * x], a1 = xa[2 * x + 1], b0 = ya[2 * y], b1 = ya[2 * y + 1];
  const int r0 = src[(size_t)y0 * sw + x0] * a0 + src[(size_t)y0 * sw + x1] * a1;
  const int r1 = src[(size_t)y1 * sw + x0] * a0 + src[(size_t)y1 * sw + x1] * a1;
  dst[(size_t)y * dw + x] = (uint8_t)((((b0 * (r0 >> 4)) >> 16) + ((b1 * (r1 >> 4)) >> 16) + 2) >> 2);
}

// ---- FAST per cell -----------------------------------------------------------------------------------------------
__device__ __forceinline__ int corner_score(const uint8_t* t, int stride, int x, int y, int lo_th) {
  const int v = t[y * stride + x];
  int d[16];
  d[0] = v - t[(y + 3) * stride + x];       d[1] = v - t[(y + 3) * stride + x + 1];
  d[2] = v - t[(y + 2) * stride + x + 2];   d[3] = v - t[(y + 1) * stride + x + 3];
  d[4] = v - t[y * stride + x + 3];         d[5] = v - t[(y - 1) * stride + x + 3];
  d[6] = v - t[(y - 2) * stride + x + 2];   d[7] = v - t[(y - 3) * stride + x + 1];
  d[8] = v - t[(y - 3) * stride + x];       d[9] = v - t[(y - 3) * stride + x - 1];
  d[10] = v - t[(y - 2) * stride + x - 2];  d[11] = v - t[(y - 1) * stride + x - 3];
  d[12] = v - t[y * stride + x - 3];        d[13] = v - t[(y + 1) * stride + x - 3];
  d[14] = v - t[(y + 2) * stride + x - 2];  d[15] = v - t[(y + 3) * stride + x - 1];
  // cornerScore<16> = the largest threshold t for which 9 contiguous ring pixels are all darker than v - t or all
  // brighter than v + t.  "Is a corner at t" is monotone in t, so the score is found by bisection on t with a 16-bit
  // ring mask per polarity and a run-length test (a min/max formulation over the 16 arcs compiled to wrong VIMNMX3
  // chains with nvcc 12.9 for sm_100a, an earlier target, so the test is written with compares and bit operations only).
  auto corner_at = [&](int t) -> bool {
    unsigned dark = 0, bright = 0;
#pragma unroll
    for (int i = 0; i < 16; i++) {
      dark |= (d[i] > t ? 1u : 0u) << i;
      bright |= (d[i] < -t ? 1u : 0u) << i;
    }
    unsigned m = dark | (dark << 16);
    unsigned r = m & (m >> 1); r &= r >> 2; r &= r >> 4; r &= m >> 8;   // bit i: 9 consecutive ones starting at i
    unsigned hit = r & 0xffffu;
    m = bright | (bright << 16);
    r = m & (m >> 1); r &= r >> 2; r &= r >> 4; r &= m >> 8;
    hit |= r & 0xffffu;
    return hit != 0u;
  };
  if (!corner_at(lo_th)) return -1;  // not even a corner at the lowest threshold anyone asks for
  int lo = lo_th, hi = 255;          // corner_at(lo) holds, corner_at(hi) does not (|d| <= 255)
  while (hi - lo > 1) {
    const int mid = (lo + hi) >> 1;
    if (corner_at(mid)) lo = mid; else hi = mid;
  }
  return lo;
}

// dynamic smem: tile (u8, tw*th) | score (short, tw*th) | flag (u8, tw*th)
__global__ void __launch_bounds__(256) k_fast_cells(const uint8_t* __restrict__ pyr, const Cell* __restrict__ cells,
                                                    int ini_th, int min_th, int tile_cap, int max_per_cell,
                                                    int* __restrict__ cell_count, ushort4* __restrict__ cell_out) {
  extern __shared__ unsigned char smem[];
  const Cell c = cells[blockIdx.x];
  const int tw = c.x1 - c.x0, th = c.y1 - c.y0;
  uint8_t* tile = smem;
  short* score = reinterpret_cast<short*>(smem + ((tile_cap + 15) & ~15));
  uint8_t* flag = smem + ((tile_cap + 15) & ~15) + 2 * tile_cap;
  __shared__ int n_ini;
  if (threadIdx.x == 0) n_ini = 0;
  const int n = tw * th;
  if (tw < 7 || th < 7) {
    if (threadIdx.x == 0) cell_count[blockIdx.x] = 0;
    return;
  }
  const uint8_t* img = pyr + c.img_off;
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    const int y = i / tw, x = i - y * tw;
    tile[i] = img[(size_t)(c.y0 + y) * c.img_w + c.x0 + x];
    score[i] = 0;
    flag[i] = 0;
  }
  __syncthreads();
  const int iw = tw - 6, ih = th - 6, ni = iw * ih;
  for (int i = threadIdx.x; i < ni; i += blockDim.x) {
    const int y = 3 + i / iw, x = 3 + i % iw;
    const int s = corner_score(tile, tw, x, y, min_th);
    score[y * tw + x] = (short)(s >= min_th ? s : 0);  // the reference's score buffer: 0 for non-corners
  }
  __syncthreads();
  int my_ini = 0;
  for (int i = threadIdx.x; i < ni; i += blockDim.x) {
    const int y = 3 + i / iw, x = 3 + i % iw;
    const int s = score[y * tw + x];
    if (s < min_th) continue;
    // strict 3x3 maximum; neighbours outside the cell interior hold 0 in the reference's buffers (never computed)
    const bool mx = s > score[(y - 1) * tw + x - 1] && s > score[(y - 1) * tw + x] && s > score[(y - 1) * tw + x + 1] &&
                    s > score[y * tw + x - 1] && s > score[y * tw + x + 1] && s > score[(y + 1) * tw + x - 1] &&
                    s > score[(y + 1) * tw + x] && s > score[(y + 1) * tw + x + 1];
    if (mx) {
      flag[y * tw + x] = s >= ini_th ? 2 : 1;
      my_ini += s >= ini_th;
    }
  }
  if (my_ini) atomicAdd(&n_ini, my_ini);
  __syncthreads();
  const int need = n_ini > 0 ? 2 : 1;  // FAST(iniThFAST) found something, else the FAST(minThFAST) rerun
  // ordered compaction by warp 0: row-major over the interior, 32 pixels at a time
  if (threadIdx.x < 32) {
    int base = 0;
    for (int i0 = 0; i0 < ni; i0 += 32) {
      const int i = i0 + threadIdx.x;
      bool keep = false;
      int x = 0, y = 0;
      if (i < ni) {
        y = 3 + i / iw; x = 3 + i % iw;
        keep = flag[y * tw + x] >= need;
      }
      const unsigned m = __ballot_sync(0xffffffffu, keep);
      if (keep) {
        const int slot = base + __popc(m & ((1u << threadIdx.x) - 1u));
        if (slot < max_per_cell)
          cell_out[(size_t)c.out_off + slot] = make_ushort4((unsigned short)(c.x0 + x), (unsigned short)(c.y0 + y),
                                                            (unsigned short)score[y * tw + x], 0);
      }
      base += __popc(m);
    }
    if (threadIdx.x == 0) cell_count[blockIdx.x] = min(base, max_per_cell);
  }
}

// exclusive scan of the per-cell counts (single block) -> offsets, total in offsets[ncells]
__global__ void __launch_bounds__(1024) k_scan_cells(const int* __restrict__ cnt, int n, int* __restrict__ off) {
  __shared__ int warp_tot[32];
  __shared__ int carry;
  if (threadIdx.x == 0) carry = 0;
  __syncthreads();
  for (int base = 0; base < n; base += 1024) {
    const int i = base + threadIdx.x;
    const int v = i < n ? cnt[i] : 0;
    int s = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int t = __shfl_up_sync(0xffffffffu, s, o);
      if ((threadIdx.x & 31) >= o) s += t;
    }
    if ((threadIdx.x & 31) == 31) warp_tot[threadIdx.x >> 5] = s;
    __syncthreads();
    if (threadIdx.x < 32) {
      int w = warp_tot[threadIdx.x];
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const int t = __shfl_up_sync(0xffffffffu, w, o);
        if (threadIdx.x >= o) w += t;
      }
      warp_tot[threadIdx.x] = w;
    }
    __syncthreads();
    const int prev = (threadIdx.x >> 5) ? warp_tot[(threadIdx.x >> 5) - 1] : 0;
    if (i < n) off[i] = carry + prev + s - v;
    __syncthreads();
    if (threadIdx.x == 0) carry += warp_tot[31];
    __syncthreads();
  }
  if (threadIdx.x == 0) off[n] = carry;
}

// one CTA per cell: copy its candidates to their global position, add the IC_Angle moments
__global__ void __launch_bounds__(128) k_gather(const uint8_t* __restrict__ pyr, const Cell* __restrict__ cells,
                                                const int* __restrict__ cell_count, const int* __restrict__ cell_off,
                                                const ushort4* __restrict__ cell_out, int max_total, Cand* __restrict__ out) {
  const Cell c = cells[blockIdx.x];
  const int n = cell_count[blockIdx.x];
  const uint8_t* img = pyr + c.img_off;
  for (int k = threadIdx.x; k < n; k += blockDim.x) {
    const int dstI = cell_off[blockIdx.x] + k;
    if (dstI >= max_total) break;
    const ushort4 e = cell_out[(size_t)c.out_off + k];
    const int cx = e.x, cy = e.y;
    int m01 = 0, m10 = 0;
    const uint8_t* center = img + (size_t)cy * c.img_w + cx;
    for (int u = -kHalfPatch; u <= kHalfPatch; ++u) m10 += u * center[u];
    for (int v = 1; v <= kHalfPatch; ++v) {
      int v_sum = 0;
      const int d = c_umax[v];
      for (int u = -d; u <= d; ++u) {
        const int vp = center[u + v * c.img_w], vm = center[u - v * c.img_w];
        v_sum += (vp - vm);
        m10 += u * (vp + vm);
      }
      m01 += v * v_sum;
    }
    Cand o;
    o.x = (float)(cx - (kEdge - 3)); o.y = (float)(cy - (kEdge - 3));
    o.score = e.z; o.level = c.level; o.m01 = m01; o.m10 = m10;
    out[dstI] = o;
  }
}

// ---- Gaussian blur 7x7, sigma 2, BORDER_REFLECT_101, fixed point ----------------------------------------------------
__device__ __forceinline__ int reflect101(int p, int n) {
  if (n == 1) return 0;
  while (p < 0 || p >= n) p = p < 0 ? -p : 2 * (n - 1) - p;
  return p;
}

__global__ void __launch_bounds__(256) k_blur(const uint8_t* __restrict__ src, uint8_t* __restrict__ dst, int w, int h,
                                              const BlurTaps taps) {
  __shared__ unsigned short rowpass[(16 + 6) * 32];  // 22 rows x 32 cols of horizontal sums (8.8 fixed point)
  const int bx = blockIdx.x * 32, by = blockIdx.y * 16;
  for (int i = threadIdx.x; i < 22 * 32; i += 256) {
    const int ry = i / 32, rx = i % 32;
    const int x = bx + rx;
    const int y = reflect101(by + ry - 3, h);
    unsigned s = 0;
    if (x < w) {
#pragma unroll
      for (int k = -3; k <= 3; k++) s += (unsigned)taps.k[k + 3] * src[(size_t)y * w + reflect101(x + k, w)];
    }
    rowpass[i] = (unsigned short)s;
  }
  __syncthreads();
  for (int i = threadIdx.x; i < 16 * 32; i += 256) {
    const int ty = i / 32, tx = i % 32;
    const int x = bx + tx, y = by + ty;
    if (x >= w || y >= h) continue;
    unsigned s = 0;
#pragma unroll
    for (int k = 0; k < 7; k++) s += (unsigned)taps.k[k] * rowpass[(ty + k) * 32 + tx];
    dst[(size_t)y * w + x] = (uint8_t)min((s + 32768u) >> 16, 255u);
  }
}

// ---- steered BRIEF ------------------------------------------------------------------------------------------------
struct LevelRef { int off, w, h; };

__global__ void __launch_bounds__(128) k_descriptors(const uint8_t* __restrict__ blurred, const LevelRef* __restrict__ levels,
                                                     const KpIn* __restrict__ kps, int n, uint8_t* __restrict__ desc) {
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (warp >= n) return;
  const KpIn k = kps[warp];
  const LevelRef L = levels[k.level];
  const uint8_t* center = blurred + L.off + (size_t)k.cy * L.w + k.cx;
  int val = 0;
#pragma unroll
  for (int bit = 0; bit < 8; bit++) {
    int t[2];
#pragma unroll
    for (int q = 0; q < 2; q++) {
      const int idx = 16 * lane + 2 * bit + q;
      const float px = (float)c_pattern[2 * idx], py = (float)c_pattern[2 * idx + 1];
      // cvRound(x*b + y*a), cvRound(x*a - y*b): separate roundings, no FMA contraction
      const int iy = __float2int_rn(__fadd_rn(__fmul_rn(px, k.b), __fmul_rn(py, k.a)));
      const int ix = __float2int_rn(__fsub_rn(__fmul_rn(px, k.a), __fmul_rn(py, k.b)));
      t[q] = center[iy * L.w + ix];
    }
    val |= (t[0] < t[1]) << bit;
  }
  desc[(size_t)warp * 32 + lane] = (uint8_t)val;
}

// ---- host side ----------------------------------------------------------------------------------------------------
inline int cv_round(float v) { return (int)lrintf(v); }

float fast_atan2_host(float y, float x) {  // cv::fastAtan2 (OCV/core/src/mathfuncs.cpp:51-77); this TU is built with -ffp-contract=off
  static const float p1 = 0.9997878412794807f * (float)(180 / M_PI);
  static const float p3 = -0.3258083974640975f * (float)(180 / M_PI);
  static const float p5 = 0.1555786518463281f * (float)(180 / M_PI);
  static const float p7 = -0.04432655554792128f * (float)(180 / M_PI);
  const float ax = std::fabs(x), ay = std::fabs(y);
  float a, c, c2;
  if (ax >= ay) {
    c = ay / (ax + (float)DBL_EPSILON);
    c2 = c * c;
    a = (((p7 * c2 + p5) * c2 + p3) * c2 + p1) * c;
  } else {
    c = ax / (ay + (float)DBL_EPSILON);
    c2 = c * c;
    a = 90.f - (((p7 * c2 + p5) * c2 + p3) * c2 + p1) * c;
  }
  if (x < 0) a = 180.f - a;
  if (y < 0) a = 360.f - a;
  return a;
}

// DistributeOctTree on an index-linked node pool.  Node order in the reference's std::list is reproduced by an intrusive
// doubly linked list with push_front; ties of the (size, pointer) sort are resolved by creation order.
struct QNode {
  int ulx, uly, brx, bry;
  std::vector<int> keys;  // candidate indices
  bool no_more = false;
  int prev = -1, next = -1;
  long seq = 0;
  bool alive = true;
};

struct Quadtree {
  std::vector<QNode> pool;
  int head = -1, tail = -1, count = 0;
  long seq = 0;
  int push_front(QNode&& n) {
    n.seq = seq++;
    n.prev = -1; n.next = head;
    pool.push_back(std::move(n));
    const int id = (int)pool.size() - 1;
    if (head >= 0) pool[head].prev = id; else tail = id;
    head = id; count++;
    return id;
  }
  int push_back(QNode&& n) {
    n.seq = seq++;
    n.next = -1; n.prev = tail;
    pool.push_back(std::move(n));
    const int id = (int)pool.size() - 1;
    if (tail >= 0) pool[tail].next = id; else head = id;
    tail = id; count++;
    return id;
  }
  int erase(int id) {  // returns the next node
    QNode& n = pool[id];
    const int nx = n.next;
    if (n.prev >= 0) pool[n.prev].next = n.next; else head = n.next;
    if (n.next >= 0) pool[n.next].prev = n.prev; else tail = n.prev;
    n.alive = false; n.keys.clear(); n.keys.shrink_to_fit();
    count--;
    return nx;
  }
};

void divide_node(const QNode& n, const Cand* cand, QNode out[4]) {
  const int halfX = (int)std::ceil(static_cast<float>(n.brx - n.ulx) / 2);
  const int halfY = (int)std::ceil(static_cast<float>(n.bry - n.uly) / 2);
  const int mx = n.ulx + halfX, my = n.uly + halfY;
  out[0].ulx = n.ulx; out[0].uly = n.uly; out[0].brx = mx;    out[0].bry = my;
  out[1].ulx = mx;    out[1].uly = n.uly; out[1].brx = n.brx; out[1].bry = my;
  out[2].ulx = n.ulx; out[2].uly = my;    out[2].brx = mx;    out[2].bry = n.bry;
  out[3].ulx = mx;    out[3].uly = my;    out[3].brx = n.brx; out[3].bry = n.bry;
  for (int k : n.keys) {
    const Cand& kp = cand[k];
    const int q = (kp.x < mx ? 0 : 1) + (kp.y < my ? 0 : 2);
    out[q].keys.push_back(k);
  }
  for (int q = 0; q < 4; q++) out[q].no_more = out[q].keys.size() == 1;
}

// number of root nodes of DistributeOctTree on a level whose bordered area is [minX, maxX) x [minY, maxY)
int quadtree_roots(int minX, int maxX, int minY, int maxY) {
  return (int)std::round(static_cast<float>(maxX - minX) / (maxY - minY));
}

std::vector<int> distribute(const Cand* cand, int n, int minX, int maxX, int minY, int maxY, int N) {
  std::vector<int> result;
  if (n == 0) return result;
  const int nIni = quadtree_roots(minX, maxX, minY, maxY);
  CCM_REQUIRE(nIni >= 1, "ccm_orb_extract: image too tall for the reference's quadtree (nIni == 0)");
  const float hX = static_cast<float>(maxX - minX) / nIni;
  Quadtree t;
  t.pool.reserve(4 * (size_t)N + 64);
  std::vector<int> ini(nIni);
  for (int i = 0; i < nIni; i++) {
    QNode q;
    q.ulx = (int)(hX * static_cast<float>(i)); q.uly = 0;
    q.brx = (int)(hX * static_cast<float>(i + 1)); q.bry = maxY - minY;
    ini[i] = t.push_back(std::move(q));
  }
  for (int k = 0; k < n; k++) t.pool[ini[(int)(cand[k].x / hX)]].keys.push_back(k);
  for (int id = t.head; id >= 0;) {
    QNode& q = t.pool[id];
    if (q.keys.size() == 1) { q.no_more = true; id = q.next; }
    else if (q.keys.empty()) id = t.erase(id);
    else id = q.next;
  }
  typedef std::pair<int, int> SP;  // (size, node id)
  std::vector<SP> expand;
  auto add_children = [&](QNode kids[4], int& nToExpand) {
    for (int c = 0; c < 4; c++)
      if (!kids[c].keys.empty()) {
        const int sz = (int)kids[c].keys.size();
        const int id = t.push_front(std::move(kids[c]));
        if (sz > 1) { nToExpand++; expand.push_back(SP(sz, id)); }
      }
  };
  bool finish = false;
  while (!finish) {
    const int prevSize = t.count;
    int nToExpand = 0;
    expand.clear();
    for (int id = t.head; id >= 0;) {
      if (t.pool[id].no_more) { id = t.pool[id].next; continue; }
      QNode kids[4];
      divide_node(t.pool[id], cand, kids);
      const int nx = t.pool[id].next;  // children go to the front, the walk continues towards the tail
      add_children(kids, nToExpand);
      t.erase(id);
      id = nx;
    }
    if (t.count >= N || t.count == prevSize) {
      finish = true;
    } else if (t.count + nToExpand * 3 > N) {
      while (!finish) {
        const int prev2 = t.count;
        std::vector<SP> prevList = expand;
        expand.clear();
        std::sort(prevList.begin(), prevList.end(), [&](const SP& a, const SP& b) {
          return a.first != b.first ? a.first < b.first : t.pool[a.second].seq < t.pool[b.second].seq;
        });
        for (int j = (int)prevList.size() - 1; j >= 0; j--) {
          QNode kids[4];
          divide_node(t.pool[prevList[j].second], cand, kids);
          int dummy = 0;
          add_children(kids, dummy);
          t.erase(prevList[j].second);
          if (t.count >= N) break;
        }
        if (t.count >= N || t.count == prev2) finish = true;
      }
    }
  }
  for (int id = t.head; id >= 0; id = t.pool[id].next) {
    const QNode& q = t.pool[id];
    int best = q.keys[0];
    float maxResp = (float)cand[best].score;
    for (size_t k = 1; k < q.keys.size(); k++)
      if ((float)cand[q.keys[k]].score > maxResp) { best = q.keys[k]; maxResp = (float)cand[best].score; }
    result.push_back(best);
  }
  return result;
}

}  // namespace

struct ccm_orb_handle {
  ccm_orb_config cfg;
  int width = 0, height = 0, device = 0;
  cudaStream_t stream = nullptr;
  std::vector<float> scale, inv_scale;
  std::vector<int> n_per_level, lw, lh, loff;
  std::vector<int> cell_begin;  // first cell of each level (+ total)
  size_t pyr_bytes = 0;
  int ncells = 0, tile_cap = 0, max_per_cell = 0, max_cand = 0, max_kp = 0;
  BlurTaps taps;
  DevBuf<uint8_t> pyr, blurred, desc;
  DevBuf<Cell> cells;
  DevBuf<LevelRef> levels;
  DevBuf<int> cell_count, cell_off, xofs, yofs;
  DevBuf<short> xa, ya;
  std::vector<size_t> tab_x, tab_y;  // per-level offsets into xofs/yofs
  DevBuf<ushort4> cell_out;
  DevBuf<Cand> cand;
  DevBuf<KpIn> kp_in;
  uint8_t* h_img = nullptr;   // pinned staging
  Cand* h_cand = nullptr;     // pinned
  int* h_total = nullptr;     // pinned
  KpIn* h_kp = nullptr;       // pinned
  uint8_t* h_desc = nullptr;  // pinned
  ~ccm_orb_handle() {
    if (h_img) cudaFreeHost(h_img);
    if (h_cand) cudaFreeHost(h_cand);
    if (h_total) cudaFreeHost(h_total);
    if (h_kp) cudaFreeHost(h_kp);
    if (h_desc) cudaFreeHost(h_desc);
    if (stream) cudaStreamDestroy(stream);
  }
};

namespace {

void orb_build(ccm_orb_handle* h, const ccm_orb_config* cfg, int width, int height) {
  ensure_device();
  CCM_REQUIRE(cfg && cfg->nlevels >= 1 && cfg->nlevels <= 16 && cfg->nfeatures > 0 && cfg->scale_factor > 1.0f, "ccm_orb_create: bad config");
  h->cfg = *cfg; h->width = width; h->height = height; h->device = current_device();
  CCM_CUDA(cudaStreamCreateWithFlags(&h->stream, cudaStreamNonBlocking));
  cudaStream_t s = h->stream;
  const int nl = cfg->nlevels;
  // ORBextractor::ORBextractor (S/ORBextractor.cpp:579-639)
  h->scale.resize(nl); h->inv_scale.resize(nl);
  h->scale[0] = 1.0f;
  for (int i = 1; i < nl; i++) h->scale[i] = h->scale[i - 1] * cfg->scale_factor;
  for (int i = 0; i < nl; i++) h->inv_scale[i] = 1.0f / h->scale[i];
  h->n_per_level.resize(nl);
  {
    const float factor = 1.0f / cfg->scale_factor;
    float nDesired = cfg->nfeatures * (1 - factor) / (1 - (float)pow((double)factor, (double)nl));
    int sum = 0;
    for (int l = 0; l < nl - 1; l++) {
      h->n_per_level[l] = cv_round(nDesired);
      sum += h->n_per_level[l];
      nDesired *= factor;
    }
    h->n_per_level[nl - 1] = std::max(cfg->nfeatures - sum, 0);
  }
  int umax[16];
  {
    int v, v0;
    const int vmax = (int)std::floor(kHalfPatch * std::sqrt(2.f) / 2 + 1);
    const int vmin = (int)std::ceil(kHalfPatch * std::sqrt(2.f) / 2);
    const double hp2 = kHalfPatch * kHalfPatch;
    for (v = 0; v <= vmax; ++v) umax[v] = (int)lrint(std::sqrt(hp2 - v * v));
    for (v = kHalfPatch, v0 = 0; v >= vmin; --v) {
      while (umax[v0] == umax[v0 + 1]) ++v0;
      umax[v] = v0;
      ++v0;
    }
  }
  CCM_CUDA(cudaMemcpyToSymbolAsync(c_umax, umax, sizeof(umax), 0, cudaMemcpyHostToDevice, s));
  CCM_CUDA(cudaMemcpyToSymbolAsync(c_pattern, kOrbPattern, 1024, 0, cudaMemcpyHostToDevice, s));
  static const BlurTaps taps4 = {{18, 34, 48, 56, 48, 34, 18}}, taps2 = {{18, 34, 49, 55, 49, 34, 18}};
  h->taps = cfg->blur_2413 ? taps2 : taps4;
  // level geometry (ComputePyramid)
  h->lw.resize(nl); h->lh.resize(nl); h->loff.resize(nl);
  size_t off = 0;
  std::vector<LevelRef> lref(nl);
  for (int l = 0; l < nl; l++) {
    h->lw[l] = cv_round((float)width * h->inv_scale[l]);
    h->lh[l] = cv_round((float)height * h->inv_scale[l]);
    CCM_REQUIRE(h->lw[l] > 2 * kEdge + 6 && h->lh[l] > 2 * kEdge + 6, "ccm_orb_create: image too small for the pyramid depth");
    h->loff[l] = (int)off;
    lref[l] = LevelRef{(int)off, h->lw[l], h->lh[l]};
    off += ((size_t)h->lw[l] * h->lh[l] + 255) / 256 * 256;
  }
  h->pyr_bytes = off;
  h->pyr.alloc(off); h->blurred.alloc(off);
  h->levels.upload(lref.data(), nl, s);
  // resize coefficient tables, as cv::resize builds them (float fraction, 11-bit fixed point, clamped)
  std::vector<int> xo, yo; std::vector<short> xal, yal;
  h->tab_x.assign(nl, 0); h->tab_y.assign(nl, 0);
  auto coeff = [](int d, double sc, int n, int& sidx, short& a0, short& a1) {
    float f = (float)((d + 0.5) * sc - 0.5);
    sidx = (int)std::floor(f);
    f -= sidx;
    if (sidx < 0) { sidx = 0; f = 0.f; }
    if (sidx >= n - 1) { sidx = n - 1; f = 0.f; }
    a0 = (short)std::max(-32768, std::min(32767, cv_round((1.f - f) * 2048.f)));
    a1 = (short)std::max(-32768, std::min(32767, cv_round(f * 2048.f)));
  };
  for (int l = 1; l < nl; l++) {
    h->tab_x[l] = xo.size(); h->tab_y[l] = yo.size();
    const double sx = (double)h->lw[l - 1] / h->lw[l], sy = (double)h->lh[l - 1] / h->lh[l];
    for (int x = 0; x < h->lw[l]; x++) { int si; short a0, a1; coeff(x, sx, h->lw[l - 1], si, a0, a1); xo.push_back(si); xal.push_back(a0); xal.push_back(a1); }
    for (int y = 0; y < h->lh[l]; y++) { int si; short a0, a1; coeff(y, sy, h->lh[l - 1], si, a0, a1); yo.push_back(si); yal.push_back(a0); yal.push_back(a1); }
  }
  if (xo.empty()) { xo.push_back(0); yo.push_back(0); xal.assign(2, 0); yal.assign(2, 0); }
  h->xofs.upload(xo.data(), xo.size(), s); h->yofs.upload(yo.data(), yo.size(), s);
  h->xa.upload(xal.data(), xal.size(), s); h->ya.upload(yal.data(), yal.size(), s);
  // FAST cells (ComputeKeyPointsOctTree, S/ORBextractor.cpp:937-976)
  std::vector<Cell> cells;
  h->cell_begin.assign(nl + 1, 0);
  int out_off = 0;
  h->tile_cap = 0; h->max_per_cell = 0;
  const float W = 30;
  for (int l = 0; l < nl; l++) {
    h->cell_begin[l] = (int)cells.size();
    const int minBX = kEdge - 3, minBY = minBX, maxBX = h->lw[l] - kEdge + 3, maxBY = h->lh[l] - kEdge + 3;
    const float wid = (float)(maxBX - minBX), hei = (float)(maxBY - minBY);
    const int nCols = (int)(wid / W), nRows = (int)(hei / W);
    CCM_REQUIRE(nCols >= 1 && nRows >= 1, "ccm_orb_create: pyramid level smaller than one FAST cell");
    const int wCell = (int)std::ceil(wid / nCols), hCell = (int)std::ceil(hei / nRows);
    for (int i = 0; i < nRows; i++) {
      const float iniY = (float)(minBY + i * hCell);
      float maxY = iniY + hCell + 6;
      if (iniY >= maxBY - 3) continue;
      if (maxY > maxBY) maxY = (float)maxBY;
      for (int j = 0; j < nCols; j++) {
        const float iniX = (float)(minBX + j * wCell);
        float maxX = iniX + wCell + 6;
        if (iniX >= maxBX - 6) continue;
        if (maxX > maxBX) maxX = (float)maxBX;
        Cell c;
        c.level = l; c.img_off = h->loff[l]; c.img_w = h->lw[l];
        c.x0 = (int)iniX; c.y0 = (int)iniY; c.x1 = (int)maxX; c.y1 = (int)maxY;
        cells.push_back(c);
        const int tw = c.x1 - c.x0, th = c.y1 - c.y0;
        h->tile_cap = std::max(h->tile_cap, tw * th);
        h->max_per_cell = std::max(h->max_per_cell, ((std::max(tw - 6, 0) + 1) / 2) * ((std::max(th - 6, 0) + 1) / 2));
      }
    }
  }
  h->cell_begin[nl] = (int)cells.size();
  h->ncells = (int)cells.size();
  h->max_per_cell = std::max(h->max_per_cell, 1);
  for (auto& c : cells) { c.out_off = out_off; out_off += h->max_per_cell; }
  CCM_REQUIRE((size_t)h->tile_cap * 4 + 64 < 200 * 1024, "ccm_orb_create: FAST cell too large for shared memory");
  h->cells.upload(cells.data(), cells.size(), s);
  h->cell_count.alloc(h->ncells); h->cell_off.alloc((size_t)h->ncells + 1);
  h->cell_out.alloc((size_t)out_off);
  // The reference never caps the candidate list (vToDistributeKeys.reserve only reserves), so the gather buffers take every
  // per-cell slot: out_off * sizeof(Cand) pinned and on the device, 7.2 MB each at 752x480 with the default configuration.
  h->max_cand = out_off;
  h->cand.alloc(h->max_cand);
  // Keypoint capacity: DistributeOctTree (S/ORBextractor.cpp:707-931) keeps one keypoint per node.  On a level with quota N
  // it starts from nIni root nodes and its first pass splits every root holding more than one candidate, so that pass alone
  // can leave 4 * nIni nodes whatever N is.  Every later full pass runs only if the node count plus three per splittable
  // node is at most N, so it cannot exceed N.  The node-by-node loop splits only while fewer than N nodes exist, and one
  // split adds at most three, so it stops below N + 3.  Hence at most max(4 * nIni, N + 3) keypoints per level.
  h->max_kp = 0;
  for (int l = 0; l < nl; l++)
    h->max_kp += std::max(4 * quadtree_roots(kEdge - 3, h->lw[l] - kEdge + 3, kEdge - 3, h->lh[l] - kEdge + 3), h->n_per_level[l] + 3);
  h->kp_in.alloc(h->max_kp); h->desc.alloc((size_t)h->max_kp * 32);
  CCM_CUDA(cudaMallocHost((void**)&h->h_img, (size_t)width * height));
  CCM_CUDA(cudaMallocHost((void**)&h->h_cand, sizeof(Cand) * (size_t)h->max_cand));
  CCM_CUDA(cudaMallocHost((void**)&h->h_total, sizeof(int) * 4));
  h->h_total[0] = 0;  // ccm_orb_debug_candidates before the first extract reports an empty list
  CCM_CUDA(cudaMallocHost((void**)&h->h_kp, sizeof(KpIn) * (size_t)h->max_kp));
  CCM_CUDA(cudaMallocHost((void**)&h->h_desc, (size_t)h->max_kp * 32));
  const size_t smem = ((size_t)h->tile_cap + 15) / 16 * 16 + 3 * (size_t)h->tile_cap + 16;
  if (smem > 48 * 1024) CCM_CUDA(cudaFuncSetAttribute(k_fast_cells, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  CCM_CUDA(cudaStreamSynchronize(s));
}

void orb_extract(ccm_orb_handle* h, const uint8_t* img, int stride, ccm_keypoint* kps, int max_kp, int* n_out, uint8_t* desc) {
  CCM_CUDA(cudaSetDevice(h->device));
  cudaStream_t s = h->stream;
  const int nl = h->cfg.nlevels;
  for (int y = 0; y < h->height; y++) memcpy(h->h_img + (size_t)y * h->width, img + (size_t)y * stride, h->width);
  CCM_CUDA(cudaMemcpyAsync(h->pyr.p, h->h_img, (size_t)h->width * h->height, cudaMemcpyHostToDevice, s));
  for (int l = 1; l < nl; l++) {
    dim3 b(32, 8), g(div_up(h->lw[l], 32), div_up(h->lh[l], 8));
    k_resize<<<g, b, 0, s>>>(h->pyr.p + h->loff[l - 1], h->lw[l - 1], h->lh[l - 1], h->pyr.p + h->loff[l], h->lw[l], h->lh[l],
                             h->xofs.p + h->tab_x[l], h->xa.p + 2 * h->tab_x[l], h->yofs.p + h->tab_y[l], h->ya.p + 2 * h->tab_y[l]);
    CCM_LAUNCHED();
  }
  const size_t smem = ((size_t)h->tile_cap + 15) / 16 * 16 + 3 * (size_t)h->tile_cap + 16;
  k_fast_cells<<<h->ncells, 256, smem, s>>>(h->pyr.p, h->cells.p, h->cfg.ini_th_fast, h->cfg.min_th_fast, h->tile_cap,
                                            h->max_per_cell, h->cell_count.p, h->cell_out.p);
  CCM_LAUNCHED();
  k_scan_cells<<<1, 1024, 0, s>>>(h->cell_count.p, h->ncells, h->cell_off.p);
  CCM_LAUNCHED();
  k_gather<<<h->ncells, 128, 0, s>>>(h->pyr.p, h->cells.p, h->cell_count.p, h->cell_off.p, h->cell_out.p, h->max_cand, h->cand.p);
  CCM_LAUNCHED();
  CCM_CUDA(cudaMemcpyAsync(h->h_total, h->cell_off.p + h->ncells, sizeof(int), cudaMemcpyDeviceToHost, s));
  // per-level first-candidate offsets = cell_off at the first cell of each level
  std::vector<int> lvl_off(nl + 1);
  // the blur of every level overlaps with the host-side quadtree below
  for (int l = 0; l < nl; l++) {
    dim3 g(div_up(h->lw[l], 32), div_up(h->lh[l], 16));
    k_blur<<<g, 256, 0, s>>>(h->pyr.p + h->loff[l], h->blurred.p + h->loff[l], h->lw[l], h->lh[l], h->taps);
    CCM_LAUNCHED();
  }
  // copy an optimistic prefix of the candidates together with the count, top up if there are more
  const int first = std::min(h->max_cand, 16384);
  CCM_CUDA(cudaMemcpyAsync(h->h_cand, h->cand.p, sizeof(Cand) * (size_t)first, cudaMemcpyDeviceToHost, s));
  CCM_CUDA(cudaStreamSynchronize(s));
  const int total = h->h_total[0];
  CCM_REQUIRE(total <= h->max_cand, "internal: more FAST candidates than per-cell slots");
  if (total > first) {
    CCM_CUDA(cudaMemcpyAsync(h->h_cand + first, h->cand.p + first, sizeof(Cand) * (size_t)(total - first), cudaMemcpyDeviceToHost, s));
    CCM_CUDA(cudaStreamSynchronize(s));
  }
  // candidates are ordered by level already (cells are level-major)
  int pos = 0;
  for (int l = 0; l < nl; l++) {
    lvl_off[l] = pos;
    while (pos < total && h->h_cand[pos].level == l) pos++;
  }
  lvl_off[nl] = pos;
  std::vector<ccm_keypoint> out;
  std::vector<KpIn> kin;
  const float factorPI = (float)(M_PI / 180.f);
  for (int l = 0; l < nl; l++) {
    const Cand* c = h->h_cand + lvl_off[l];
    const int nc = lvl_off[l + 1] - lvl_off[l];
    const int minBX = kEdge - 3, minBY = minBX, maxBX = h->lw[l] - kEdge + 3, maxBY = h->lh[l] - kEdge + 3;
    const std::vector<int> sel = distribute(c, nc, minBX, maxBX, minBY, maxBY, h->n_per_level[l]);
    const int scaledPatch = (int)(kPatch * h->scale[l]);
    for (int id : sel) {
      const Cand& k = c[id];
      ccm_keypoint kp;
      kp.x = k.x + minBX; kp.y = k.y + minBY;
      kp.octave = l; kp.size = (float)scaledPatch; kp.response = (float)k.score;
      kp.angle = fast_atan2_host((float)k.m01, (float)k.m10);
      KpIn ki;
      ki.level = l; ki.cx = cv_round(kp.x); ki.cy = cv_round(kp.y);
      const float ang = kp.angle * factorPI;
      ki.a = cosf(ang); ki.b = sinf(ang);
      kin.push_back(ki);
      if (l != 0) { kp.x *= h->scale[l]; kp.y *= h->scale[l]; }
      out.push_back(kp);
    }
  }
  const int n = (int)out.size();
  CCM_REQUIRE(n <= h->max_kp, "internal: more keypoints than ccm_orb_max_keypoints");
  *n_out = n;
  CCM_REQUIRE(n <= max_kp, "ccm_orb_extract: " + std::to_string(n) + " keypoints, max_kp is " + std::to_string(max_kp) +
                               " (size kps and desc with ccm_orb_max_keypoints)");
  if (n > 0) {
    memcpy(h->h_kp, kin.data(), sizeof(KpIn) * (size_t)n);
    CCM_CUDA(cudaMemcpyAsync(h->kp_in.p, h->h_kp, sizeof(KpIn) * (size_t)n, cudaMemcpyHostToDevice, s));
    k_descriptors<<<div_up((long long)n * 32, 128), 128, 0, s>>>(h->blurred.p, h->levels.p, h->kp_in.p, n, h->desc.p);
    CCM_LAUNCHED();
    CCM_CUDA(cudaMemcpyAsync(h->h_desc, h->desc.p, (size_t)n * 32, cudaMemcpyDeviceToHost, s));
    CCM_CUDA(cudaStreamSynchronize(s));
  }
  for (int i = 0; i < n; i++) kps[i] = out[i];
  if (desc && n) memcpy(desc, h->h_desc, (size_t)n * 32);
}

}  // namespace

extern "C" int ccm_orb_create(const ccm_orb_config* cfg, int32_t width, int32_t height, ccm_orb_handle** out) {
  return guarded([&] {
    CCM_REQUIRE(out, "ccm_orb_create: out is NULL");
    *out = nullptr;
    ccm_orb_handle* h = new ccm_orb_handle();
    try {
      orb_build(h, cfg, width, height);
    } catch (...) {
      delete h;
      throw;
    }
    *out = h;
  });
}

extern "C" int ccm_orb_extract(ccm_orb_handle* h, const uint8_t* img, int32_t stride, ccm_keypoint* kps, int32_t max_kp,
                               int32_t* n, uint8_t* desc) {
  return guarded([&] {
    CCM_REQUIRE(h && img && kps && n && max_kp >= 0 && stride >= h->width, "ccm_orb_extract: bad argument");
    orb_extract(h, img, stride, kps, max_kp, n, desc);
  });
}

extern "C" int ccm_orb_max_keypoints(const ccm_orb_handle* h, int32_t* n) {
  return guarded([&] {
    CCM_REQUIRE(h && n, "ccm_orb_max_keypoints: null argument");
    *n = h->max_kp;
  });
}

// debug: the candidate list of the last ccm_orb_extract call (x, y relative to minBorder, score, level), reference order
extern "C" int ccm_orb_debug_candidates(ccm_orb_handle* h, float* xys, int32_t* level, int32_t max_out, int32_t* n) {
  return guarded([&] {
    CCM_REQUIRE(h && n, "null argument");
    const int total = h->h_total[0];
    *n = total;
    for (int i = 0; i < std::min(total, max_out); i++) {
      xys[3 * i] = h->h_cand[i].x; xys[3 * i + 1] = h->h_cand[i].y; xys[3 * i + 2] = (float)h->h_cand[i].score;
      level[i] = h->h_cand[i].level;
    }
  });
}

extern "C" int ccm_orb_get_level(ccm_orb_handle* h, int32_t level, uint8_t* out, int32_t* w, int32_t* hgt) {
  return guarded([&] {
    CCM_REQUIRE(h && level >= 0 && level < h->cfg.nlevels, "ccm_orb_get_level: bad level");
    CCM_CUDA(cudaSetDevice(h->device));
    if (w) *w = h->lw[level];
    if (hgt) *hgt = h->lh[level];
    if (out) {
      CCM_CUDA(cudaMemcpyAsync(out, h->pyr.p + h->loff[level], (size_t)h->lw[level] * h->lh[level], cudaMemcpyDeviceToHost, h->stream));
      CCM_CUDA(cudaStreamSynchronize(h->stream));
    }
  });
}

// debug: the blurred pyramid level the descriptors of the last ccm_orb_extract call sampled
extern "C" int ccm_orb_debug_blurred(ccm_orb_handle* h, int32_t level, uint8_t* out) {
  return guarded([&] {
    CCM_REQUIRE(h && out && level >= 0 && level < h->cfg.nlevels, "ccm_orb_debug_blurred: bad argument");
    CCM_CUDA(cudaSetDevice(h->device));
    CCM_CUDA(cudaMemcpyAsync(out, h->blurred.p + h->loff[level], (size_t)h->lw[level] * h->lh[level], cudaMemcpyDeviceToHost, h->stream));
    CCM_CUDA(cudaStreamSynchronize(h->stream));
  });
}

extern "C" void ccm_orb_destroy(ccm_orb_handle* h) {
  if (!h) return;
  cudaSetDevice(h->device);
  if (h->stream) cudaStreamSynchronize(h->stream);
  delete h;
}

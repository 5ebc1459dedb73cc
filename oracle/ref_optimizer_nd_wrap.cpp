// ref_optimizer_nd_wrap.cpp — TEST INFRASTRUCTURE: what the five write-back loops of shim/Optimizer_shim.cpp leave in the map points
// when shim/MapPoint_shim.cpp is linked next to it (oracle/Makefile: _ref/liboptimizer_nd_shim{,_gpu}.so).
//
// The optimiser calls themselves are ref_optimizer_wrap.cpp's (optw_gba, optw_gba_mirror, optw_local_ba, optw_essential_graph), linked
// unchanged into the same library over the stand-ins of ref_stub_opt_mp.  Their scene is destroyed when they return; each MapPoint
// hands itself to MapPoint::on_destroy first, and the sink installed here records, per point (indexed by mUniqueId - uid_base):
//   * the members the write-back left (mNormalVector, mfMaxDistance, mfMinDistance; written = mNormalVector non-empty);
//   * the same members recomputed for that point alone on the host: the parked table is empty by then, so the member takes its
//     single-point path (ccm_normal_depth_host) on the state the write-back left.
// The member's outcome counters (ccm_b200_normals_stats) are read before the first recomputation.
#include <cslam/MapPoint.h>

#include <cstdint>
#include <cstring>

#include "../shim/MapPoint_shim.h"

using namespace cslam;

void (*MapPoint::on_destroy)(MapPoint&) = nullptr;

namespace {

struct Sink {
  int64_t uid_base = 0;
  int32_t P = 0;
  float *loop_normal = nullptr, *loop_max = nullptr, *loop_min = nullptr, *host_normal = nullptr, *host_max = nullptr, *host_min = nullptr;
  uint8_t *loop_written = nullptr, *host_written = nullptr;
  unsigned long long counts[3] = {0, 0, 0};
  bool counted = false;
} g_sink;

void read_members(MapPoint& m, float* normal, float* dmax, float* dmin, uint8_t* written) {
  *written = m.mNormalVector.empty() ? 0 : 1;
  if (*written) for (int j = 0; j < 3; j++) normal[j] = m.mNormalVector.at<float>(j);
  *dmax = m.mfMaxDistance; *dmin = m.mfMinDistance;
}

void record(MapPoint& m) {
  Sink& s = g_sink;
  if (!s.counted) { ccm_b200_normals_stats(&s.counts[0], &s.counts[1], &s.counts[2]); s.counted = true; }
  const int64_t j = (int64_t)m.mUniqueId - s.uid_base;
  if (j < 0 || j >= s.P) return;
  read_members(m, s.loop_normal + 3 * j, s.loop_max + j, s.loop_min + j, s.loop_written + j);
  m.mNormalVector.release(); m.mfMaxDistance = m.mfMinDistance = 0.f;
  m.UpdateNormalAndDepth();
  read_members(m, s.host_normal + 3 * j, s.host_max + j, s.host_min + j, s.host_written + j);
}

}  // namespace

extern "C" {

/* arm the sink for the next optw_* call on a scene of P points with mUniqueId = uid_base + j; all arrays P (normals P*3) */
void ndw_arm(int64_t uid_base, int32_t P, float* loop_normal, float* loop_max, float* loop_min, uint8_t* loop_written, float* host_normal,
             float* host_max, float* host_min, uint8_t* host_written) {
  g_sink = Sink();
  g_sink.uid_base = uid_base; g_sink.P = P;
  g_sink.loop_normal = loop_normal; g_sink.loop_max = loop_max; g_sink.loop_min = loop_min; g_sink.loop_written = loop_written;
  g_sink.host_normal = host_normal; g_sink.host_max = host_max; g_sink.host_min = host_min; g_sink.host_written = host_written;
  std::memset(loop_written, 0, (size_t)P); std::memset(host_written, 0, (size_t)P);
  MapPoint::on_destroy = record;
}

/* disarm; counts[3] = the member's outcome counters (hits, stale, host) as they stood when the scene went away */
void ndw_disarm(unsigned long long* counts) {
  MapPoint::on_destroy = nullptr;
  if (!g_sink.counted) ccm_b200_normals_stats(&g_sink.counts[0], &g_sink.counts[1], &g_sink.counts[2]);
  for (int i = 0; i < 3; i++) counts[i] = g_sink.counts[i];
}

void ndw_stats(unsigned long long* counts) { ccm_b200_normals_stats(&counts[0], &counts[1], &counts[2]); }

}  // extern "C"

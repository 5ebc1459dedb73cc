// KeyFrameConnections_shim.h — the batch entry of shim/KeyFrameConnections_shim.cpp, for the loops that call
// KeyFrame::UpdateConnections on many keyframes (INTEGRATION.md §4e).
#ifndef CCM_KEYFRAME_CONNECTIONS_SHIM_H
#define CCM_KEYFRAME_CONNECTIONS_SHIM_H
#include <vector>

#include <boost/shared_ptr.hpp>

namespace cslam {

class KeyFrame;

// Counts the covisibility weights of every keyframe in one ccm_covisibility call and parks each keyframe's counter, per thread, for
// the KeyFrame::UpdateConnections() calls that follow.  Each distinct map point's observations are copied once.  A parked counter is
// used only while the keyframe's mvpMapPoints is element for element the one it was counted from and every point in it still has the
// isBad() and Observations() it had then; the member counts on the host otherwise.
void ccm_b200_prepare_connections(const std::vector<boost::shared_ptr<KeyFrame> >& keyframes);
// Drops every counter parked on this thread.
void ccm_b200_clear_connections();
// Counts of KeyFrame::UpdateConnections() calls since the process started, by how they ended: a parked counter used, a parked
// counter found stale (then counted on the host), counted on the host.
void ccm_b200_connections_stats(unsigned long long* hits, unsigned long long* stale, unsigned long long* host);

// Clears the parked counters when a loop ends, by any path.
struct ParkedConnectionsGuard {
  ParkedConnectionsGuard() {}
  ~ParkedConnectionsGuard() { ccm_b200_clear_connections(); }
  ParkedConnectionsGuard(const ParkedConnectionsGuard&) = delete;
  ParkedConnectionsGuard& operator=(const ParkedConnectionsGuard&) = delete;
};

}  // namespace cslam
#endif

// KeyFrameCulling_shim.h — what shim/KeyFrameCulling_shim.cpp offers besides the member it defines, LocalMapping::KeyFrameCullingV3
// (INTEGRATION.md §4j).
#ifndef CCM_KEYFRAME_CULLING_SHIM_H
#define CCM_KEYFRAME_CULLING_SHIM_H

namespace cslam {

// Counts since the process started: library calls made by LocalMapping::KeyFrameCullingV3, and candidates the library counted again on
// the host because an earlier cull of the same call reached one of their points (the call's n_settled, summed).
void ccm_b200_keyframe_culling_stats(unsigned long long* calls, unsigned long long* settled);

}  // namespace cslam
#endif

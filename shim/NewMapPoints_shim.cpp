// NewMapPoints_shim.cpp — LocalMapping::CreateNewMapPoints (cslam/src/Mapping.cpp:284-469) over ccm_new_map_points.
//
// Replace the member's body in Mapping.cpp by this translation unit (INTEGRATION.md §4f).  What stays the reference's own, verbatim:
// the neighbour list, the baseline / ComputeSceneMedianDepth skip (:320-328), ComputeF12 (:331), the epipole as SearchForTriangulation
// forms it (cslam/src/ORBmatcher.cpp:707-714), and the sequence applied to each new point (:451-466).  What the library does in one
// call: SearchForTriangulation for every neighbour, the triangulation of every match and its gates (:333-448).
//
// The reference polls CheckNewKeyFrames() before each neighbour after the first (:314) and returns.  The shim polls at the same points
// while applying the result, neighbour by neighbour over the ORIGINAL neighbour list (skipped ones included, as the poll precedes
// the skip), and drops the points of the remaining neighbours.  That is the prefix the reference would have produced, because the
// result for neighbour i depends only on the neighbours before it.
#include "NewMapPoints_shim.h"

#include <atomic>
#include <vector>

#include <cslam/Mapping.h>
#include <cslam/estd.h>

#include "ccm_b200.h"

namespace cslam {

namespace {
std::atomic<unsigned long long> g_calls(0), g_created(0), g_dropped(0);

struct FlatView {   // keeps the arrays a ccm_newpts_view points to
  std::vector<uint8_t> has_mp;
  std::vector<float> xy, angle;
  std::vector<int32_t> octave, node_ptr;
  std::vector<uint32_t> node_id, feat;
  ccm_feature_vector fv;
};

void flatten(const LocalMapping::kfptr& pKF, FlatView& f, ccm_newpts_view& v) {
  const int N = pKF->N;
  f.has_mp.resize(N); f.xy.resize(2 * (size_t)N); f.angle.resize(N); f.octave.resize(N);
  for (int i = 0; i < N; i++) {
    f.has_mp[i] = pKF->GetMapPoint(i) ? 1 : 0;
    const cv::KeyPoint& kp = pKF->mvKeysUn[i];
    f.xy[2 * i] = kp.pt.x; f.xy[2 * i + 1] = kp.pt.y; f.angle[i] = kp.angle; f.octave[i] = kp.octave;
  }
  f.node_ptr.assign(1, 0);
  for (DBoW2::FeatureVector::const_iterator it = pKF->mFeatVec.begin(); it != pKF->mFeatVec.end(); ++it) {   // std::map: node ids ascending
    f.node_id.push_back(it->first);
    f.feat.insert(f.feat.end(), it->second.begin(), it->second.end());
    f.node_ptr.push_back((int32_t)f.feat.size());
  }
  f.fv.n_nodes = (int32_t)f.node_id.size(); f.fv.node_id = f.node_id.data(); f.fv.node_ptr = f.node_ptr.data(); f.fv.feat = f.feat.data();
  v.v.desc = pKF->mDescriptors.ptr(); v.v.n = N; v.v.has_mp = f.has_mp.data(); v.v.kp_xy = f.xy.data(); v.v.octave = f.octave.data();
  v.v.angle = f.angle.data(); v.v.fv = &f.fv;
  v.v.fx = pKF->fx; v.v.fy = pKF->fy; v.v.cx = pKF->cx; v.v.cy = pKF->cy;
  const cv::Mat R = pKF->GetRotation(), t = pKF->GetTranslation(), O = pKF->GetCameraCenter();
  for (int r = 0; r < 3; r++) {
    for (int c = 0; c < 3; c++) v.Tcw[4 * r + c] = R.at<float>(r, c);
    v.Tcw[4 * r + 3] = t.at<float>(r);
    v.Ow[r] = O.at<float>(r);
  }
  v.level_sigma2 = pKF->mvLevelSigma2.data(); v.scale_factors = pKF->mvScaleFactors.data();
  v.nlevels = (int32_t)pKF->mvScaleFactors.size(); v.scale_factor = pKF->mfScaleFactor;
}
}  // namespace

void ccm_b200_new_map_points_stats(unsigned long long* calls, unsigned long long* created, unsigned long long* dropped) {
  if (calls) *calls = g_calls.load();
  if (created) *created = g_created.load();
  if (dropped) *dropped = g_dropped.load();
}

void LocalMapping::CreateNewMapPoints()
{
    // Retrieve neighbor keyframes in covisibility graph
    int nn=20;
    const std::vector<kfptr> vpNeighKFs = mpCurrentKeyFrame->GetBestCovisibilityKeyFrames(nn);

    cv::Mat Ow1 = mpCurrentKeyFrame->GetCameraCenter();

    // the prelude of every neighbour (:317-331); vPassed[k] = index into vpNeighKFs of the k-th neighbour handed to the library
    std::vector<int> vPassed;
    std::vector<ccm_newpts_neighbour> vNb;
    std::vector<FlatView> vFlat(vpNeighKFs.size() + 1);
    ccm_newpts_view cur;
    flatten(mpCurrentKeyFrame, vFlat[0], cur);
    vNb.reserve(vpNeighKFs.size());
    for(size_t i=0; i<vpNeighKFs.size(); i++)
    {
        kfptr pKF2 = vpNeighKFs[i];

        // Check first that baseline is not too short
        cv::Mat Ow2 = pKF2->GetCameraCenter();
        cv::Mat vBaseline = Ow2-Ow1;
        const float baseline = cv::norm(vBaseline);

        const float medianDepthKF2 = pKF2->ComputeSceneMedianDepth(2);
        const float ratioBaselineDepth = baseline/medianDepthKF2;

        if(ratioBaselineDepth<0.01)
            continue;

        // Compute Fundamental Matrix
        cv::Mat F12 = ComputeF12(mpCurrentKeyFrame,pKF2);

        ccm_newpts_neighbour nb;
        flatten(pKF2, vFlat[i + 1], nb.view);
        for (int r = 0; r < 3; r++) for (int c = 0; c < 3; c++) nb.F12[3 * r + c] = F12.at<float>(r, c);
        // Compute epipole in second image (ORBmatcher.cpp:707-714)
        cv::Mat Cw = mpCurrentKeyFrame->GetCameraCenter();
        cv::Mat R2w = pKF2->GetRotation();
        cv::Mat t2w = pKF2->GetTranslation();
        cv::Mat C2 = R2w*Cw+t2w;
        const float invz = 1.0f/C2.at<float>(2);
        nb.ex =pKF2->fx*C2.at<float>(0)*invz+pKF2->cx;
        nb.ey =pKF2->fy*C2.at<float>(1)*invz+pKF2->cy;
        vNb.push_back(nb);
        vPassed.push_back((int)i);
    }

    std::vector<ccm_new_point> vOut((size_t)mpCurrentKeyFrame->N * vNb.size() + 1);
    int32_t nOut = 0;
    g_calls++;
    if (ccm_new_map_points(&cur, vNb.data(), (int32_t)vNb.size(), vOut.data(), (int32_t)vOut.size(), &nOut, nullptr, nullptr) != CCM_OK)
        throw estd::infrastructure_ex();

    // apply, neighbour by neighbour over the original list, polling where the reference polls (:314)
    int at = 0;      // next record of vOut
    size_t k = 0;    // next entry of vPassed
    for(size_t i=0; i<vpNeighKFs.size(); i++)
    {
        if(i>0 && CheckNewKeyFrames())
        {
            g_dropped += (unsigned long long)(nOut - at);
            return;
        }
        if (k >= vPassed.size() || vPassed[k] != (int)i)
            continue;   // skipped for its baseline
        kfptr pKF2 = vpNeighKFs[i];
        for (; at < nOut && vOut[at].nb == (int32_t)k; at++)
        {
            const int idx1 = vOut[at].idx1;
            const int idx2 = vOut[at].idx2;
            cv::Mat x3D(3,1,CV_32F);
            for (int r = 0; r < 3; r++) x3D.at<float>(r) = vOut[at].x3D[r];

            // Triangulation is succesfull
            mpptr pMP{new MapPoint(x3D,mpCurrentKeyFrame,mpMap,mClientId,mpComm,mpCC->mSysState,-1)};

            pMP->AddObservation(mpCurrentKeyFrame,idx1);
            pMP->AddObservation(pKF2,idx2);

            mpCurrentKeyFrame->AddMapPoint(pMP,idx1);
            pKF2->AddMapPoint(pMP,idx2);

            pMP->ComputeDistinctiveDescriptors();

            pMP->UpdateNormalAndDepth();

            mpMap->AddMapPoint(pMP);
            mlpRecentAddedMapPoints.push_back(pMP);
            g_created++;
        }
        k++;
    }
}

}  // namespace cslam

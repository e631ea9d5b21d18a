// Drop-in DEFINITIONS of Optimizer::PoseOptimization / LocalBundleAdjustment / BundleAdjustment / GlobalBundleAdjustemnt on top of
// libcubemap_b200.so. This file is compiled INSIDE the CubemapSLAM tree against the reference's own, unmodified headers
// (include/Optimizer.h:42-63 declares exactly these signatures), so Tracking.cpp:585,647,688 and LocalMapping.cpp:86 call them unchanged.
// src/Optimizer.cpp keeps OptimizeEssentialGraph / OptimizeSim3; its four replaced bodies are renamed away at compile time
// (INTEGRATION.md: per-file COMPILE_DEFINITIONS PoseOptimization=PoseOptimization_g2o ...), no source edit.
//
// What stays caller-side logic of the reference and is therefore restated here (src/Optimizer.cpp): the gathering of correspondences
// (:80-131), the local window (:194-243), the vertex/edge list (:262-357), the outlier erase under Map::mMutexMapUpdate and the float32
// write-back (:399-450). The g2o graph, LM and Schur solve are cslam_pose_optimization / cslam_local_ba.
#include "Optimizer.h"

#include <cstdio>
#include <cstdlib>
#include <list>
#include <map>
#include <mutex>
#include <vector>

#include "cubemap_b200.h"

namespace {
cslam_optimizer* b200_optimizer() {   // one handle per host thread (Tracking, LocalMapping and the GBA thread all optimise)
    static thread_local cslam_optimizer* o = nullptr;
    if (!o && cslam_optimizer_create(&o, 0) != CSLAM_OK) { std::fprintf(stderr, "Optimizer (cubemap_b200): %s\n", cslam_last_error()); std::exit(EXIT_FAILURE); }
    return o;
}
void b200_fatal() { std::fprintf(stderr, "Optimizer (cubemap_b200): %s\n", cslam_last_error()); std::exit(EXIT_FAILURE); }
cv::Mat mat44(const float* T) { cv::Mat m(4, 4, CV_32F); for (int r = 0; r < 4; r++) for (int c = 0; c < 4; c++) m.at<float>(r, c) = T[4 * r + c]; return m; }
}  // namespace

// reference src/Optimizer.cpp:48-190
int Optimizer::PoseOptimization(Frame* pFrame) {
    CamModelGeneral* cam = CamModelGeneral::GetCamera();
    const int N = pFrame->N;
    std::vector<float> Xw, kp, w; std::vector<int> idx;
    {
        std::unique_lock<std::mutex> lock(MapPoint::mGlobalMutex);
        for (int i = 0; i < N; i++) {
            const cv::Vec3f& ray = pFrame->mvKeyRays[i];
            if (ray(2) < cam->GetCosFovTh()) continue;
            MapPoint* pMP = pFrame->mvpMapPoints[i];
            if (!pMP) continue;
            pFrame->mvbOutlier[i] = false;
            const cv::KeyPoint& k = pFrame->mvKeys[i];
            const cv::Mat P = pMP->GetWorldPos();
            Xw.push_back(P.at<float>(0)); Xw.push_back(P.at<float>(1)); Xw.push_back(P.at<float>(2));
            kp.push_back(k.pt.x); kp.push_back(k.pt.y);
            w.push_back(pFrame->mvInvLevelSigma2[k.octave]); idx.push_back(i);
        }
    }
    const int n = (int)idx.size();
    if (n < 3) return 0;
    float T[16];
    for (int r = 0; r < 4; r++) for (int c = 0; c < 4; c++) T[4 * r + c] = pFrame->mTcw.at<float>(r, c);
    std::vector<uint8_t> out(n); int32_t off[2] = {0, n}, inl = 0;
    if (cslam_pose_optimization(b200_optimizer(), 1, off, T, Xw.data(), kp.data(), w.data(), cam->GetCubeFaceWidth(), cam->GetCubeFaceHeight(), out.data(), &inl, NULL) != CSLAM_OK) b200_fatal();
    for (int k = 0; k < n; k++) pFrame->mvbOutlier[idx[k]] = out[k] != 0;
    pFrame->SetPose(mat44(T));
    return inl;
}

namespace {
// the vertex / edge lists of one bundle adjustment in g2o's order (key frames by mnId, points by mnId), flat for the C ABI
struct Window {
    std::vector<KeyFrame*> kfList; std::vector<MapPoint*> mpList; std::vector<uint8_t> fixed;
    std::vector<float> Tcw, pts, kp, w; std::vector<int32_t> eMP, eKF; std::vector<std::pair<KeyFrame*, MapPoint*> > edgeOwner;
    void build(const std::map<unsigned long, KeyFrame*>& kfs, const std::map<unsigned long, bool>& fixedFlag, const std::map<unsigned long, MapPoint*>& mps) {
        CamModelGeneral* cam = CamModelGeneral::GetCamera();
        std::map<KeyFrame*, int> kfIndex;
        for (std::map<unsigned long, KeyFrame*>::const_iterator it = kfs.begin(); it != kfs.end(); ++it) {
            kfIndex[it->second] = (int)kfList.size(); kfList.push_back(it->second); fixed.push_back(fixedFlag.find(it->first)->second ? 1 : 0);
            const cv::Mat T = it->second->GetPose();
            for (int r = 0; r < 4; r++) for (int c = 0; c < 4; c++) Tcw.push_back(T.at<float>(r, c));
        }
        for (std::map<unsigned long, MapPoint*>::const_iterator it = mps.begin(); it != mps.end(); ++it) {
            MapPoint* pMP = it->second; const int li = (int)mpList.size(); mpList.push_back(pMP);
            const cv::Mat P = pMP->GetWorldPos();
            pts.push_back(P.at<float>(0)); pts.push_back(P.at<float>(1)); pts.push_back(P.at<float>(2));
            const std::map<KeyFrame*, size_t> observations = pMP->GetObservations();
            for (std::map<KeyFrame*, size_t>::const_iterator mit = observations.begin(); mit != observations.end(); ++mit) {
                KeyFrame* pKFi = mit->first;
                if (pKFi->isBad() || !kfIndex.count(pKFi)) continue;
                if (pKFi->mvKeyRays[mit->second](2) < cam->GetCosFovTh()) continue;       // reference :323-325 / :513-515
                const cv::KeyPoint& k = pKFi->mvKeys[mit->second];
                eMP.push_back(li); eKF.push_back(kfIndex[pKFi]); kp.push_back(k.pt.x); kp.push_back(k.pt.y);
                w.push_back(pKFi->mvInvLevelSigma2[k.octave]); edgeOwner.push_back(std::make_pair(pKFi, pMP));
            }
        }
    }
    int run(bool* pbStopFlag, int its1, int its2, std::vector<uint8_t>& outlier) {
        CamModelGeneral* cam = CamModelGeneral::GetCamera();
        cslam_ba_problem p; p.n_kf = (int)kfList.size(); p.n_mp = (int)mpList.size(); p.n_edges = (int)eMP.size();
        p.Tcw = Tcw.data(); p.kf_fixed = fixed.data(); p.points = pts.data(); p.edge_mp = eMP.data(); p.edge_kf = eKF.data(); p.kp_xy = kp.data();
        p.inv_sigma2 = w.data(); p.face_w = cam->GetCubeFaceWidth(); p.face_h = cam->GetCubeFaceHeight();
        outlier.assign(eMP.size() + 1, 0);
        cslam_ba_result r; r.outlier = outlier.data(); r.pose_fp64 = NULL; r.points_fp64 = NULL; r.lm_log = NULL; r.log_cap = 0; r.stop_after_trials = 0;
        return cslam_local_ba(b200_optimizer(), &p, reinterpret_cast<const volatile uint8_t*>(pbStopFlag), its1, its2, &r);
    }
};
}  // namespace

// reference src/Optimizer.cpp:192-451
void Optimizer::LocalBundleAdjustment(KeyFrame* pKF, bool* pbStopFlag, Map* pMap) {
    std::list<KeyFrame*> lLocalKeyFrames;
    lLocalKeyFrames.push_back(pKF);
    pKF->mnBALocalForKF = pKF->mnId;
    const std::vector<KeyFrame*> vNeighKFs = pKF->GetVectorCovisibleKeyFrames();
    for (size_t i = 0; i < vNeighKFs.size(); i++) { KeyFrame* pKFi = vNeighKFs[i]; pKFi->mnBALocalForKF = pKF->mnId; if (!pKFi->isBad()) lLocalKeyFrames.push_back(pKFi); }
    std::list<MapPoint*> lLocalMapPoints;
    for (std::list<KeyFrame*>::iterator lit = lLocalKeyFrames.begin(); lit != lLocalKeyFrames.end(); ++lit) {
        const std::vector<MapPoint*> vpMPs = (*lit)->GetMapPointMatches();
        for (size_t i = 0; i < vpMPs.size(); i++) {
            MapPoint* pMP = vpMPs[i];
            if (pMP && !pMP->isBad() && pMP->mnBALocalForKF != pKF->mnId) { lLocalMapPoints.push_back(pMP); pMP->mnBALocalForKF = pKF->mnId; }
        }
    }
    std::list<KeyFrame*> lFixedCameras;
    for (std::list<MapPoint*>::iterator lit = lLocalMapPoints.begin(); lit != lLocalMapPoints.end(); ++lit) {
        const std::map<KeyFrame*, size_t> observations = (*lit)->GetObservations();
        for (std::map<KeyFrame*, size_t>::const_iterator mit = observations.begin(); mit != observations.end(); ++mit) {
            KeyFrame* pKFi = mit->first;
            if (pKFi->mnBALocalForKF != pKF->mnId && pKFi->mnBAFixedForKF != pKF->mnId) { pKFi->mnBAFixedForKF = pKF->mnId; if (!pKFi->isBad()) lFixedCameras.push_back(pKFi); }
        }
    }
    std::map<unsigned long, KeyFrame*> kfs; std::map<unsigned long, bool> fixedFlag; std::map<unsigned long, MapPoint*> mps;
    for (std::list<KeyFrame*>::iterator it = lLocalKeyFrames.begin(); it != lLocalKeyFrames.end(); ++it) { kfs[(*it)->mnId] = *it; fixedFlag[(*it)->mnId] = ((*it)->mnId == 0); }
    for (std::list<KeyFrame*>::iterator it = lFixedCameras.begin(); it != lFixedCameras.end(); ++it) { kfs[(*it)->mnId] = *it; fixedFlag[(*it)->mnId] = true; }
    for (std::list<MapPoint*>::iterator it = lLocalMapPoints.begin(); it != lLocalMapPoints.end(); ++it) mps[(*it)->mnId] = *it;
    Window W; W.build(kfs, fixedFlag, mps);
    if (pbStopFlag && *pbStopFlag) return;                                   // reference :359-361
    std::vector<uint8_t> outlier;
    if (W.run(pbStopFlag, 5, 10, outlier) != CSLAM_OK) b200_fatal();
    std::unique_lock<std::mutex> lock(pMap->mMutexMapUpdate);                // reference :419
    for (size_t e = 0; e < W.edgeOwner.size(); e++)
        if (outlier[e] && !W.edgeOwner[e].second->isBad()) { W.edgeOwner[e].first->EraseMapPointMatch(W.edgeOwner[e].second); W.edgeOwner[e].second->EraseObservation(W.edgeOwner[e].first); }
    std::map<KeyFrame*, int> kfIndex;
    for (size_t i = 0; i < W.kfList.size(); i++) kfIndex[W.kfList[i]] = (int)i;
    for (std::list<KeyFrame*>::iterator it = lLocalKeyFrames.begin(); it != lLocalKeyFrames.end(); ++it) (*it)->SetPose(mat44(&W.Tcw[16 * kfIndex[*it]]));
    for (size_t i = 0; i < W.mpList.size(); i++) {
        cv::Mat P(3, 1, CV_32F);
        for (int c = 0; c < 3; c++) P.at<float>(c) = W.pts[3 * i + c];
        W.mpList[i]->SetWorldPos(P); W.mpList[i]->UpdateNormalAndDepth();
    }
}

// reference src/Optimizer.cpp:453-459
void Optimizer::GlobalBundleAdjustemnt(Map* pMap, int nIterations, bool* pbStopFlag, const unsigned long nLoopKF, const bool bRobust) {
    std::vector<KeyFrame*> vpKFs = pMap->GetAllKeyFrames();
    std::vector<MapPoint*> vpMP = pMap->GetAllMapPoints();
    BundleAdjustment(vpKFs, vpMP, nIterations, pbStopFlag, nLoopKF, bRobust);
}

// reference src/Optimizer.cpp:461-621: all key frames / map points, one optimize(nIterations), no outlier stage. The same cubemap edge and
// solver as LocalBA: cslam_local_ba with its1 = nIterations, its2 = 0. (bRobust = false has no caller in the reference: LoopClosing.cpp:649 and
// Tracking.cpp:514 use the default; it is rejected rather than silently run with the kernel on.)
void Optimizer::BundleAdjustment(const std::vector<KeyFrame*>& vpKFs, const std::vector<MapPoint*>& vpMP, int nIterations, bool* pbStopFlag, const unsigned long nLoopKF, const bool bRobust) {
    if (!bRobust) { std::fprintf(stderr, "Optimizer::BundleAdjustment (cubemap_b200): bRobust=false is not supported\n"); std::exit(EXIT_FAILURE); }
    std::map<unsigned long, KeyFrame*> kfs; std::map<unsigned long, bool> fixedFlag; std::map<unsigned long, MapPoint*> mps;
    for (size_t i = 0; i < vpKFs.size(); i++) { KeyFrame* pKF = vpKFs[i]; if (pKF->isBad()) continue; kfs[pKF->mnId] = pKF; fixedFlag[pKF->mnId] = (pKF->mnId == 0); }
    for (size_t i = 0; i < vpMP.size(); i++) { MapPoint* pMP = vpMP[i]; if (pMP->isBad()) continue; mps[pMP->mnId] = pMP; }
    Window W; W.build(kfs, fixedFlag, mps);
    std::vector<uint8_t> outlier;
    if (W.run(pbStopFlag, nIterations, 0, outlier) != CSLAM_OK) b200_fatal();
    // write-back conventions of :584-618
    std::vector<int> nEdges(W.mpList.size(), 0);
    for (size_t e = 0; e < W.eMP.size(); e++) nEdges[W.eMP[e]]++;
    for (size_t i = 0; i < W.kfList.size(); i++) {
        KeyFrame* pKF = W.kfList[i];
        if (nLoopKF == 0) pKF->SetPose(mat44(&W.Tcw[16 * i]));
        else { pKF->mTcwGBA.create(4, 4, CV_32F); mat44(&W.Tcw[16 * i]).copyTo(pKF->mTcwGBA); pKF->mnBAGlobalForKF = nLoopKF; }
    }
    for (size_t i = 0; i < W.mpList.size(); i++) {
        if (nEdges[i] == 0) continue;                                        // vbNotIncludedMP
        MapPoint* pMP = W.mpList[i];
        cv::Mat P(3, 1, CV_32F);
        for (int c = 0; c < 3; c++) P.at<float>(c) = W.pts[3 * i + c];
        if (nLoopKF == 0) { pMP->SetWorldPos(P); pMP->UpdateNormalAndDepth(); }
        else { pMP->mPosGBA.create(3, 1, CV_32F); P.copyTo(pMP->mPosGBA); pMP->mnBAGlobalForKF = nLoopKF; }
    }
}

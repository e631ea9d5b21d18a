// Drop-in DEFINITIONS of the ORBMatcher searches that run on libcubemap_b200.so, compiled INSIDE the CubemapSLAM tree against the
// reference's own, unmodified include/ORBMatcher.h (:42-104). Everything else of the class (constructor, DescriptorDistance - the 8-word
// host popcount of src/ORBMatcher.cpp:951-967 -, ComputeThreeMaxima, the projection / epipolar / Sim3 / Fuse searches not listed here)
// stays the reference's src/ORBMatcher.cpp; the bodies replaced here are renamed away at compile time
// (INTEGRATION.md: COMPILE_DEFINITIONS "SearchByBoW=SearchByBoW_cpu;SearchByProjection=SearchByProjection_cpu" on that one file), no source edit.
#include "ORBMatcher.h"

#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>

#include "FeatureVector_csr_b200.h"
#include "cubemap_b200.h"

// the reference's own CPU bodies, exported by dropin/ORBMatcher_cpu_forward.cpp
int cslam_cpu_SearchByProjection(ORBMatcher* m, Frame& CurrentFrame, KeyFrame* pKF, const std::set<MapPoint*>& sAlreadyFound, const float th, const int ORBdist);
int cslam_cpu_SearchByProjection(ORBMatcher* m, KeyFrame* pKF, cv::Mat Scw, const std::vector<MapPoint*>& vpPoints, std::vector<MapPoint*>& vpMatched, int th);

namespace {
cslam_matcher* b200_matcher() {   // ORBMatcher objects live on three threads in the reference: one device handle per host thread
    static thread_local cslam_matcher* m = nullptr;
    if (!m && cslam_matcher_create(&m, 0, 1, 4096) != CSLAM_OK) { std::fprintf(stderr, "ORBMatcher (cubemap_b200): %s\n", cslam_last_error()); std::exit(EXIT_FAILURE); }
    return m;
}
void b200_fatal() { std::fprintf(stderr, "ORBMatcher (cubemap_b200): %s\n", cslam_last_error()); std::exit(EXIT_FAILURE); }
void gather(const cv::Mat& desc, const std::vector<cv::KeyPoint>& keys, int n, std::vector<uint8_t>& d, std::vector<float>& a) {
    d.resize((size_t)n * 32); a.resize(n);
    for (int i = 0; i < n; i++) { std::memcpy(&d[(size_t)i * 32], desc.ptr<uchar>(i), 32); a[i] = keys[i].angle; }
}
cslam_tracker* b200_tracker() {
    static thread_local cslam_tracker* t = nullptr;
    if (!t && cslam_tracker_create(&t, 0, 1, 4096) != CSLAM_OK) b200_fatal();
    return t;
}
}  // namespace

// the calling thread's tracker handle, shared with dropin/ORBMatcher_init_b200.cpp
cslam_tracker* cubemap_b200_thread_tracker() { return b200_tracker(); }

// reference src/ORBMatcher.cpp:130-251 (Tracking::TrackWithMotionModel :634, with the retry at twice the window :641). The reference walks
// LastFrame's MapPoints on the host; here their world positions / descriptors / observation flags are gathered and the projection, the
// cube-face window lookup (Frame::GetFeaturesInArea), the Hamming search and the rotation-consistency filter run on the device.
int ORBMatcher::SearchByProjection(Frame& CurrentFrame, const Frame& LastFrame, const float th, const bool bMono) {
    if (!bMono) { std::fprintf(stderr, "ORBMatcher (cubemap_b200): SearchByProjection(Frame, Frame) is monocular only (the reference's callers pass true)\n"); std::exit(EXIT_FAILURE); }
    CamModelGeneral* cam = CamModelGeneral::GetCamera();
    const int nC = CurrentFrame.N, nL = LastFrame.N;
    if (nC == 0 || nL == 0) return 0;
    std::vector<uint8_t> dC, dMP((size_t)nL * 32, 0), has(nL, 0), obs(nL, 0), taken(nC, 0); std::vector<float> aC, Xw((size_t)nL * 3, 0.f);
    gather(CurrentFrame.mDescriptors, CurrentFrame.mvKeys, nC, dC, aC);
    for (int i = 0; i < nL; i++) {
        MapPoint* pMP = LastFrame.mvpMapPoints[i];
        if (!pMP || LastFrame.mvbOutlier[i]) continue;
        has[i] = 1; obs[i] = pMP->Observations() > 0;
        const cv::Mat P = pMP->GetWorldPos(), d = pMP->GetDescriptor();
        for (int c = 0; c < 3; c++) Xw[3 * (size_t)i + c] = P.at<float>(c);
        std::memcpy(&dMP[(size_t)i * 32], d.ptr<uchar>(0), 32);
    }
    for (int i = 0; i < nC; i++) taken[i] = CurrentFrame.mvpMapPoints[i] && CurrentFrame.mvpMapPoints[i]->Observations() > 0;
    float T[16];
    for (int r = 0; r < 4; r++) for (int c = 0; c < 4; c++) T[4 * r + c] = CurrentFrame.mTcw.at<float>(r, c);
    std::vector<int32_t> match(nC); int32_t n = 0, nc = nC, nl = nL;
    static_assert(sizeof(cv::KeyPoint) == sizeof(cslam_keypoint), "cv::KeyPoint layout");
    if (cslam_search_by_projection_last(b200_tracker(), 1, reinterpret_cast<const cslam_keypoint*>(CurrentFrame.mvKeys.data()), dC.data(), &nc, nC, taken.data(), T,
                                        reinterpret_cast<const cslam_keypoint*>(LastFrame.mvKeys.data()), &nl, nL, has.data(), Xw.data(), dMP.data(), obs.data(),
                                        cam->GetCubeFaceWidth(), cam->GetCubeFaceHeight(), cam->GetCosFovTh(), th, mbCheckOrientation, CurrentFrame.mfScaleFactor,
                                        CurrentFrame.mnScaleLevels, match.data(), &n) != CSLAM_OK) b200_fatal();
    // write-back: slots the search assigned hold LastFrame's MapPoint; slots assigned and then cleared by the rotation filter (-2) become NULL;
    // untouched slots (-1) keep whatever pointer they held
    for (int i2 = 0; i2 < nC; i2++) {
        if (match[i2] >= 0) CurrentFrame.mvpMapPoints[i2] = LastFrame.mvpMapPoints[match[i2]];
        else if (match[i2] == -2) CurrentFrame.mvpMapPoints[i2] = static_cast<MapPoint*>(NULL);
    }
    return n;
}

// reference src/ORBMatcher.cpp:51-128 (Tracking::SearchLocalPoints :841): the MapPoints carry what Frame::isInFrustum stored in them
int ORBMatcher::SearchByProjection(Frame& F, const std::vector<MapPoint*>& vpMapPoints, const float th) {
    CamModelGeneral* cam = CamModelGeneral::GetCamera();
    const int nF = F.N, nM = (int)vpMapPoints.size();
    if (nF == 0 || nM == 0) return 0;
    if (nM > CSLAM_LOCAL_MAP_MAX_POINTS) {
        std::fprintf(stderr, "ORBMatcher (cubemap_b200): more than %d local MapPoints in one SearchByProjection call\n", CSLAM_LOCAL_MAP_MAX_POINTS); std::exit(EXIT_FAILURE);
    }
    std::vector<uint8_t> dF, dMP((size_t)nM * 32, 0), inView(nM, 0), obs(nM, 0), taken(nF, 0); std::vector<float> aF, proj((size_t)nM * 2, 0.f), vcos(nM, 0.f); std::vector<int32_t> lvl(nM, 0);
    gather(F.mDescriptors, F.mvKeys, nF, dF, aF);
    for (int m = 0; m < nM; m++) {
        MapPoint* pMP = vpMapPoints[m];
        if (!pMP->mbTrackInView || pMP->isBad()) continue;
        inView[m] = 1; obs[m] = pMP->Observations() > 0; lvl[m] = pMP->mnTrackScaleLevel; vcos[m] = pMP->mTrackViewCos;
        proj[2 * (size_t)m] = pMP->mTrackProjX; proj[2 * (size_t)m + 1] = pMP->mTrackProjY;
        const cv::Mat d = pMP->GetDescriptor();
        std::memcpy(&dMP[(size_t)m * 32], d.ptr<uchar>(0), 32);
    }
    for (int i = 0; i < nF; i++) taken[i] = F.mvpMapPoints[i] && F.mvpMapPoints[i]->Observations() > 0;
    std::vector<int32_t> match(nF); int32_t n = 0, nf = nF, nm = nM;
    // Every size goes to the _large entry (Tracking::UpdateLocalPoints takes every point of every local key frame, past 4096 as the map grows).
    // It is also the faster one below 4096: median host-call latency on an H100 80GB HBM3 (700 W), one frame of 4096 key points, face 650,
    // th 5, two runs of tools/local_map_latency.py: 0.82-0.85 ms against 1.77-1.79 ms for cslam_search_by_projection_local at 1024
    // MapPoints, 2.06-2.14 against 6.43-6.70 ms at 4096.
    if (cslam_search_by_projection_local_large(b200_tracker(), 1, reinterpret_cast<const cslam_keypoint*>(F.mvKeys.data()), dF.data(), &nf, nF, taken.data(), &nm, nM,
                                               inView.data(), proj.data(), lvl.data(), vcos.data(), dMP.data(), obs.data(), cam->GetCubeFaceWidth(),
                                               cam->GetCubeFaceHeight(), th, mfNNratio, F.mfScaleFactor, F.mnScaleLevels, match.data(), &n) != CSLAM_OK) b200_fatal();
    for (int i = 0; i < nF; i++) if (match[i] >= 0) F.mvpMapPoints[i] = vpMapPoints[match[i]];
    return n;
}

// the two overloads that stay on the reference's CPU code (src/ORBMatcher.cpp:253-378 relocalisation, :796-903 loop closing): the rename of
// `SearchByProjection` in src/ORBMatcher.cpp covers all four overloads, these two are forwarded straight back
int ORBMatcher::SearchByProjection(Frame& CurrentFrame, KeyFrame* pKF, const std::set<MapPoint*>& sAlreadyFound, const float th, const int ORBdist) {
    return cslam_cpu_SearchByProjection(this, CurrentFrame, pKF, sAlreadyFound, th, ORBdist);
}
int ORBMatcher::SearchByProjection(KeyFrame* pKF, cv::Mat Scw, const std::vector<MapPoint*>& vpPoints, std::vector<MapPoint*>& vpMatched, int th) {
    return cslam_cpu_SearchByProjection(this, pKF, Scw, vpPoints, vpMatched, th);
}

// reference src/ORBMatcher.cpp:409-539 (Tracking::TrackReferenceKeyFrame :577, Relocalization :1045). Both FeatureVectors go to the device as
// they are (cslam_search_by_bow_fv), so key frames of the initialisation extractor (up to 3*nFeatures + 3*nlevels key points) are taken too.
int ORBMatcher::SearchByBoW(KeyFrame* pKF, Frame& F, std::vector<MapPoint*>& vpMapPointMatches) {
    const std::vector<MapPoint*> vpMapPointsKF = pKF->GetMapPointMatches();
    const int32_t nKF = (int32_t)vpMapPointsKF.size(), nF = F.N;
    vpMapPointMatches = std::vector<MapPoint*>(nF, static_cast<MapPoint*>(NULL));
    if (nKF == 0 || nF == 0) return 0;
    std::vector<uint8_t> dK, dF, valid(nKF); std::vector<float> aK, aF;
    gather(pKF->mDescriptors, pKF->mvKeys, nKF, dK, aK); gather(F.mDescriptors, F.mvKeys, nF, dF, aF);
    for (int i = 0; i < nKF; i++) valid[i] = vpMapPointsKF[i] && !vpMapPointsKF[i]->isBad();
    const cubemap_b200::FeatureVectorCsr fK(pKF->mFeatVec, nKF), fF(F.mFeatVec, nF);
    std::vector<int32_t> matchF(nF); int32_t n = 0;
    if (cslam_search_by_bow_fv(b200_matcher(), 1, dK.data(), aK.data(), valid.data(), &nKF, nKF, fK.node.data(), fK.start.data(), fK.feat.data(), &fK.count, dF.data(),
                               aF.data(), &nF, nF, fF.node.data(), fF.start.data(), fF.feat.data(), &fF.count, mfNNratio, mbCheckOrientation, matchF.data(), &n) != CSLAM_OK)
        b200_fatal();
    for (int j = 0; j < nF; j++) if (matchF[j] >= 0) vpMapPointMatches[j] = vpMapPointsKF[matchF[j]];
    return n;
}

// reference src/ORBMatcher.cpp:541-674 (LoopClosing::ComputeSim3 :238), through cslam_search_by_bow_kf_fv likewise
int ORBMatcher::SearchByBoW(KeyFrame* pKF1, KeyFrame* pKF2, std::vector<MapPoint*>& vpMatches12) {
    const std::vector<MapPoint*> mp1 = pKF1->GetMapPointMatches(), mp2 = pKF2->GetMapPointMatches();
    const int32_t n1 = (int32_t)mp1.size(), n2 = (int32_t)mp2.size();
    vpMatches12 = std::vector<MapPoint*>(n1, static_cast<MapPoint*>(NULL));
    if (n1 == 0 || n2 == 0) return 0;
    std::vector<uint8_t> d1, d2, v1(n1), v2(n2); std::vector<float> a1, a2;
    gather(pKF1->mDescriptors, pKF1->mvKeys, n1, d1, a1); gather(pKF2->mDescriptors, pKF2->mvKeys, n2, d2, a2);
    for (int i = 0; i < n1; i++) v1[i] = mp1[i] && !mp1[i]->isBad();
    for (int i = 0; i < n2; i++) v2[i] = mp2[i] && !mp2[i]->isBad();
    const cubemap_b200::FeatureVectorCsr f1(pKF1->mFeatVec, n1), f2(pKF2->mFeatVec, n2);
    std::vector<int32_t> m12(n1); int32_t n = 0;
    if (cslam_search_by_bow_kf_fv(b200_matcher(), 1, d1.data(), a1.data(), v1.data(), &n1, n1, f1.node.data(), f1.start.data(), f1.feat.data(), &f1.count, d2.data(),
                                  a2.data(), v2.data(), &n2, n2, f2.node.data(), f2.start.data(), f2.feat.data(), &f2.count, mfNNratio, mbCheckOrientation, m12.data(),
                                  &n) != CSLAM_OK)
        b200_fatal();
    for (int i = 0; i < n1; i++) if (m12[i] >= 0) vpMatches12[i] = mp2[m12[i]];
    return n;
}

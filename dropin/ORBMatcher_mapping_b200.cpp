// Drop-in DEFINITIONS of the two ORBMatcher searches LocalMapping runs either side of LocalBA, on libcubemap_b200.so, compiled INSIDE the CubemapSLAM
// tree against the reference's own, unmodified include/ORBMatcher.h. The replaced bodies of src/ORBMatcher.cpp are renamed away at compile time
// (INTEGRATION.md: COMPILE_DEFINITIONS "...;Fuse=Fuse_cpu;SearchForTriangulation=SearchForTriangulation_cpu" on that one file), no source edit.
//   ORBMatcher::SearchForTriangulation  reference src/ORBMatcher.cpp:971-1124   (LocalMapping::CreateNewMapPoints, src/LocalMapping.cpp:262)
//   ORBMatcher::Fuse(pKF, vpMapPoints)  reference src/ORBMatcher.cpp:1126-1240  (LocalMapping::SearchInNeighbors, src/LocalMapping.cpp:390-425)
//   ORBMatcher::Fuse(pKF, Scw, ...)     loop closing with a Sim3: forwarded to the reference's own body (the rename cannot tell overloads apart)
#include "ORBMatcher.h"

#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>

#include "FeatureVector_csr_b200.h"
#include "cubemap_b200.h"

int cslam_cpu_Fuse(ORBMatcher* m, KeyFrame* pKF, cv::Mat Scw, const std::vector<MapPoint*>& vpPoints, float th, std::vector<MapPoint*>& vpReplacePoint);

namespace {
cslam_mapper* b200_mapper() {   // one device handle per host thread (LocalMapping and LoopClosing both own ORBMatcher objects)
    static thread_local cslam_mapper* m = nullptr;
    if (!m && cslam_mapper_create(&m, 0) != CSLAM_OK) { std::fprintf(stderr, "ORBMatcher (cubemap_b200): %s\n", cslam_last_error()); std::exit(EXIT_FAILURE); }
    return m;
}
void b200_fatal() { std::fprintf(stderr, "ORBMatcher (cubemap_b200): %s\n", cslam_last_error()); std::exit(EXIT_FAILURE); }
void gather_desc(const cv::Mat& desc, int n, std::vector<uint8_t>& d) {
    d.resize((size_t)n * 32);
    for (int i = 0; i < n; i++) std::memcpy(&d[(size_t)i * 32], desc.ptr<uchar>(i), 32);
}
}  // namespace

int ORBMatcher::Fuse(KeyFrame* pKF, cv::Mat Scw, const std::vector<MapPoint*>& vpPoints, float th, std::vector<MapPoint*>& vpReplacePoint) {
    return cslam_cpu_Fuse(this, pKF, Scw, vpPoints, th, vpReplacePoint);
}

int ORBMatcher::Fuse(KeyFrame* pKF, const std::vector<MapPoint*>& vpMapPoints, const float th) {
    CamModelGeneral* cam = CamModelGeneral::GetCamera();
    cv::Mat Ow = pKF->GetCameraCenter();
    const int nMPs = (int)vpMapPoints.size(), nKF = pKF->N;
    if (nMPs == 0) return 0;
    // (1) what the reference tests before its search (src/ORBMatcher.cpp:1141-1178), with the reference's own accessors. None of it can be changed
    //     by a fusion made earlier in the list except isBad / IsInKeyFrame, which are looked at again in (3).
    std::vector<uint8_t> valid(nMPs, 0), dMP((size_t)nMPs * 32, 0); std::vector<float> Xw((size_t)nMPs * 3, 0.f); std::vector<int32_t> level(nMPs, 0);
    for (int i = 0; i < nMPs; i++) {
        MapPoint* pMP = vpMapPoints[i];
        if (!pMP) continue;
        if (pMP->isBad() || pMP->IsInKeyFrame(pKF)) continue;
        cv::Mat p3Dw = pMP->GetWorldPos();
        const float maxDistance = pMP->GetMaxDistanceInvariance();
        const float minDistance = pMP->GetMinDistanceInvariance();
        cv::Mat PO = p3Dw - Ow;
        const float dist3D = cv::norm(PO);
        if (dist3D < minDistance || dist3D > maxDistance) continue;
        cv::Mat Pn = pMP->GetNormal();
        if (PO.dot(Pn) < 0.5 * dist3D) continue;
        valid[i] = 1; level[i] = pMP->PredictScale(dist3D, pKF);
        for (int c = 0; c < 3; c++) Xw[3 * (size_t)i + c] = p3Dw.at<float>(c);
        const cv::Mat d = pMP->GetDescriptor();
        std::memcpy(&dMP[(size_t)i * 32], d.ptr<uchar>(0), 32);
    }
    // (2) projection, window lookup, Hamming on the device
    std::vector<uint8_t> dKF; gather_desc(pKF->mDescriptors, nKF, dKF);
    const cv::Mat Tcw = pKF->GetPose();
    float T[16];
    for (int r = 0; r < 4; r++) for (int c = 0; c < 4; c++) T[4 * r + c] = Tcw.at<float>(r, c);
    std::vector<int32_t> bestIdx(nMPs), bestDist(nMPs);
    static_assert(sizeof(cv::KeyPoint) == sizeof(cslam_keypoint), "cv::KeyPoint layout");
    if (cslam_fuse_search_large(b200_mapper(), reinterpret_cast<const cslam_keypoint*>(pKF->mvKeys.data()), dKF.data(), nKF, T, nMPs, valid.data(), Xw.data(), level.data(), dMP.data(), th,
                                pKF->mvScaleFactors.data(), pKF->mvInvLevelSigma2.data(), pKF->mnScaleLevels, cam->GetCubeFaceWidth(), cam->GetCubeFaceHeight(),
                                bestIdx.data(), bestDist.data()) != CSLAM_OK) b200_fatal();
    // (3) the order-dependent bookkeeping, verbatim in effect (src/ORBMatcher.cpp:1217-1236)
    int nFused = 0;
    for (int i = 0; i < nMPs; i++) {
        MapPoint* pMP = vpMapPoints[i];
        if (!pMP || !valid[i]) continue;
        if (pMP->isBad() || pMP->IsInKeyFrame(pKF)) continue;
        if (bestDist[i] <= TH_LOW) {
            MapPoint* pMPinKF = pKF->GetMapPoint(bestIdx[i]);
            if (pMPinKF) {
                if (!pMPinKF->isBad()) {
                    if (pMPinKF->Observations() > pMP->Observations()) pMP->Replace(pMPinKF);
                    else pMPinKF->Replace(pMP);
                }
            } else {
                pMP->AddObservation(pKF, bestIdx[i]);
                pKF->AddMapPoint(pMP, bestIdx[i]);
            }
            nFused++;
        }
    }
    return nFused;
}

int ORBMatcher::SearchForTriangulation(KeyFrame* pKF1, KeyFrame* pKF2, cv::Mat E12, std::vector<std::pair<size_t, size_t> >& vMatchedPairs) {
    CamModelGeneral* cam = CamModelGeneral::GetCamera();
    const int32_t n1 = pKF1->N, n2 = pKF2->N;
    vMatchedPairs.clear();
    if (n1 == 0 || n2 == 0) return 0;
    std::vector<uint8_t> d1, d2, has1(n1, 0), has2(n2, 0); std::vector<float> r1((size_t)n1 * 3), r2((size_t)n2 * 3);
    gather_desc(pKF1->mDescriptors, n1, d1); gather_desc(pKF2->mDescriptors, n2, d2);
    const cubemap_b200::FeatureVectorCsr f1(pKF1->mFeatVec, n1), f2(pKF2->mFeatVec, n2);
    for (int i = 0; i < n1; i++) { has1[i] = pKF1->GetMapPoint(i) != NULL; for (int c = 0; c < 3; c++) r1[3 * (size_t)i + c] = pKF1->mvKeyRays[i](c); }
    for (int i = 0; i < n2; i++) { has2[i] = pKF2->GetMapPoint(i) != NULL; for (int c = 0; c < 3; c++) r2[3 * (size_t)i + c] = pKF2->mvKeyRays[i](c); }
    const cv::Mat Cw = pKF1->GetCameraCenter(), T2 = pKF2->GetPose();
    float Ow1[3], Tcw2[16], E[9];
    for (int c = 0; c < 3; c++) Ow1[c] = Cw.at<float>(c);
    for (int r = 0; r < 4; r++) for (int c = 0; c < 4; c++) Tcw2[4 * r + c] = T2.at<float>(r, c);
    for (int r = 0; r < 3; r++) for (int c = 0; c < 3; c++) E[3 * r + c] = E12.at<float>(r, c);
    std::vector<int32_t> match(n1); int32_t nm = 0;
    if (cslam_search_for_triangulation_fv(b200_mapper(), 1, reinterpret_cast<const cslam_keypoint*>(pKF1->mvKeys.data()), d1.data(), r1.data(), has1.data(), &n1, n1,
                                          f1.node.data(), f1.start.data(), f1.feat.data(), &f1.count, reinterpret_cast<const cslam_keypoint*>(pKF2->mvKeys.data()),
                                          d2.data(), r2.data(), has2.data(), &n2, n2, f2.node.data(), f2.start.data(), f2.feat.data(), &f2.count, Ow1, Tcw2, E,
                                          pKF2->mvScaleFactors.data(), pKF2->mvLevelSigma2.data(), pKF2->mnScaleLevels, cam->GetCubeFaceWidth(),
                                          cam->GetCubeFaceHeight(), mbCheckOrientation, match.data(), &nm) != CSLAM_OK) b200_fatal();
    vMatchedPairs.reserve(nm);
    for (int i = 0; i < n1; i++) if (match[i] >= 0) vMatchedPairs.push_back(std::make_pair((size_t)i, (size_t)match[i]));
    return nm;
}

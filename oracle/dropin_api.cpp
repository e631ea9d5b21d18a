// ORACLE / TEST HARNESS (not product code): links the drop-in definitions of dropin/*.cpp (the product's reference-facing boundary) with
// the reference's OWN data-model classes - Frame, KeyFrame, MapPoint, Map, KeyFrameDatabase, CamModelGeneral, DBoW2, compiled unmodified from
// /root/reference against the cv:: shim - into oracle/_ref/libdropin.so, and exposes flat C entry points for tests/test_gpu_dropin.py.
// It proves on the GPU box what INTEGRATION.md claims: the reference's call sites
//     Frame::Frame -> ExtractORB -> (*mpORBextractor)(im, mask, mvKeys, mDescriptors)      src/Frame.cpp:104-156,178-181
//     ORBMatcher(0.7,true).SearchByBoW(pKF, F, vpMapPointMatches)                          src/Tracking.cpp:574-577
//     Optimizer::PoseOptimization(&mCurrentFrame)                                          src/Tracking.cpp:585,647,688
//     Optimizer::LocalBundleAdjustment(mpCurrentKeyFrame, &mbAbortBA, mpMap)               src/LocalMapping.cpp:86
// run unchanged against libcubemap_b200.so. The reference's own src/ORBMatcher.cpp is linked too, with the replaced method renamed
// (-DSearchByBoW=SearchByBoW_cpu -DSearchByProjection=SearchByProjection_cpu, see oracle/Makefile) so the same objects can be matched by the reference's CPU code for comparison.
// The objects come from oracle/ref_scene.cpp, which libref.so shares: the drop-in is checked on the scenes the CPU reference tests check.
#include <algorithm>
#include <cstring>
#include <map>
#include <vector>

#include "KeyFrameDatabase.h"
#include "ORBExtractor.h"
#include "ORBMatcher.h"
#include "Optimizer.h"
#include "ref_scene.h"

using namespace scene;

// the out-of-scope optimisations declared by include/Optimizer.h are never called by the harness
// (src/Optimizer.cpp needs g2o / Eigen and is not part of this library)

// the reference's own CPU bodies on the same objects (dropin/ORBMatcher_cpu_forward.cpp)
int cslam_cpu_SearchByBoW(ORBMatcher* m, KeyFrame* pKF, Frame& F, std::vector<MapPoint*>& vpMapPointMatches);
int cslam_cpu_SearchByProjection(ORBMatcher* m, Frame& CurrentFrame, const Frame& LastFrame, const float th, const bool bMono);
int cslam_cpu_SearchByProjection(ORBMatcher* m, Frame& F, const std::vector<MapPoint*>& vpMapPoints, const float th);
int cslam_cpu_Fuse(ORBMatcher* m, KeyFrame* pKF, const std::vector<MapPoint*>& vpMapPoints, const float th);
int cslam_cpu_SearchForTriangulation(ORBMatcher* m, KeyFrame* pKF1, KeyFrame* pKF2, cv::Mat E12, std::vector<std::pair<size_t, size_t> >& vMatchedPairs);
namespace cubemap_b200 { void DistinctiveDescriptors(const std::vector<MapPoint*>& vpMPs, std::vector<cv::Mat>& out); }

namespace {
void fill_featvec(DBoW2::FeatureVector& fv, const int32_t* node, int n) { for (int i = 0; i < n; i++) if (node[i] >= 0) fv.addFeature((DBoW2::NodeId)node[i], (unsigned)i); }

// A Map built through the reference's own API (KeyFrame / MapPoint / Map, AddObservation, AddMapPoint) from nE edges (MapPoint eMP[e] seen by key
// frame eKF[e] at kpxy[e] with octave[e]); key frame k has pose Tcw[16k], MapPoint l position pts[3l], and both are numbered from 0 (mnId).
struct BAMap {
    Map map; KFArray kfs; std::vector<MapPoint*> mps;
    BAMap(int nKF, int nMP, int nE, const float* Tcw, const float* pts, const int32_t* eMP, const int32_t* eKF, const float* kpxy, const int32_t* octave)
        : kfs(nKF), mps(nMP, static_cast<MapPoint*>(NULL)) {
        KeyFrame::nNextId = 0; MapPoint::nNextId = 0;
        std::vector<std::vector<int> > edgesOfKF(nKF);
        for (int e = 0; e < nE; e++) edgesOfKF[eKF[e]].push_back(e);
        std::vector<int> slot(nE);
        for (int k = 0; k < nKF; k++) {
            const int n = (int)edgesOfKF[k].size();
            std::vector<KpPOD> kps(n);
            for (int i = 0; i < n; i++) { const int e = edgesOfKF[k][i]; slot[e] = i; kps[i] = KpPOD{kpxy[2 * e], kpxy[2 * e + 1], 31, 0, 0, octave[e], -1}; }
            Frame* F = make_frame(n, kps.data(), NULL, Tcw + 16 * k);
            map.AddKeyFrame(kfs.make(k, *F, &map));
            delete F;
        }
        for (int e = 0; e < nE; e++) {
            const int l = eMP[e];
            if (!mps[l]) { mps[l] = new MapPoint(mat_from(pts + 3 * l, 3, 1), kfs.kf[eKF[e]], &map); map.AddMapPoint(mps[l]); }
        }
        for (int l = 0; l < nMP; l++) if (!mps[l]) mps[l] = new MapPoint(mat_from(pts + 3 * l, 3, 1), kfs.kf[0], &map);   // unobserved point (keeps mnId == l)
        for (int e = 0; e < nE; e++) { mps[eMP[e]]->AddObservation(kfs.kf[eKF[e]], slot[e]); kfs.kf[eKF[e]]->AddMapPoint(mps[eMP[e]], slot[e]); }
    }
    ~BAMap() { for (MapPoint* mp : mps) delete mp; }
    // KeyFrame::GetPose / MapPoint::GetWorldPos of every key frame and point
    void read(float* Tcw, float* pts) const {
        for (size_t k = 0; k < kfs.kf.size(); k++) { const cv::Mat T = kfs.kf[k]->GetPose(); for (int r = 0; r < 4; r++) for (int c = 0; c < 4; c++) Tcw[16 * k + 4 * r + c] = T.at<float>(r, c); }
        for (size_t l = 0; l < mps.size(); l++) { const cv::Mat P = mps[l]->GetWorldPos(); for (int c = 0; c < 3; c++) pts[3 * l + c] = P.at<float>(c); }
    }
};
}  // namespace

extern "C" {

void dropin_set_camera(const RefCam* cp) { set_camera(cp); }

// Frame::Frame(imGray, mask, timeStamp, extractor, voc) with the GPU drop-in ORBextractor: extraction, rays, grid. Returns N.
// kps: cap x 28 B, desc: cap x 32, rays: cap x 3, gridCount: 5*50*50 (mGrid[face][col][row].size())
int dropin_frame_from_image(const uint8_t* img, const uint8_t* mask, int rows, int cols, int nfeatures, float scaleFactor, int nlevels, int iniTh, int minTh, int cap,
                            KpPOD* kps, uint8_t* desc, float* rays, int32_t* gridCount) {
    static std::map<std::vector<int>, ORBextractor*> extractors;   // long-lived like Tracking's mpORBextractor (src/Tracking.cpp:95-96)
    const std::vector<int> key = {nfeatures, (int)(scaleFactor * 1000), nlevels, iniTh, minTh, rows, cols};
    ORBextractor*& ex = extractors[key];
    if (!ex) ex = new ORBextractor(nfeatures, scaleFactor, nlevels, iniTh, minTh);
    cv::Mat im(rows, cols, CV_8UC1, (void*)img), mk(rows, cols, CV_8UC1, (void*)mask);
    Frame::mbInitialComputations = true;
    Frame F(im, mk, 0.0, ex, static_cast<ORBVocabulary*>(NULL));
    read_frame(F, std::min(F.N, cap), kps, desc, rays, gridCount);
    return F.N;
}

// ORBMatcher(nnratio, checkOri).SearchByBoW(pKF, F, vpMapPointMatches) on reference objects: GPU drop-in and the reference's own CPU body.
// valid[i]: the KF feature has a (good) MapPoint. matchGpu / matchCpu: per F feature the index of the KF feature whose MapPoint was assigned, or -1.
void dropin_search_by_bow(int nKF, const KpPOD* kpK, const uint8_t* descK, const uint8_t* valid, const int32_t* nodeK, int nF, const KpPOD* kpF, const uint8_t* descF,
                          const int32_t* nodeF, float nnratio, int checkOri, int32_t* matchGpu, int32_t* nGpu, int32_t* matchCpu, int32_t* nCpu) {
    Map map; KeyFrameDatabase* db = NULL;
    Frame* FK = make_frame(nKF, kpK, descK, I4);
    fill_featvec(FK->mFeatVec, nodeK, nKF);
    KeyFrame* pKF = new KeyFrame(*FK, &map, db);
    std::map<MapPoint*, int> idxOf;
    for (int i = 0; i < nKF; i++) if (valid[i]) { MapPoint* mp = new MapPoint(mat_from(P0, 3, 1), pKF, &map); pKF->AddMapPoint(mp, i); idxOf[mp] = i; }
    Frame* F = make_frame(nF, kpF, descF, I4);
    fill_featvec(F->mFeatVec, nodeF, nF);
    std::vector<MapPoint*> out;
    ORBMatcher matcher(nnratio, checkOri != 0);
    *nGpu = matcher.SearchByBoW(pKF, *F, out);                              // dropin/ORBMatcher_b200.cpp -> libcubemap_b200.so
    for (int j = 0; j < nF; j++) matchGpu[j] = out[j] ? idxOf[out[j]] : -1;
    *nCpu = cslam_cpu_SearchByBoW(&matcher, pKF, *F, out);                  // the reference's src/ORBMatcher.cpp:409-539
    for (int j = 0; j < nF; j++) matchCpu[j] = out[j] ? idxOf[out[j]] : -1;
    for (std::map<MapPoint*, int>::iterator it = idxOf.begin(); it != idxOf.end(); ++it) delete it->first;
    delete pKF; delete FK; delete F;
}

// ORBMatcher(0.9, checkOri).SearchByProjection(CurrentFrame, LastFrame, th, true) (src/Tracking.cpp:634) on ProjectionLastScene: GPU drop-in and
// the reference's CPU body from identical starting states (the search only writes CurrentFrame.mvpMapPoints, which is restored in between).
void dropin_search_by_projection_last(int nCur, const KpPOD* kCur, const uint8_t* dCur, const float* TcwCur, int nLast, const KpPOD* kLast, const float* TcwLast,
                                      const uint8_t* hasMP, const float* Xw, const uint8_t* dMP, const int32_t* mpObs, const uint8_t* curTaken, float th, int checkOri,
                                      int32_t* matchGpu, int32_t* nGpu, int32_t* matchCpu, int32_t* nCpu) {
    ProjectionLastScene s(nCur, kCur, dCur, TcwCur, nLast, kLast, TcwLast, hasMP, Xw, dMP, mpObs, curTaken);
    const std::vector<MapPoint*> pre = s.cur->mvpMapPoints;
    ORBMatcher matcher(0.9f, checkOri != 0);
    *nGpu = matcher.SearchByProjection(*s.cur, *s.last, th, true);                         // dropin/ORBMatcher_b200.cpp -> libcubemap_b200.so
    s.read(matchGpu);
    s.cur->mvpMapPoints = pre;
    *nCpu = cslam_cpu_SearchByProjection(&matcher, *s.cur, *s.last, th, true);             // src/ORBMatcher.cpp:130-251
    s.read(matchCpu);
}

// Optimizer::PoseOptimization(&frame): n correspondences (keypoint, octave, world point). Returns inliers; Tcw in/out; outlier[n] = mvbOutlier.
int dropin_pose_optimization(int n, const float* kpxy, const int32_t* octave, const float* Xw, float* Tcw, uint8_t* outlier) {
    Map map;
    std::vector<KpPOD> kps(n);
    for (int i = 0; i < n; i++) kps[i] = KpPOD{kpxy[2 * i], kpxy[2 * i + 1], 31, 0, 0, octave[i], -1};
    Frame* F = make_frame(n, kps.data(), NULL, Tcw);
    std::vector<MapPoint*> mps(n);
    for (int i = 0; i < n; i++) { mps[i] = new MapPoint(mat_from(Xw + 3 * i, 3, 1), &map, F, i); F->mvpMapPoints[i] = mps[i]; }
    const int inl = Optimizer::PoseOptimization(F);                          // dropin/Optimizer_b200.cpp
    for (int i = 0; i < n; i++) outlier[i] = F->mvbOutlier[i] ? 1 : 0;
    for (int r = 0; r < 4; r++) for (int c = 0; c < 4; c++) Tcw[4 * r + c] = F->mTcw.at<float>(r, c);
    for (int i = 0; i < n; i++) delete mps[i];
    delete F;
    return inl;
}

// Optimizer::LocalBundleAdjustment(pKF, &stop, &map) on a BAMap whose key frames ran UpdateConnections. On return Tcw / pts hold KeyFrame::GetPose /
// MapPoint::GetWorldPos and erased[e] = 1 where the observation was erased. Returns the number of key frames in the local window (covisible with
// curKF, incl. itself).
int dropin_local_ba(int nKF, int nMP, int nE, float* Tcw, float* pts, const int32_t* eMP, const int32_t* eKF, const float* kpxy, const int32_t* octave, int curKF,
                    uint8_t* erased) {
    BAMap m(nKF, nMP, nE, Tcw, pts, eMP, eKF, kpxy, octave);
    for (int k = 0; k < nKF; k++) m.kfs.kf[k]->UpdateConnections();
    bool stop = false;
    const int window = (int)m.kfs.kf[curKF]->GetVectorCovisibleKeyFrames().size() + 1;
    Optimizer::LocalBundleAdjustment(m.kfs.kf[curKF], &stop, &m.map);       // dropin/Optimizer_b200.cpp
    m.read(Tcw, pts);
    for (int e = 0; e < nE; e++) erased[e] = m.mps[eMP[e]]->IsInKeyFrame(m.kfs.kf[eKF[e]]) ? 0 : 1;
    return window;
}

// Optimizer::GlobalBundleAdjustemnt(pMap, nIterations, NULL, 0, true) (src/Tracking.cpp:514 after map initialisation, src/LoopClosing.cpp:649) on a
// BAMap: all key frames / MapPoints, one optimize(nIterations), poses / points written back through SetPose / SetWorldPos.
void dropin_global_ba(int nKF, int nMP, int nE, float* Tcw, float* pts, const int32_t* eMP, const int32_t* eKF, const float* kpxy, const int32_t* octave, int nIterations) {
    BAMap m(nKF, nMP, nE, Tcw, pts, eMP, eKF, kpxy, octave);
    Optimizer::GlobalBundleAdjustemnt(&m.map, nIterations, NULL, 0, true);  // dropin/Optimizer_b200.cpp
    m.read(Tcw, pts);
}

// ORBMatcher(0.6).Fuse(pKF, vpMapPoints, th) (LocalMapping::SearchInNeighbors): the GPU drop-in and the reference's own CPU body, each on a fresh
// FuseScene. idx*[m] = FuseScene::index_in_kf afterwards; bad*[m] = isBad(). nFused by return values.
void dropin_fuse(int nKF, const KpPOD* kKF, const uint8_t* dKF, const float* Tcw, int nMP, const float* Xw, const KpPOD* kObs, const uint8_t* dMP, const float* TcwObs, float th,
                 int32_t* idxGpu, uint8_t* badGpu, int32_t* nGpu, int32_t* idxCpu, uint8_t* badCpu, int32_t* nCpu) {
    for (int pass = 0; pass < 2; pass++) {
        FuseScene s(nKF, kKF, dKF, Tcw, nMP, Xw, kObs, dMP, TcwObs);
        ORBMatcher matcher(0.6f, true);
        const int n = pass == 0 ? matcher.Fuse(s.pKF, s.mps, th)                 // dropin/ORBMatcher_mapping_b200.cpp -> libcubemap_b200.so
                                : cslam_cpu_Fuse(&matcher, s.pKF, s.mps, th);    // src/ORBMatcher.cpp:1126-1240
        (pass == 0 ? *nGpu : *nCpu) = n;
        int32_t* idx = pass == 0 ? idxGpu : idxCpu; uint8_t* bad = pass == 0 ? badGpu : badCpu;
        for (int m = 0; m < nMP; m++) { bad[m] = s.mps[m]->isBad(); idx[m] = s.index_in_kf(m); }
    }
}

// ORBMatcher(0.6, checkOri).SearchForTriangulation(pKF1, pKF2, E12, pairs) (LocalMapping::CreateNewMapPoints) on TriangulationScene: GPU drop-in vs
// the reference's CPU body
void dropin_search_for_triangulation(int n1, const KpPOD* k1, const uint8_t* d1, const float* Tcw1, const uint8_t* hasMP1, const int32_t* node1, int n2, const KpPOD* k2,
                                     const uint8_t* d2, const float* Tcw2, const uint8_t* hasMP2, const int32_t* node2, const float* E12, int checkOri, int32_t* matchGpu,
                                     int32_t* nGpu, int32_t* matchCpu, int32_t* nCpu) {
    TriangulationScene s(n1, k1, d1, Tcw1, hasMP1, node1, n2, k2, d2, Tcw2, hasMP2, node2);
    for (int pass = 0; pass < 2; pass++) {
        ORBMatcher matcher(0.6f, checkOri != 0);
        std::vector<std::pair<size_t, size_t> > pairs;
        const int n = pass == 0 ? matcher.SearchForTriangulation(s.kf1, s.kf2, mat_from(E12, 3, 3), pairs)                  // dropin/ORBMatcher_mapping_b200.cpp
                                : cslam_cpu_SearchForTriangulation(&matcher, s.kf1, s.kf2, mat_from(E12, 3, 3), pairs);    // src/ORBMatcher.cpp:971-1124
        (pass == 0 ? *nGpu : *nCpu) = n;
        s.read(pairs, pass == 0 ? matchGpu : matchCpu);
    }
}

// cubemap_b200::DistinctiveDescriptors (the batched form of MapPoint::ComputeDistinctiveDescriptors) vs the member itself, on DistinctiveScene.
// equal[p] = the batched descriptor is byte-identical to mDescriptor after the member ran.
void dropin_distinctive_batch(int nPoints, const int32_t* offset, const uint8_t* desc, uint8_t* equal) {
    DistinctiveScene s(nPoints, offset, desc);
    std::vector<cv::Mat> batched;
    cubemap_b200::DistinctiveDescriptors(s.mps, batched);                      // dropin/MapPoint_batch_b200.cpp -> libcubemap_b200.so
    for (int p = 0; p < nPoints; p++) {
        s.mps[p]->ComputeDistinctiveDescriptors();                             // src/MapPoint.cpp:243-303
        const cv::Mat d = s.mps[p]->GetDescriptor();
        if (offset[p + 1] == offset[p]) equal[p] = batched[p].empty();
        else equal[p] = !batched[p].empty() && std::memcmp(batched[p].ptr<uchar>(0), d.ptr<uchar>(0), 32) == 0;
    }
}

}  // extern "C"

// ORACLE (test infrastructure, not product code): see ref_scene.h.
#include "ref_scene.h"

#include <algorithm>
#include <cstdlib>
#include <cstring>
#include <iostream>
#include <new>

#include "Converter.h"

// src/Converter.cpp:29-39 (Converter.cpp itself needs Eigen / g2o): one Mat per descriptor row
std::vector<cv::Mat> Converter::toDescriptorVector(const cv::Mat& Descriptors) {
    std::vector<cv::Mat> vDesc;
    vDesc.reserve(Descriptors.rows);
    for (int j = 0; j < Descriptors.rows; j++) vDesc.push_back(Descriptors.row(j));
    return vDesc;
}

namespace scene {

cv::Mat mat_from(const float* T, int r, int c) { cv::Mat m(r, c, CV_32F); for (int i = 0; i < r * c; i++) m.at<float>(i / c, i % c) = T[i]; return m; }

void set_camera(const RefCam* cp) {
    cv::Mat_<double> poly = cv::Mat::zeros(5, 1, CV_64F), invpoly = cv::Mat::zeros(12, 1, CV_64F);
    for (int i = 0; i < 5; ++i) poly.at<double>(i, 0) = cp->p[i];
    for (int i = 0; i < 12; ++i) invpoly.at<double>(i, 0) = cp->invp[i];
    double cdeu0v0[5] = {cp->c, cp->d, cp->e, cp->u0, cp->v0};
    const double fx = static_cast<double>(cp->faceW) / 2, fy = static_cast<double>(cp->faceH) / 2;
    std::streambuf* old = std::cout.rdbuf(nullptr);   // SetCosFovTh prints two lines
    CamModelGeneral::GetCamera()->SetCamParams(cdeu0v0, poly, invpoly, cp->Iw, cp->Ih, fx, fy, fx, fy, cp->faceW, cp->faceH, cp->fov);
    std::cout.rdbuf(old);
}

Frame* make_frame(int n, const KpPOD* kps, const uint8_t* desc, const float* Tcw) {
    const int nlevels = 8; const float scaleFactor = 1.2f;
    Frame* F = new Frame();
    F->mnId = Frame::nNextId++;
    F->N = n;
    F->mvKeys.resize(n);
    if (n) std::memcpy((void*)F->mvKeys.data(), kps, (size_t)n * sizeof(KpPOD));
    F->mDescriptors = cv::Mat(n, 32, CV_8UC1);
    if (desc) for (int i = 0; i < n; i++) std::memcpy(F->mDescriptors.ptr<uchar>(i), desc + 32 * (size_t)i, 32); else F->mDescriptors.setTo(0);
    F->mvKeyRays.resize(n);
    for (int i = 0; i < n; i++) CamModelGeneral::GetCamera()->TransformCubemapToRays(F->mvKeyRays[i], F->mvKeys[i].pt);   // Frame::ComputeKeyPointRays
    F->mvpMapPoints.assign(n, static_cast<MapPoint*>(NULL));
    F->mvbOutlier.assign(n, false);
    F->mnScaleLevels = nlevels; F->mfScaleFactor = scaleFactor; F->mfLogScaleFactor = log(scaleFactor);
    F->mvScaleFactors.resize(nlevels); F->mvLevelSigma2.resize(nlevels); F->mvInvScaleFactors.resize(nlevels); F->mvInvLevelSigma2.resize(nlevels);
    F->mvScaleFactors[0] = 1.0f; F->mvLevelSigma2[0] = 1.0f;
    for (int i = 1; i < nlevels; i++) { F->mvScaleFactors[i] = F->mvScaleFactors[i - 1] * scaleFactor; F->mvLevelSigma2[i] = F->mvScaleFactors[i] * F->mvScaleFactors[i]; }
    for (int i = 0; i < nlevels; i++) { F->mvInvScaleFactors[i] = 1.0f / F->mvScaleFactors[i]; F->mvInvLevelSigma2[i] = 1.0f / F->mvLevelSigma2[i]; }
    if (Tcw) F->SetPose(mat_from(Tcw, 4, 4));
    // Frame::AssignFeaturesToGrid is private: replay it (src/Frame.cpp:158-176) with the public PosInGrid
    const int W3 = 3 * CamModelGeneral::GetCamera()->GetCubeFaceWidth();
    Frame::mnMinX = 0.0f; Frame::mnMaxX = (float)W3; Frame::mnMinY = 0.0f; Frame::mnMaxY = (float)(3 * CamModelGeneral::GetCamera()->GetCubeFaceHeight());
    Frame::mfGridElementLengthInv = static_cast<float>(3 * CUBEFACE_GRID_COLS) / static_cast<float>(Frame::mnMaxX - Frame::mnMinX);
    Frame::mfGridElementLength = static_cast<float>(Frame::mnMaxX - Frame::mnMinX) / static_cast<float>(3 * CUBEFACE_GRID_COLS);
    for (int i = 0; i < n; i++) {
        CamModelGeneral::eFace face; int gx, gy;
        if (F->PosInGrid(F->mvKeys[i], face, gx, gy)) F->mGrid[face][gx][gy].push_back(i);
    }
    return F;
}

void read_frame(const Frame& F, int n, KpPOD* kps, uint8_t* desc, float* rays, int32_t* gridCount) {
    if (n && kps) std::memcpy((void*)kps, F.mvKeys.data(), (size_t)n * sizeof(KpPOD));
    for (int i = 0; i < n; i++) {
        if (desc) std::memcpy(desc + 32 * (size_t)i, F.mDescriptors.ptr<uchar>(i), 32);
        if (rays) for (int c = 0; c < 3; c++) rays[3 * i + c] = F.mvKeyRays[i](c);
    }
    if (gridCount)
        for (int f = 0; f < CUBEMAP_FACES; f++) for (int x = 0; x < CUBEFACE_GRID_COLS; x++) for (int y = 0; y < CUBEFACE_GRID_ROWS; y++)
            gridCount[(f * CUBEFACE_GRID_COLS + x) * CUBEFACE_GRID_ROWS + y] = (int)F.mGrid[f][x][y].size();
}

KFArray::KFArray(int n) : buf((char*)std::malloc((size_t)n * sizeof(KeyFrame) + 64)), kf(n, static_cast<KeyFrame*>(NULL)) {}
KFArray::~KFArray() { for (KeyFrame* k : kf) if (k) k->~KeyFrame(); std::free(buf); }
KeyFrame* KFArray::make(int i, Frame& F, Map* map) { kf[i] = new (buf + (size_t)i * sizeof(KeyFrame)) KeyFrame(F, map, NULL); return kf[i]; }

// key frame i of A from a Frame that only lives for the KeyFrame constructor
static KeyFrame* make_kf(KFArray& A, int i, Map* map, int n, const KpPOD* kps, const uint8_t* desc, const float* Tcw) {
    Frame* F = make_frame(n, kps, desc, Tcw);
    KeyFrame* kf = A.make(i, *F, map);
    delete F;
    return kf;
}

ProjectionLastScene::ProjectionLastScene(int nCur, const KpPOD* kCur, const uint8_t* dCur, const float* TcwCur, int nLast, const KpPOD* kLast,
                                         const float* TcwLast, const uint8_t* hasMP, const float* Xw, const uint8_t* dMP, const int32_t* mpObs,
                                         const uint8_t* curTaken)
    : kfs(1), cur(make_frame(nCur, kCur, dCur, TcwCur)), last(make_frame(nLast, kLast, dMP, TcwLast)) {
    KeyFrame* kfObs = kfs.make(0, *last, &map);
    for (int i = 0; i < nLast; i++) {
        if (!hasMP[i]) continue;
        MapPoint* mp = new MapPoint(mat_from(Xw + 3 * i, 3, 1), &map, last, i);
        if (mpObs[i] > 0) mp->AddObservation(kfObs, i);
        last->mvpMapPoints[i] = mp; idxOf[mp] = i; owned.push_back(mp);
    }
    for (int i2 = 0; i2 < nCur; i2++) {
        if (!curTaken[i2]) continue;
        MapPoint* mp = new MapPoint(mat_from(P0, 3, 1), kfObs, &map);
        mp->AddObservation(kfObs, 0);
        cur->mvpMapPoints[i2] = mp; idxOf[mp] = -2; owned.push_back(mp);
    }
}
ProjectionLastScene::~ProjectionLastScene() { for (MapPoint* mp : owned) delete mp; delete cur; delete last; }
void ProjectionLastScene::read(int32_t* matchCur) const {
    for (int i2 = 0; i2 < cur->N; i2++) matchCur[i2] = cur->mvpMapPoints[i2] ? idxOf.at(cur->mvpMapPoints[i2]) : -1;
}

FuseScene::FuseScene(int nKF, const KpPOD* kKF, const uint8_t* dKF, const float* Tcw, int nMP, const float* Xw, const KpPOD* kObs, const uint8_t* dMP,
                     const float* TcwObs)
    : kfs(2), pKF(make_kf(kfs, 0, &map, nKF, kKF, dKF, Tcw)), pObs(make_kf(kfs, 1, &map, nMP, kObs, dMP, TcwObs)), mps(nMP) {
    for (int m = 0; m < nMP; m++) {
        MapPoint* mp = new MapPoint(mat_from(Xw + 3 * m, 3, 1), pObs, &map);
        mp->AddObservation(pObs, m); pObs->AddMapPoint(mp, m);
        mp->ComputeDistinctiveDescriptors(); mp->UpdateNormalAndDepth();
        mps[m] = mp;
    }
}
FuseScene::~FuseScene() { for (MapPoint* mp : mps) delete mp; }   // Fuse only re-seats these: it creates no MapPoint
int FuseScene::index_in_kf(int m) const {
    MapPoint* q = mps[m];
    while (q->GetReplaced()) q = q->GetReplaced();
    return q->GetIndexInKeyFrame(pKF);
}

TriangulationScene::TriangulationScene(int n1, const KpPOD* k1, const uint8_t* d1, const float* Tcw1, const uint8_t* hasMP1, const int32_t* node1, int n2,
                                       const KpPOD* k2, const uint8_t* d2, const float* Tcw2, const uint8_t* hasMP2, const int32_t* node2)
    : kfs(2), kf1(make_kf(kfs, 0, &map, n1, k1, d1, Tcw1)), kf2(make_kf(kfs, 1, &map, n2, k2, d2, Tcw2)) {
    for (int i = 0; i < n1; i++) kf1->mFeatVec.addFeature(node1[i], i);
    for (int i = 0; i < n2; i++) kf2->mFeatVec.addFeature(node2[i], i);
    for (int i = 0; i < n1; i++) if (hasMP1[i]) { MapPoint* mp = new MapPoint(mat_from(P0, 3, 1), kf1, &map); kf1->AddMapPoint(mp, i); owned.push_back(mp); }
    for (int i = 0; i < n2; i++) if (hasMP2[i]) { MapPoint* mp = new MapPoint(mat_from(P0, 3, 1), kf2, &map); kf2->AddMapPoint(mp, i); owned.push_back(mp); }
}
TriangulationScene::~TriangulationScene() { for (MapPoint* mp : owned) delete mp; }
void TriangulationScene::read(const std::vector<std::pair<size_t, size_t> >& pairs, int32_t* match12) const {
    for (int i = 0; i < kf1->N; i++) match12[i] = -1;
    for (size_t i = 0; i < pairs.size(); i++) match12[pairs[i].first] = (int32_t)pairs[i].second;
}

static int max_count(int n, const int32_t* offset) {
    int m = 0;
    for (int p = 0; p < n; p++) m = std::max(m, offset[p + 1] - offset[p]);
    return m;
}
DistinctiveScene::DistinctiveScene(int nPoints, const int32_t* offset, const uint8_t* desc) : kfs(max_count(nPoints, offset)), mps(nPoints) {
    const int maxObs = (int)kfs.kf.size();
    for (int j = 0; j < maxObs; j++) {
        std::vector<KpPOD> kps(nPoints, kHolderKp); std::vector<uint8_t> d((size_t)nPoints * 32, 0);   // rows of points with fewer observations stay unused
        for (int p = 0; p < nPoints; p++) if (offset[p] + j < offset[p + 1]) std::memcpy(&d[(size_t)p * 32], desc + 32 * (size_t)(offset[p] + j), 32);
        make_kf(kfs, j, &map, nPoints, kps.data(), d.data(), I4);
    }
    for (int p = 0; p < nPoints; p++) {
        mps[p] = new MapPoint(mat_from(P0, 3, 1), maxObs ? kfs.kf[0] : static_cast<KeyFrame*>(NULL), &map);
        for (int j = 0; offset[p] + j < offset[p + 1]; j++) mps[p]->AddObservation(kfs.kf[j], p);
    }
}
DistinctiveScene::~DistinctiveScene() { for (MapPoint* mp : mps) delete mp; }

}  // namespace scene

// ORACLE (test infrastructure, not product code): the reference objects both harnesses build from flat arrays, defined once.
// oracle/ref_api.cpp (libref.so, libref_fma.so) runs the reference's methods on these scenes; oracle/dropin_api.cpp (libdropin.so) runs the
// drop-in definitions and the reference's CPU bodies on them. Compiled against the reference's unmodified headers, like both API files.
#pragma once
#include <cstdint>
#include <map>
#include <utility>
#include <vector>

#include "CamModelGeneral.h"
#include "Frame.h"
#include "KeyFrame.h"
#include "Map.h"
#include "MapPoint.h"

struct RefCam { double c, d, e, u0, v0, p[5], invp[12]; int Iw, Ih, faceW, faceH; double fov; };   // same layout as orc::CamParams / oracle.CamParams

namespace scene {

struct KpPOD { float x, y, size, angle, response; int octave, class_id; };   // cv::KeyPoint's layout
const float I4[16] = {1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1};
const float P0[3] = {0, 0, 1};
const KpPOD kHolderKp = {700, 700, 31, 0, 0, 0, -1};   // key point of a frame that only lends descriptor rows

cv::Mat mat_from(const float* T, int r, int c);
// System::System, src/System.cpp:63-89
void set_camera(const RefCam* cp);
// a Frame carrying given key points / descriptors (NULL: zero rows) instead of extracted ones, with rays, scale tables, pose (if Tcw) and grid:
// what Tracking holds after Frame::Frame with the ORB settings of the reference's configs (8 levels, factor 1.2)
Frame* make_frame(int n, const KpPOD* kps, const uint8_t* desc, const float* Tcw);
// the first n key points, descriptors, rays and mGrid[face][col][row] sizes of F; any output may be NULL
void read_frame(const Frame& F, int n, KpPOD* kps, uint8_t* desc, float* rays, int32_t* gridCount);

// KeyFrames at ascending addresses, so that std::map<KeyFrame*, ...> (MapPoint::mObservations) iterates them in creation order
struct KFArray {
    char* buf; std::vector<KeyFrame*> kf;
    explicit KFArray(int n);
    KFArray(const KFArray&) = delete;
    KFArray& operator=(const KFArray&) = delete;
    ~KFArray();
    KeyFrame* make(int i, Frame& F, Map* map);
};

// SearchByProjection(CurrentFrame, LastFrame, th, true) (src/Tracking.cpp:634). LastFrame feature i holds a MapPoint at Xw[i] where hasMP[i],
// observed by one key frame where mpObs[i] > 0 (dMP: LastFrame's descriptors, which the MapPoint constructor copies). CurrentFrame slot i2
// holds a pre-existing, observed MapPoint where curTaken[i2].
struct ProjectionLastScene {
    Map map; KFArray kfs; Frame *cur, *last; std::vector<MapPoint*> owned; std::map<MapPoint*, int> idxOf;
    ProjectionLastScene(int nCur, const KpPOD* kCur, const uint8_t* dCur, const float* TcwCur, int nLast, const KpPOD* kLast, const float* TcwLast,
                        const uint8_t* hasMP, const float* Xw, const uint8_t* dMP, const int32_t* mpObs, const uint8_t* curTaken);
    ~ProjectionLastScene();
    // matchCur[i2]: LastFrame feature whose MapPoint sits in CurrentFrame.mvpMapPoints[i2], -1 empty, -2 a pre-existing MapPoint
    void read(int32_t* matchCur) const;
};

// Fuse(pKF, vpMapPoints, th) (LocalMapping::SearchInNeighbors) on a key frame pKF without MapPoints. MapPoint m: position Xw[m], observed once, by
// key point m of key frame pObs (pose TcwObs, key points kObs - their octave fixes the scale-invariance distances - and descriptors dMP), with
// normal, distances and descriptor from UpdateNormalAndDepth / ComputeDistinctiveDescriptors the way LocalMapping gives them.
struct FuseScene {
    Map map; KFArray kfs; KeyFrame *pKF, *pObs; std::vector<MapPoint*> mps;
    FuseScene(int nKF, const KpPOD* kKF, const uint8_t* dKF, const float* Tcw, int nMP, const float* Xw, const KpPOD* kObs, const uint8_t* dMP,
              const float* TcwObs);
    ~FuseScene();
    // key point of pKF on which MapPoint m, or what replaced it, sits; -1 none
    int index_in_kf(int m) const;
};

// SearchForTriangulation(pKF1, pKF2, E12, pairs) (LocalMapping::CreateNewMapPoints). node*: vocabulary node of every feature (mFeatVec),
// hasMP*: the key point already has a MapPoint.
struct TriangulationScene {
    Map map; KFArray kfs; KeyFrame *kf1, *kf2; std::vector<MapPoint*> owned;
    TriangulationScene(int n1, const KpPOD* k1, const uint8_t* d1, const float* Tcw1, const uint8_t* hasMP1, const int32_t* node1, int n2, const KpPOD* k2,
                       const uint8_t* d2, const float* Tcw2, const uint8_t* hasMP2, const int32_t* node2);
    ~TriangulationScene();
    // match12[i1] = i2 of the pair, or -1
    void read(const std::vector<std::pair<size_t, size_t> >& pairs, int32_t* match12) const;
};

// MapPoint p observed by the key frames 0 .. offset[p+1]-offset[p]-1 (MapPoint::ComputeDistinctiveDescriptors): key frame j lends row p of its
// descriptors, desc row offset[p]+j, to MapPoint p
struct DistinctiveScene {
    Map map; KFArray kfs; std::vector<MapPoint*> mps;
    DistinctiveScene(int nPoints, const int32_t* offset, const uint8_t* desc);
    ~DistinctiveScene();
};

}  // namespace scene

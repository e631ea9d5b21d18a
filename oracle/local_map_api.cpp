// ORACLE / TEST HARNESS (not product code): entries of oracle/_ref/libdropin_local_map.so (recipe oracle/local_map_dropin.mk), which links
// libdropin.so's ingredients with this file. It runs the local-map ORBMatcher::SearchByProjection(F, vpMapPoints, th) (Tracking::SearchLocalPoints)
// on reference Frame / MapPoint objects: the drop-in definition (dropin/ORBMatcher_b200.cpp -> libcubemap_b200.so) and the reference's own CPU
// body (dropin/ORBMatcher_cpu_forward.cpp), for local maps past 4096 MapPoints (tests/test_gpu_local_map.py, tools/local_map_latency.py).
#include <chrono>
#include <map>
#include <vector>

#include "ORBMatcher.h"
#include "ref_scene.h"

using namespace scene;

int cslam_cpu_SearchByProjection(ORBMatcher* m, Frame& F, const std::vector<MapPoint*>& vpMapPoints, const float th);

namespace {
// A Frame with nF key points and nMP MapPoints carrying what Frame::isInFrustum leaves in them (mbTrackInView, mTrackProjX/Y,
// mnTrackScaleLevel, mTrackViewCos), with one observation where mpObs; slots with fTaken hold a MapPoint with an observation before the
// search. run(): ORBMatcher(nnratio).SearchByProjection(F, vpMapPoints, th) through the drop-in (gpu) or the reference's CPU body; match[i] =
// the index of the MapPoint in F.mvpMapPoints[i] afterwards (-1: NULL, -2: the MapPoint it held before).
struct LocalMapScene {
    Map map; Frame* F; Frame* holder; KeyFrame* kfObs; std::vector<MapPoint*> mps, owned; std::map<MapPoint*, int> idxOf;
    LocalMapScene(int nF, const KpPOD* kF, const uint8_t* dF, int nMP, const uint8_t* inView, const float* projXY, const int32_t* level, const float* viewCos,
                  const uint8_t* dMP, const int32_t* mpObs, const uint8_t* fTaken) : mps(nMP) {
        F = make_frame(nF, kF, dF, I4);
        std::vector<KpPOD> kd(nMP, kHolderKp);
        holder = make_frame(nMP, kd.data(), dMP, I4);   // lends its descriptor rows to the MapPoint constructor
        kfObs = new KeyFrame(*holder, &map, NULL);
        for (int m = 0; m < nMP; m++) {
            MapPoint* mp = new MapPoint(mat_from(P0, 3, 1), &map, holder, m);
            if (mpObs[m] > 0) mp->AddObservation(kfObs, m);
            mp->mbTrackInView = inView[m] != 0; mp->mTrackProjX = projXY[2 * m]; mp->mTrackProjY = projXY[2 * m + 1]; mp->mnTrackScaleLevel = level[m];
            mp->mTrackViewCos = viewCos[m];
            mps[m] = mp; idxOf[mp] = m; owned.push_back(mp);
        }
        for (int i = 0; i < nF; i++)
            if (fTaken[i]) { MapPoint* mp = new MapPoint(mat_from(P0, 3, 1), kfObs, &map); mp->AddObservation(kfObs, 0); F->mvpMapPoints[i] = mp; idxOf[mp] = -2; owned.push_back(mp); }
    }
    ~LocalMapScene() { for (MapPoint* mp : owned) delete mp; delete kfObs; delete F; delete holder; }
    int run(bool gpu, float th, float nnratio, int32_t* match) {
        ORBMatcher matcher(nnratio, true);
        const int n = gpu ? matcher.SearchByProjection(*F, mps, th) : cslam_cpu_SearchByProjection(&matcher, *F, mps, th);
        for (int i = 0; i < F->N; i++) match[i] = F->mvpMapPoints[i] ? idxOf[F->mvpMapPoints[i]] : -1;
        return n;
    }
};
}  // namespace

extern "C" {

// SearchByProjection(F, vpMapPoints, th) (Tracking::SearchLocalPoints): the GPU drop-in and the reference's CPU body, each on a scene of its own
void dropin_search_by_projection_local(int nF, const KpPOD* kF, const uint8_t* dF, int nMP, const uint8_t* inView, const float* projXY, const int32_t* level,
                                       const float* viewCos, const uint8_t* dMP, const int32_t* mpObs, const uint8_t* fTaken, float th, float nnratio, int32_t* matchGpu,
                                       int32_t* nGpu, int32_t* matchCpu, int32_t* nCpu) {
    { LocalMapScene s(nF, kF, dF, nMP, inView, projXY, level, viewCos, dMP, mpObs, fTaken); *nGpu = s.run(true, th, nnratio, matchGpu); }
    { LocalMapScene s(nF, kF, dF, nMP, inView, projXY, level, viewCos, dMP, mpObs, fTaken); *nCpu = s.run(false, th, nnratio, matchCpu); }
}

// The reference's CPU body alone on such a scene (tools/local_map_latency.py): *ms = the milliseconds of the search itself, scene building excluded
void ref_search_by_projection_local_cpu(int nF, const KpPOD* kF, const uint8_t* dF, int nMP, const uint8_t* inView, const float* projXY, const int32_t* level,
                                        const float* viewCos, const uint8_t* dMP, const int32_t* mpObs, const uint8_t* fTaken, float th, float nnratio, int32_t* match,
                                        double* ms) {
    LocalMapScene s(nF, kF, dF, nMP, inView, projXY, level, viewCos, dMP, mpObs, fTaken);
    const auto t0 = std::chrono::steady_clock::now();
    s.run(false, th, nnratio, match);
    *ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
}

}  // extern "C"

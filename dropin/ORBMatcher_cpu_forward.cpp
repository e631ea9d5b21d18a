// Compiled with the SAME rename as the reference's src/ORBMatcher.cpp (COMPILE_DEFINITIONS
// "SearchByBoW=SearchByBoW_cpu;SearchByProjection=SearchByProjection_cpu;Fuse=Fuse_cpu;SearchForTriangulation=SearchForTriangulation_cpu;
// SearchForInitialization=SearchForInitialization_cpu"),
// so inside this file the names below refer to the reference's own CPU bodies. It exports them as free functions:
//  * for the two SearchByProjection overloads that are NOT moved to the GPU (relocalisation against a KeyFrame, loop-closing with a Sim3) -
//    the preprocessor rename cannot tell overloads apart, so dropin/ORBMatcher_b200.cpp forwards those two back to the reference's code;
//  * for A/B runs and for the link-and-run test (tests/test_gpu_dropin.py), which matches the same objects with both implementations.
#include "ORBMatcher.h"

int cslam_cpu_SearchByProjection(ORBMatcher* m, Frame& CurrentFrame, KeyFrame* pKF, const std::set<MapPoint*>& sAlreadyFound, const float th, const int ORBdist) {
    return m->SearchByProjection(CurrentFrame, pKF, sAlreadyFound, th, ORBdist);
}
int cslam_cpu_SearchByProjection(ORBMatcher* m, KeyFrame* pKF, cv::Mat Scw, const std::vector<MapPoint*>& vpPoints, std::vector<MapPoint*>& vpMatched, int th) {
    return m->SearchByProjection(pKF, Scw, vpPoints, vpMatched, th);
}
int cslam_cpu_SearchByProjection(ORBMatcher* m, Frame& CurrentFrame, const Frame& LastFrame, const float th, const bool bMono) { return m->SearchByProjection(CurrentFrame, LastFrame, th, bMono); }
int cslam_cpu_SearchByProjection(ORBMatcher* m, Frame& F, const std::vector<MapPoint*>& vpMapPoints, const float th) { return m->SearchByProjection(F, vpMapPoints, th); }
int cslam_cpu_SearchByBoW(ORBMatcher* m, KeyFrame* pKF, Frame& F, std::vector<MapPoint*>& vpMapPointMatches) { return m->SearchByBoW(pKF, F, vpMapPointMatches); }
int cslam_cpu_SearchByBoW(ORBMatcher* m, KeyFrame* pKF1, KeyFrame* pKF2, std::vector<MapPoint*>& vpMatches12) { return m->SearchByBoW(pKF1, pKF2, vpMatches12); }
int cslam_cpu_Fuse(ORBMatcher* m, KeyFrame* pKF, const std::vector<MapPoint*>& vpMapPoints, const float th) { return m->Fuse(pKF, vpMapPoints, th); }
int cslam_cpu_Fuse(ORBMatcher* m, KeyFrame* pKF, cv::Mat Scw, const std::vector<MapPoint*>& vpPoints, float th, std::vector<MapPoint*>& vpReplacePoint) { return m->Fuse(pKF, Scw, vpPoints, th, vpReplacePoint); }
int cslam_cpu_SearchForTriangulation(ORBMatcher* m, KeyFrame* pKF1, KeyFrame* pKF2, cv::Mat E12, std::vector<std::pair<size_t, size_t> >& vMatchedPairs) {
    return m->SearchForTriangulation(pKF1, pKF2, E12, vMatchedPairs);
}
int cslam_cpu_SearchForInitialization(ORBMatcher* m, Frame& F1, Frame& F2, std::vector<cv::Point2f>& vbPrevMatched, std::vector<int>& vnMatches12, int windowSize) {
    return m->SearchForInitialization(F1, F2, vbPrevMatched, vnMatches12, windowSize);
}

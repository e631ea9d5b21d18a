// ORACLE / TEST HARNESS (not product code): entries of oracle/_ref/libref_init.so (recipe oracle/init_search_dropin.mk), which links the
// reference's own objects of libref.so with ref_scene.cpp and this file, and needs no GPU. It runs the reference's SearchForInitialization and
// GetFeaturesInArea on Frames holding given key points (tests/test_oracle_init_search.py pins the oracle to them).
#include <vector>

#include "ORBMatcher.h"
#include "ref_scene.h"

using namespace scene;

extern "C" {

void ref_init_set_camera(const RefCam* cp) { set_camera(cp); }

// ORBMatcher(nnratio, checkOri).SearchForInitialization(F1, F2, vbPrevMatched, vnMatches12, windowSize)   src/ORBMatcher.cpp:676-794 ; prevXY (n1 x 2) in / out
int ref_init_search_for_initialization(int n1, const KpPOD* k1, const uint8_t* d1, int n2, const KpPOD* k2, const uint8_t* d2, float* prevXY, int windowSize, float nnratio,
                                       int checkOri, int32_t* match12) {
    Frame* F1 = make_frame(n1, k1, d1, I4);
    Frame* F2 = make_frame(n2, k2, d2, I4);
    std::vector<cv::Point2f> prev(n1); std::vector<int> m12;
    for (int i = 0; i < n1; i++) prev[i] = cv::Point2f(prevXY[2 * i], prevXY[2 * i + 1]);
    ORBMatcher matcher(nnratio, checkOri != 0);
    const int n = matcher.SearchForInitialization(*F1, *F2, prev, m12, windowSize);
    for (int i = 0; i < n1; i++) { match12[i] = m12[i]; prevXY[2 * i] = prev[i].x; prevXY[2 * i + 1] = prev[i].y; }
    delete F1; delete F2;
    return n;
}

// Frame::GetFeaturesInArea (src/Frame.cpp:251-716) on a Frame holding the given key points, for nq windows (x, y, r) with levels (min, max):
// counts[q] indices each, concatenated into idx (at most cap in all). Returns the total.
int ref_init_features_in_area(int n, const KpPOD* kps, int nq, const float* xyr, const int32_t* levels, int32_t* counts, int32_t* idx, int cap) {
    Frame* F = make_frame(n, kps, NULL, NULL);
    int m = 0;
    for (int q = 0; q < nq; q++) {
        const std::vector<size_t> v = F->GetFeaturesInArea(xyr[3 * q], xyr[3 * q + 1], xyr[3 * q + 2], levels[2 * q], levels[2 * q + 1]);
        counts[q] = (int32_t)v.size();
        for (size_t j = 0; j < v.size(); j++) { if (m < cap) idx[m] = (int32_t)v[j]; m++; }
    }
    delete F;
    return m;
}

}  // extern "C"

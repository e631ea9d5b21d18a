// ORACLE / TEST HARNESS (not product code): entries of oracle/_ref/libdropin_init.so (recipe oracle/init_search_dropin.mk), which links
// libdropin.so's ingredients with this file. It runs ORBMatcher::SearchForInitialization(F1, F2, vbPrevMatched, vnMatches12, windowSize)
// (Tracking::CubemapInitialization) on reference Frames built from flat arrays: the drop-in definition (dropin/ORBMatcher_b200.cpp ->
// libcubemap_b200.so) and the reference's own CPU body (dropin/ORBMatcher_cpu_forward.cpp), for tests/test_gpu_init_search.py and
// tools/init_search_latency.py.
#include <chrono>
#include <vector>

#include "ORBMatcher.h"
#include "ref_scene.h"

using namespace scene;

int cslam_cpu_SearchForInitialization(ORBMatcher* m, Frame& F1, Frame& F2, std::vector<cv::Point2f>& vbPrevMatched, std::vector<int>& vnMatches12, int windowSize);

namespace {
// F1 and F2 holding the given key points and descriptors. run(): one call through the drop-in (gpu) or the reference's CPU body on
// vbPrevMatched = prevXY, which is updated in place; match12 = vnMatches12 afterwards.
struct InitScene {
    Frame *F1, *F2;
    InitScene(int n1, const KpPOD* k1, const uint8_t* d1, int n2, const KpPOD* k2, const uint8_t* d2) : F1(make_frame(n1, k1, d1, I4)), F2(make_frame(n2, k2, d2, I4)) {}
    ~InitScene() { delete F1; delete F2; }
    int run(bool gpu, float* prevXY, int windowSize, float nnratio, int checkOri, int32_t* match12, double* ms) {
        std::vector<cv::Point2f> prev(F1->N); std::vector<int> m12;
        for (int i = 0; i < F1->N; i++) prev[i] = cv::Point2f(prevXY[2 * i], prevXY[2 * i + 1]);
        ORBMatcher matcher(nnratio, checkOri != 0);
        const auto t0 = std::chrono::steady_clock::now();
        const int n = gpu ? matcher.SearchForInitialization(*F1, *F2, prev, m12, windowSize) : cslam_cpu_SearchForInitialization(&matcher, *F1, *F2, prev, m12, windowSize);
        if (ms) *ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
        for (int i = 0; i < F1->N; i++) { match12[i] = m12[i]; prevXY[2 * i] = prev[i].x; prevXY[2 * i + 1] = prev[i].y; }
        return n;
    }
};
}  // namespace

extern "C" {

// The GPU drop-in and the reference's CPU body on the same Frames, each on its own copy of the centres (xyGpu / xyCpu: in / out)
void dropin_search_for_initialization(int n1, const KpPOD* k1, const uint8_t* d1, int n2, const KpPOD* k2, const uint8_t* d2, int windowSize, float nnratio, int checkOri,
                                      float* xyGpu, int32_t* matchGpu, int32_t* nGpu, float* xyCpu, int32_t* matchCpu, int32_t* nCpu) {
    InitScene s(n1, k1, d1, n2, k2, d2);
    *nGpu = s.run(true, xyGpu, windowSize, nnratio, checkOri, matchGpu, NULL);
    *nCpu = s.run(false, xyCpu, windowSize, nnratio, checkOri, matchCpu, NULL);
}

// reps calls of one implementation on one pair of Frames built once, each from the same centres prevXY (not modified): ms[r] = the
// milliseconds of call r, the method call alone
void time_search_for_initialization(int gpu, int n1, const KpPOD* k1, const uint8_t* d1, int n2, const KpPOD* k2, const uint8_t* d2, const float* prevXY, int windowSize,
                                    float nnratio, int checkOri, int reps, double* ms) {
    InitScene s(n1, k1, d1, n2, k2, d2);
    std::vector<float> xy(2 * (size_t)n1); std::vector<int32_t> m(n1);
    for (int r = 0; r < reps; r++) {
        xy.assign(prevXY, prevXY + 2 * (size_t)n1);
        s.run(gpu != 0, xy.data(), windowSize, nnratio, checkOri, m.data(), ms + r);
    }
}

}  // extern "C"

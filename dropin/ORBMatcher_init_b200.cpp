// Drop-in DEFINITION of ORBMatcher::SearchForInitialization (include/ORBMatcher.h:71) on libcubemap_b200.so, compiled INSIDE the CubemapSLAM
// tree against the reference's own, unmodified include/ORBMatcher.h, like dropin/ORBMatcher_b200.cpp, whose per-thread tracker handle it
// shares. The reference's body in src/ORBMatcher.cpp is renamed away at compile time (INTEGRATION.md: SearchForInitialization=
// SearchForInitialization_cpu in that file's COMPILE_DEFINITIONS); dropin/ORBMatcher_cpu_forward.cpp exports it as cslam_cpu_SearchForInitialization.
#include "ORBMatcher.h"

#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>

#include "cubemap_b200.h"

cslam_tracker* cubemap_b200_thread_tracker();   // dropin/ORBMatcher_b200.cpp

// reference src/ORBMatcher.cpp:676-794 (Tracking::CubemapInitialization :428-429, on every frame until the map initialises). Frames of the
// initialisation extractor (3*nFeatures + 3*nlevels key points) are taken up to CSLAM_BOW_FV_MAX_FEATURES; past that, or with a vbPrevMatched
// that does not hold one centre per F1 key point, the call fails loudly.
int ORBMatcher::SearchForInitialization(Frame& F1, Frame& F2, std::vector<cv::Point2f>& vbPrevMatched, std::vector<int>& vnMatches12, int windowSize) {
    const int n1 = (int)F1.mvKeys.size(), n2 = (int)F2.mvKeys.size();
    if (n1 > CSLAM_BOW_FV_MAX_FEATURES || n2 > CSLAM_BOW_FV_MAX_FEATURES) {
        std::fprintf(stderr, "ORBMatcher (cubemap_b200): SearchForInitialization on frames of %d and %d key points (at most %d)\n", n1, n2, CSLAM_BOW_FV_MAX_FEATURES);
        std::exit(EXIT_FAILURE);
    }
    if (vbPrevMatched.size() != (size_t)F1.N) {
        std::fprintf(stderr, "ORBMatcher (cubemap_b200): SearchForInitialization with %zu previous matches for %d key points\n", vbPrevMatched.size(), F1.N);
        std::exit(EXIT_FAILURE);
    }
    vnMatches12 = std::vector<int>(n1, -1);
    if (n1 == 0 || n2 == 0) return 0;
    std::vector<uint8_t> d1((size_t)n1 * 32), d2((size_t)n2 * 32);
    for (int i = 0; i < n1; i++) std::memcpy(&d1[(size_t)i * 32], F1.mDescriptors.ptr<uchar>(i), 32);
    for (int i = 0; i < n2; i++) std::memcpy(&d2[(size_t)i * 32], F2.mDescriptors.ptr<uchar>(i), 32);
    static_assert(sizeof(cv::KeyPoint) == sizeof(cslam_keypoint), "cv::KeyPoint layout");
    static_assert(sizeof(cv::Point2f) == 2 * sizeof(float), "cv::Point2f layout");
    CamModelGeneral* cam = CamModelGeneral::GetCamera();
    int32_t n = 0;
    if (cslam_search_for_initialization(cubemap_b200_thread_tracker(), reinterpret_cast<const cslam_keypoint*>(F1.mvKeys.data()), d1.data(), n1,
                                        reinterpret_cast<const float*>(vbPrevMatched.data()), reinterpret_cast<const cslam_keypoint*>(F2.mvKeys.data()), d2.data(), n2,
                                        cam->GetCubeFaceWidth(), cam->GetCubeFaceHeight(), windowSize, mfNNratio, mbCheckOrientation, vnMatches12.data(), &n) != CSLAM_OK) {
        std::fprintf(stderr, "ORBMatcher (cubemap_b200): %s\n", cslam_last_error());
        std::exit(EXIT_FAILURE);
    }
    for (int i1 = 0; i1 < n1; i1++) if (vnMatches12[i1] >= 0) vbPrevMatched[i1] = F2.mvKeys[vnMatches12[i1]].pt;
    return n;
}

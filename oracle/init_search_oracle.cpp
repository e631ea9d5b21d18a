// ORACLE (test infrastructure, not product code): C entries of oracle/liboracle_init.so (recipe oracle/init_search_dropin.mk): the oracle's
// SearchForInitialization (init_search.h) and an uncapped GetFeaturesInArea, each on a grid built from the given F2 key points.
#include "init_search.h"

using namespace orc;

extern "C" {

int orc_init_search(const KeyPoint* k2, const uint8_t* d2, int n2, int faceW, const KeyPoint* k1, const uint8_t* d1, int n1, float* prevXY, int windowSize, float nnratio,
                    int checkOri, int* match12) {
    FrameGrid g; g.build(k2, n2, faceW, faceW);
    return fi_search_for_initialization(g, k2, d2, n2, k1, d1, n1, prevXY, windowSize, nnratio, checkOri != 0, match12);
}

// nq windows (x, y, r) with levels (min, max): counts[q] indices each, concatenated into idx (at most cap in all). Returns the total.
int orc_init_features_in_area(const KeyPoint* kps, int n, int faceW, int nq, const float* xyr, const int* levels, int* counts, int* idx, int cap) {
    FrameGrid g; g.build(kps, n, faceW, faceW);
    std::vector<int> v;
    int m = 0;
    for (int q = 0; q < nq; q++) {
        fi_features_in_area(g, kps, xyr[3 * q], xyr[3 * q + 1], xyr[3 * q + 2], levels[2 * q], levels[2 * q + 1], v);
        counts[q] = (int)v.size();
        for (int i : v) { if (m < cap) idx[m] = i; m++; }
    }
    return m;
}

}  // extern "C"

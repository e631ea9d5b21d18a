// ORACLE (test infrastructure, not product code): CPU restatement of ORBMatcher::SearchForInitialization (src/ORBMatcher.cpp:676-794,
// Tracking::CubemapInitialization :428-429) on frame_index.h's grid and window lookup. Pinned against the reference's own compiled body in
// tests/test_oracle_init_search.py; built into oracle/liboracle_init.so (recipe oracle/init_search_dropin.mk, entries init_search_oracle.cpp).
#pragma once
#include <climits>
#include <cmath>
#include <vector>
#include "frame_index.h"

namespace orc {

// g = F2's grid over k2 (n2 key points). prevXY (n1 x 2, in / out): vbPrevMatched. match12[i1] = i2 or -1. Returns nmatches.
static inline int fi_search_for_initialization(const FrameGrid& g, const KeyPoint* k2, const uint8_t* d2, int n2, const KeyPoint* k1, const uint8_t* d1, int n1,
                                               float* prevXY, int windowSize, float nnratio, bool checkOri, int* match12) {
    const int nBins = 30;   // ceil(360 / HISTO_LENGTH)
    std::vector<std::vector<int> > rotHist(nBins);
    const float factor = 1.0f / 12;
    int nmatches = 0;
    for (int i = 0; i < n1; i++) match12[i] = -1;
    std::vector<int> matchedDist(n2, INT_MAX), matches21(n2, -1);   // vMatchedDistance, vnMatches21
    std::vector<int> vIdx;
    for (int i1 = 0; i1 < n1; i1++) {
        const int level1 = k1[i1].octave;
        if (level1 > 0) continue;
        fi_features_in_area(g, k2, prevXY[2 * i1], prevXY[2 * i1 + 1], (float)windowSize, level1, level1, vIdx);
        if (vIdx.empty()) continue;
        int bestDist = INT_MAX, bestDist2 = INT_MAX, bestIdx2 = -1;
        for (int i2 : vIdx) {
            const int dist = descriptor_distance(d1 + 32 * (size_t)i1, d2 + 32 * (size_t)i2);
            if (matchedDist[i2] <= dist) continue;
            if (dist < bestDist) { bestDist2 = bestDist; bestDist = dist; bestIdx2 = i2; }
            else if (dist < bestDist2) bestDist2 = dist;
        }
        if (bestDist <= 50 && bestDist < (float)bestDist2 * nnratio) {   // TH_LOW, ratio test
            if (matches21[bestIdx2] >= 0) { match12[matches21[bestIdx2]] = -1; nmatches--; }
            match12[i1] = bestIdx2; matches21[bestIdx2] = i1; matchedDist[bestIdx2] = bestDist;
            nmatches++;
            if (checkOri) {
                float rot = k1[i1].angle - k2[bestIdx2].angle;
                if (rot < 0.0) rot += 360.0f;
                int bin = (int)roundf(rot * factor);
                if (bin == nBins) bin = 0;
                rotHist[bin].push_back(i1);   // stays listed when a later i1 takes its key point
            }
        }
    }
    if (checkOri) {
        int ind1 = -1, ind2 = -1, ind3 = -1;
        compute_three_maxima(rotHist.data(), nBins, ind1, ind2, ind3);
        for (int b = 0; b < nBins; b++)
            if (b != ind1 && b != ind2 && b != ind3)
                for (int j : rotHist[b]) if (match12[j] >= 0) { match12[j] = -1; nmatches--; }
    }
    for (int i1 = 0; i1 < n1; i1++)
        if (match12[i1] >= 0) { prevXY[2 * i1] = k2[match12[i1]].x; prevXY[2 * i1 + 1] = k2[match12[i1]].y; }
    return nmatches;
}

}  // namespace orc

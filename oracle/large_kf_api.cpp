// ORACLE / TEST HARNESS (not product code): entries of oracle/_ref/libdropin_large.so (recipe oracle/large_kf_dropin.mk), which links
// libdropin.so's ingredients with this file. It runs ORBMatcher::SearchByBoW in both forms on reference KeyFrame / Frame / MapPoint objects:
// the drop-in definitions (dropin/ORBMatcher_b200.cpp -> libcubemap_b200.so) and the reference's own CPU bodies
// (dropin/ORBMatcher_cpu_forward.cpp), or the CPU bodies alone, which need no GPU (tests/test_oracle_large_kf.py pins the oracle to them).
#include <map>
#include <vector>

#include "ORBMatcher.h"
#include "ref_scene.h"

using namespace scene;

int cslam_cpu_SearchByBoW(ORBMatcher* m, KeyFrame* pKF, Frame& F, std::vector<MapPoint*>& vpMapPointMatches);
int cslam_cpu_SearchByBoW(ORBMatcher* m, KeyFrame* pKF1, KeyFrame* pKF2, std::vector<MapPoint*>& vpMatches12);

namespace {
// Side s of a SearchByBoW call: a Frame with the given key points, descriptors and FeatureVector (node[i] < 0: feature i is in no node), and,
// for a key frame, a MapPoint on every feature with valid[i]
struct BowSide {
    Frame* F; KeyFrame* pKF = NULL; std::map<MapPoint*, int> idxOf;
    BowSide(Map* map, int n, const KpPOD* kp, const uint8_t* desc, const uint8_t* valid, const int32_t* node, bool keyFrame) {
        F = make_frame(n, kp, desc, I4);
        for (int i = 0; i < n; i++) if (node[i] >= 0) F->mFeatVec.addFeature((DBoW2::NodeId)node[i], (unsigned)i);
        if (!keyFrame) return;
        pKF = new KeyFrame(*F, map, static_cast<KeyFrameDatabase*>(NULL));
        for (int i = 0; i < n; i++) if (valid[i]) { MapPoint* mp = new MapPoint(mat_from(P0, 3, 1), pKF, map); pKF->AddMapPoint(mp, i); idxOf[mp] = i; }
    }
    ~BowSide() { for (std::map<MapPoint*, int>::iterator it = idxOf.begin(); it != idxOf.end(); ++it) delete it->first; delete pKF; delete F; }
    int index(MapPoint* mp) const { return mp ? idxOf.at(mp) : -1; }
};

// kfkf = 0: ORBMatcher(nnratio, checkOri).SearchByBoW(pKF, F, matches), match[j] per F feature = the KF feature whose MapPoint F feature j got.
// kfkf = 1: SearchByBoW(pKF1, pKF2, matches12), match[i] per feature of key frame 1 = the feature of key frame 2 whose MapPoint it got.
// runGpu = 0: only the reference's CPU body (matchGpu / nGpu untouched).
void search_by_bow(int kfkf, int n1, const KpPOD* k1, const uint8_t* d1, const uint8_t* valid1, const int32_t* node1, int n2, const KpPOD* k2, const uint8_t* d2,
                   const uint8_t* valid2, const int32_t* node2, float nnratio, int checkOri, int runGpu, int32_t* matchGpu, int32_t* nGpu, int32_t* matchCpu,
                   int32_t* nCpu) {
    Map map;
    BowSide s1(&map, n1, k1, d1, valid1, node1, true), s2(&map, n2, k2, d2, valid2, node2, kfkf != 0);
    ORBMatcher matcher(nnratio, checkOri != 0);
    for (int pass = runGpu ? 0 : 1; pass < 2; pass++) {
        std::vector<MapPoint*> out;
        int n;
        if (kfkf) n = pass == 0 ? matcher.SearchByBoW(s1.pKF, s2.pKF, out) : cslam_cpu_SearchByBoW(&matcher, s1.pKF, s2.pKF, out);
        else n = pass == 0 ? matcher.SearchByBoW(s1.pKF, *s2.F, out) : cslam_cpu_SearchByBoW(&matcher, s1.pKF, *s2.F, out);
        int32_t* m = pass == 0 ? matchGpu : matchCpu;
        for (size_t j = 0; j < out.size(); j++) m[j] = kfkf ? s2.index(out[j]) : s1.index(out[j]);
        (pass == 0 ? *nGpu : *nCpu) = n;
    }
}
}  // namespace

extern "C" {

// SearchByBoW(pKF1, pKF2, matches12) (LoopClosing::ComputeSim3): the GPU drop-in and the reference's CPU body on the same key frames
void dropin_search_by_bow_kf(int n1, const KpPOD* k1, const uint8_t* d1, const uint8_t* valid1, const int32_t* node1, int n2, const KpPOD* k2, const uint8_t* d2,
                             const uint8_t* valid2, const int32_t* node2, float nnratio, int checkOri, int32_t* matchGpu, int32_t* nGpu, int32_t* matchCpu, int32_t* nCpu) {
    search_by_bow(1, n1, k1, d1, valid1, node1, n2, k2, d2, valid2, node2, nnratio, checkOri, 1, matchGpu, nGpu, matchCpu, nCpu);
}

// The reference's CPU body alone, both forms (valid2 is not read for kfkf = 0). Returns nmatches.
int ref_search_by_bow_cpu(int kfkf, int n1, const KpPOD* k1, const uint8_t* d1, const uint8_t* valid1, const int32_t* node1, int n2, const KpPOD* k2, const uint8_t* d2,
                          const uint8_t* valid2, const int32_t* node2, float nnratio, int checkOri, int32_t* match) {
    int32_t n = 0;
    search_by_bow(kfkf, n1, k1, d1, valid1, node1, n2, k2, d2, valid2, node2, nnratio, checkOri, 0, NULL, NULL, match, &n);
    return n;
}

}  // extern "C"

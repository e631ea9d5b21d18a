// ORACLE / TEST HARNESS (not product code): the ComputeBoW drop-in (dropin/ComputeBoW_b200.cpp) against the reference's own bodies, on the
// reference's own Frame / KeyFrame objects (oracle/ref_scene.cpp) and a vocabulary loaded by the reference's own loader. Linked by oracle/bow_dropin.mk
// into oracle/_ref/libdropin_bow.so, for tests/test_oracle_compute_bow.py, tests/test_gpu_compute_bow.py and tools/bow_latency.py: libdropin.so's
// ingredients with the reference's src/Frame.cpp and src/KeyFrame.cpp compiled with -DComputeBoW=ComputeBoW_cpu, exactly as INTEGRATION.md
// prescribes, plus the two ComputeBoW drop-in sources.
#include <algorithm>
#include <chrono>
#include <cstring>
#include <thread>
#include <vector>

#include "KeyFrame.h"
#include "ORBVocabulary.h"
#include "ref_scene.h"

using namespace scene;

// the reference's ComputeBoW bodies (dropin/ComputeBoW_cpu_forward.cpp) and the drop-in's vocabulary import (dropin/ComputeBoW_b200.cpp)
void cslam_cpu_Frame_ComputeBoW(Frame& F);
void cslam_cpu_KeyFrame_ComputeBoW(KeyFrame* pKF);
namespace cubemap_b200 {
void ExportVocabulary(const ORBVocabulary* voc, int* k, int* L, int* n_nodes, const int32_t** parent, const uint8_t** is_leaf, const uint8_t** desc, const double** weight);
}

namespace {

// A Frame (keyframe = 0) or a KeyFrame (1) of n features with the given descriptors and vocabulary; preset bit 1 / 2: mBowVec / mFeatVec already
// hold one entry (word 7 -> 0.5 / node 3 -> {0}) before ComputeBoW runs, as after an earlier call
struct BowScene {
    Map map; Frame* F; KeyFrame* kf = NULL;
    BowScene(ORBVocabulary* voc, int keyframe, int n, const uint8_t* desc, int preset) {
        const std::vector<KpPOD> kps(std::max(n, 1), kHolderKp);
        F = make_frame(n, kps.data(), desc, I4);
        F->mpORBvocabulary = voc;
        if (preset & 1) F->mBowVec[7] = 0.5;
        if (preset & 2) F->mFeatVec[3].push_back(0);
        if (keyframe) kf = new KeyFrame(*F, &map, NULL);                 // copies the vocabulary, mBowVec and mFeatVec of F
    }
    ~BowScene() { delete kf; delete F; }
    DBoW2::BowVector& bow() { return kf ? kf->mBowVec : F->mBowVec; }
    DBoW2::FeatureVector& fv() { return kf ? kf->mFeatVec : F->mFeatVec; }
    void run(int cpu) {
        if (kf) { if (cpu) cslam_cpu_KeyFrame_ComputeBoW(kf); else kf->ComputeBoW(); }      // src/KeyFrame.cpp:94-103 / dropin/ComputeBoW_b200.cpp
        else { if (cpu) cslam_cpu_Frame_ComputeBoW(*F); else F->ComputeBoW(); }           // src/Frame.cpp:719-726 / dropin/ComputeBoW_b200.cpp
    }
    // mBowVec as (word, value) in map order; mFeatVec as CSR: node j holds fvFeat[fvStart[j] .. fvStart[j+1])
    void read(int32_t* bowWord, double* bowVal, int32_t* nBow, int32_t* fvNode, int32_t* fvStart, int32_t* fvFeat, int32_t* nFv) {
        int j = 0;
        for (DBoW2::BowVector::const_iterator it = bow().begin(); it != bow().end(); ++it, ++j) { bowWord[j] = (int32_t)it->first; bowVal[j] = it->second; }
        *nBow = j;
        j = 0; int p = 0;
        for (DBoW2::FeatureVector::const_iterator it = fv().begin(); it != fv().end(); ++it, ++j) {
            fvNode[j] = (int32_t)it->first; fvStart[j] = p;
            for (size_t q = 0; q < it->second.size(); q++) fvFeat[p++] = (int32_t)it->second[q];
        }
        fvStart[j] = p; *nFv = j;
    }
};

}  // namespace

extern "C" {

// ORBVocabulary::loadFromTextFile(path) (ThirdParty/DBoW2/DBoW2/TemplatedVocabulary.h:1337-1424) into *out; returns 0, or -1 if it fails. The
// object lives as long as the process, like System's: the drop-in imports a vocabulary once per address, so a freed one must not be followed by
// another at its address.
int dropin_voc_load(const char* path, void** out) {
    ORBVocabulary* voc = new ORBVocabulary();
    if (!voc->loadFromTextFile(path)) { delete voc; *out = NULL; return -1; }
    *out = voc;
    return 0;
}

// info = k, L, number of nodes past the root, number of words (ORBVocabulary::size)
void dropin_voc_info(void* voc, int32_t* info) {
    const int32_t* parent; const uint8_t *isLeaf, *desc; const double* weight;
    cubemap_b200::ExportVocabulary(static_cast<ORBVocabulary*>(voc), &info[0], &info[1], &info[2], &parent, &isLeaf, &desc, &weight);
    info[3] = (int32_t)static_cast<ORBVocabulary*>(voc)->size();
}
// the drop-in importer's arrays for nodes 1..n (what it uploads): parent, word flag, 32 descriptor bytes, weight
void dropin_voc_export(void* voc, int32_t* parent, uint8_t* isLeaf, uint8_t* desc, double* weight) {
    int k, L, n; const int32_t* p; const uint8_t *l, *d; const double* w;
    cubemap_b200::ExportVocabulary(static_cast<ORBVocabulary*>(voc), &k, &L, &n, &p, &l, &d, &w);
    std::memcpy(parent, p, (size_t)n * 4); std::memcpy(isLeaf, l, n); std::memcpy(desc, d, (size_t)n * 32); std::memcpy(weight, w, (size_t)n * 8);
}

// ComputeBoW (cpu = 0: the drop-in, 1: the reference's body) on a BowScene; outputs read back as BowScene::read (capacities n + 1)
void dropin_compute_bow(void* voc, int keyframe, int cpu, int n, const uint8_t* desc, int preset, int32_t* bowWord, double* bowVal, int32_t* nBow, int32_t* fvNode,
                        int32_t* fvStart, int32_t* fvFeat, int32_t* nFv) {
    BowScene s(static_cast<ORBVocabulary*>(voc), keyframe, n, desc, preset);
    s.run(cpu);
    s.read(bowWord, bowVal, nBow, fvNode, fvStart, fvFeat, nFv);
}

// nthreads host threads (even: a Frame, odd: a KeyFrame, like Tracking and LocalMapping) each run the drop-in ComputeBoW `reps` times on their own
// scene, concurrently; thread t's scene has descriptors desc + t*n*32, its results go to row t of every output (row length n + 1)
void dropin_compute_bow_threads(void* voc, int nthreads, int reps, int n, const uint8_t* desc, int32_t* bowWord, double* bowVal, int32_t* nBow, int32_t* fvNode,
                                int32_t* fvStart, int32_t* fvFeat, int32_t* nFv) {
    std::vector<BowScene*> scenes;
    for (int t = 0; t < nthreads; t++) scenes.push_back(new BowScene(static_cast<ORBVocabulary*>(voc), t & 1, n, desc + (size_t)t * n * 32, 0));
    std::vector<std::thread> th;
    for (int t = 0; t < nthreads; t++)
        th.push_back(std::thread([&scenes, t, reps]() { for (int r = 0; r < reps; r++) { scenes[t]->bow().clear(); scenes[t]->run(0); } }));
    for (size_t t = 0; t < th.size(); t++) th[t].join();
    const size_t row = (size_t)n + 1;
    for (int t = 0; t < nthreads; t++) {
        scenes[t]->read(bowWord + t * row, bowVal + t * row, nBow + t, fvNode + t * row, fvStart + t * row, fvFeat + t * row, nFv + t);
        delete scenes[t];
    }
}

// wall time of `reps` successive Frame::ComputeBoW calls (cpu: the reference's body) on one Frame, mBowVec cleared before each; ms[r] per call
void dropin_time_compute_bow(void* voc, int cpu, int n, const uint8_t* desc, int reps, double* ms) {
    BowScene s(static_cast<ORBVocabulary*>(voc), 0, n, desc, 0);
    for (int r = 0; r < reps; r++) {
        s.bow().clear();
        const std::chrono::steady_clock::time_point t0 = std::chrono::steady_clock::now();
        s.run(cpu);
        ms[r] = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
    }
}

}  // extern "C"

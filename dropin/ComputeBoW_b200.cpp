// Frame::ComputeBoW() and KeyFrame::ComputeBoW() (include/Frame.h:65, include/KeyFrame.h:64) on libcubemap_b200.so: the DBoW2 transform
// mpORBvocabulary->transform(descriptors, mBowVec, mFeatVec, 4) (src/Frame.cpp:719-726, src/KeyFrame.cpp:94-103) as one
// cslam_bow_transform_fv call. The reference's bodies stay in src/Frame.cpp / src/KeyFrame.cpp, renamed ComputeBoW_cpu
// (dropin/ComputeBoW_cpu_forward.cpp exports them for A/B runs).
//
// The vocabulary is copied from the loaded ORBVocabulary object, not re-read from ORBvoc.txt: the object is what the reference transforms with.
// (The loader's while(!f.eof()) loop turns the file's final newline into one more node, built from a failed stream: ORBvoc.txt lists 971 814
// leaves and the loaded object holds 971 815 words.) The copy is made once per process per ORBVocabulary*, under a mutex; each host thread that
// calls ComputeBoW (Tracking, LocalMapping) gets its own device handle holding the whole tree, like the other drop-ins' handles.
// A vocabulary the device transform does not model - scoring other than L1_NORM, weighting other than TF_IDF, 2^20 words or more, children not in
// ascending id order, a word with children or a childless node that is no word - is the drop-ins' loud failure (message + exit), never a CPU fallback.
#include "Frame.h"
#include "KeyFrame.h"
#include "ORBVocabulary.h"

#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <map>
#include <mutex>
#include <vector>

#include "cubemap_b200.h"

namespace {

void fatal(const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    std::fprintf(stderr, "ComputeBoW (cubemap_b200): ");
    std::vfprintf(stderr, fmt, ap);
    std::fprintf(stderr, "\n");
    va_end(ap);
    std::exit(EXIT_FAILURE);
}

// The loaded tree's protected members, named through a derived type's using-declarations: the pointers to member apply to the ORBVocabulary
// object itself, no cast of it.
struct VocMembers : ORBVocabulary {
    typedef ORBVocabulary::Node Node;
    using ORBVocabulary::m_nodes;
    using ORBVocabulary::m_words;
    using ORBVocabulary::m_k;
    using ORBVocabulary::m_L;
};
std::vector<VocMembers::Node> ORBVocabulary::* const kNodes = &VocMembers::m_nodes;
std::vector<VocMembers::Node*> ORBVocabulary::* const kWords = &VocMembers::m_words;
int ORBVocabulary::* const kK = &VocMembers::m_k;
int ORBVocabulary::* const kL = &VocMembers::m_L;

// nodes 1..n in id order, as cslam_vocabulary_create takes them
struct Imported {
    int k = 0, L = 0, n = 0;
    std::vector<int32_t> parent; std::vector<uint8_t> isLeaf, desc; std::vector<double> weight;
};

const Imported& import(const ORBVocabulary* voc) {
    static std::mutex mu;
    static std::map<const ORBVocabulary*, Imported*> done;
    std::lock_guard<std::mutex> lock(mu);
    Imported*& im = done[voc];
    if (im) return *im;
    if (voc->getScoringType() != DBoW2::L1_NORM) fatal("the vocabulary's scoring type %d is not L1_NORM", (int)voc->getScoringType());
    if (voc->getWeightingType() != DBoW2::TF_IDF) fatal("the vocabulary's weighting type %d is not TF_IDF", (int)voc->getWeightingType());
    const std::vector<VocMembers::Node>& nodes = voc->*kNodes;
    const std::vector<VocMembers::Node*>& words = voc->*kWords;
    if (words.size() >= (1u << 20)) fatal("the vocabulary has %zu words; the device transform holds word ids < 2^20", words.size());
    Imported* out = new Imported;
    const int n = (int)nodes.size() - 1;
    out->k = voc->*kK; out->L = voc->*kL; out->n = n;
    out->parent.resize(n); out->isLeaf.assign(n, 0); out->desc.resize((size_t)n * 32); out->weight.resize(n);
    // word membership from m_words; the device numbers words in node-id order, so m_words must list them in that order
    long prev = 0;
    for (size_t w = 0; w < words.size(); w++) {
        const long id = words[w] - nodes.data();
        if (id < 1 || id > n || &nodes[id] != words[w]) fatal("word %zu does not point into the vocabulary's nodes", w);
        if (id <= prev || nodes[id].word_id != (DBoW2::WordId)w) fatal("word %zu (node %ld) is not numbered in node order", w, id);
        out->isLeaf[id - 1] = 1; prev = id;
    }
    size_t nChildren = 0;
    for (int i = 0; i <= n; i++) {
        const std::vector<DBoW2::NodeId>& c = nodes[i].children;
        for (size_t j = 0; j < c.size(); j++)
            if ((int)c[j] <= i || (int)c[j] > n || nodes[c[j]].parent != (DBoW2::NodeId)i || (j > 0 && c[j] <= c[j - 1]))
                fatal("children of node %d are not in ascending id order or do not name it as parent", i);
        nChildren += c.size();
        if (i == 0) continue;
        if (c.empty() != (out->isLeaf[i - 1] != 0)) fatal("node %d: %s", i, c.empty() ? "childless but no word" : "a word with children");
        const cv::Mat& d = nodes[i].descriptor;
        if (d.rows != 1 || d.cols != 32 || d.type() != CV_8U) fatal("node %d: the descriptor is not 1 x 32 bytes", i);
        std::memcpy(&out->desc[(size_t)(i - 1) * 32], d.ptr<uchar>(0), 32);
        out->parent[i - 1] = (int32_t)nodes[i].parent;
        out->weight[i - 1] = nodes[i].weight;
    }
    if (nChildren != (size_t)n) fatal("the vocabulary's children lists hold %zu nodes, not %d", nChildren, n);
    im = out;
    return *im;
}

cslam_vocabulary* handle(const ORBVocabulary* voc) {
    static thread_local std::map<const ORBVocabulary*, cslam_vocabulary*> handles;
    cslam_vocabulary*& h = handles[voc];
    if (!h) {
        const Imported& im = import(voc);
        // max_features 4096: the handle's first staging chunk holds a call at stride <= 2048; larger strides add chunks that later calls reuse
        if (cslam_vocabulary_create(&h, 0, im.k, im.L, im.n, im.parent.data(), im.isLeaf.data(), im.desc.data(), im.weight.data(), 1, 4096) != CSLAM_OK)
            fatal("%s", cslam_last_error());
    }
    return h;
}

// ORBVocabulary::transform(descriptors, bow, fv, 4): both vectors cleared, then filled in map order with end hints
void transform(const ORBVocabulary* voc, const cv::Mat& D, DBoW2::BowVector& bow, DBoW2::FeatureVector& fv) {
    bow.clear(); fv.clear();
    if (voc->empty() || D.rows == 0) return;     // TemplatedVocabulary::transform returns empty vectors for an empty vocabulary or no features
    const int n = D.rows;
    if (n > CSLAM_BOW_FV_MAX_FEATURES) fatal("%d features in one frame; the device transform takes at most %d", n, CSLAM_BOW_FV_MAX_FEATURES);
    if (D.cols != 32 || D.type() != CV_8U) fatal("descriptors must be N x 32 bytes");
    cslam_vocabulary* h = handle(voc);
    // the stride is a power of two >= 1024: a handle sees at most five call shapes, so its staging stops growing after the first few calls
    int stride = 1024;
    while (stride < n) stride <<= 1;
    static thread_local std::vector<uint8_t> desc;
    static thread_local std::vector<int32_t> bw, fn, fs, ff;
    static thread_local std::vector<double> bv;
    desc.resize((size_t)stride * 32); bw.resize(stride); bv.resize(stride); fn.resize(stride); fs.resize(stride + 1); ff.resize(stride);
    for (int i = 0; i < n; i++) std::memcpy(&desc[(size_t)i * 32], D.ptr<uchar>(i), 32);
    int32_t nn = n, nb = 0, nf = 0;
    if (cslam_bow_transform_fv(h, desc.data(), &nn, stride, 1, 4, bw.data(), bv.data(), &nb, fn.data(), fs.data(), ff.data(), &nf) != CSLAM_OK)
        fatal("%s", cslam_last_error());
    for (int j = 0; j < nb; j++) bow.insert(bow.end(), DBoW2::BowVector::value_type((DBoW2::WordId)bw[j], bv[j]));
    for (int j = 0; j < nf; j++)
        fv.insert(fv.end(), DBoW2::FeatureVector::value_type((DBoW2::NodeId)fn[j], std::vector<unsigned int>(ff.begin() + fs[j], ff.begin() + fs[j + 1])));
}

}  // namespace

namespace cubemap_b200 {
// The arrays the drop-in uploads for `voc` (nodes 1..n_nodes: parent, word flag, 32 descriptor bytes, weight), valid while the process runs
void ExportVocabulary(const ORBVocabulary* voc, int* k, int* L, int* n_nodes, const int32_t** parent, const uint8_t** is_leaf, const uint8_t** desc, const double** weight) {
    const Imported& im = import(voc);
    *k = im.k; *L = im.L; *n_nodes = im.n; *parent = im.parent.data(); *is_leaf = im.isLeaf.data(); *desc = im.desc.data(); *weight = im.weight.data();
}
}  // namespace cubemap_b200

void Frame::ComputeBoW() {
    if (mBowVec.empty()) transform(mpORBvocabulary, mDescriptors, mBowVec, mFeatVec);
}

void KeyFrame::ComputeBoW() {
    if (mBowVec.empty() || mFeatVec.empty()) transform(mpORBvocabulary, mDescriptors, mBowVec, mFeatVec);
}

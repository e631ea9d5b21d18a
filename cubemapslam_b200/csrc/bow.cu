// DBoW2 vocabulary-tree transform of libcubemap_b200.so (SURVEY 8(f) row 2), sm_90a.
//
// Reference (CPU): Frame::ComputeBoW / KeyFrame::ComputeBoW (src/Frame.cpp:719-726) -> TemplatedVocabulary::transform(features, BowVector&, FeatureVector&, 4)
//   ThirdParty/DBoW2/DBoW2/TemplatedVocabulary.h:1127-1193 (per feature :1218-1262: greedy descent, first minimum wins; FORB::distance is hamming256 in orb_match.cuh),
//   BowVector::addWeight / normalize(L1) BowVector.cpp:31-45,62-85. ORBvoc.txt is k = 10, L = 6, L1_NORM scoring, TF_IDF weighting.
//
// k_bow_descend   thread per feature: L levels x k children, 256-bit Hamming against node descriptors (35 MB for the full vocabulary: L2-resident);
//                 output word id, leaf node, FeatureVector node (level L - levelsup)
// k_bow_vector    CTA per frame: the BowVector std::map restated as sort by (word, feature index) + in-order segment sums (double, the order
//                 addWeight sees) + the L1 normalisation summed in word order like BowVector::normalize -> bit-identical doubles
// k_bow_vector_fv CTA of 1024 threads per frame, up to 16384 features (the initialisation extractor's key frames reach 3*nFeatures + 3*nlevels,
//                 9024 at 3000 features): the BowVector as k_bow_vector builds it, then the FeatureVector (std::map<NodeId, std::vector<unsigned>>)
//                 as a second sort of the same live features by (node, feature index), written as CSR: node ascending, indices ascending.
//                 Keys are 64-bit, id << 14 | index: a word id needs 20 bits and an index 14, one more than the 32-bit keys of k_bow_vector hold.
//                 One CTA per frame keeps both sorts and every segment on chip: 16384 keys x 8 B + 16384 ranks x 4 B = 192 KB of shared
//                 memory, inside the 227 KB an sm_90 CTA may use, and no cross-CTA merge. A call is two launches (k_bow_descend, k_bow_vector_fv)
//                 whatever the number of frames.
#include <cstring>
#include <vector>
#include "common.cuh"
#include "orb_match.cuh"

namespace cslam {

struct VocDev { int k, L, nNodes; const int* childStart; const int* childList; const uint4* desc; const double* weight; const int* wordId; };

__global__ void __launch_bounds__(128) k_bow_descend(VocDev V, const uint8_t* __restrict__ feats, const int32_t* __restrict__ n, int stride, int levelsup,
                                                      int32_t* __restrict__ word, int32_t* __restrict__ leaf, int32_t* __restrict__ node) {
    const int f = blockIdx.y, i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= min(n[f], stride)) return;
    const uint4* F4 = reinterpret_cast<const uint4*>(feats + ((size_t)f * stride + i) * 32);
    const uint4 a0 = __ldg(F4), a1 = __ldg(F4 + 1);
    const int nidLevel = V.L - levelsup;
    int fin = 0, level = 0, nid = 0;
    do {
        ++level;
        const int s = V.childStart[fin], e = V.childStart[fin + 1];
        int best = 0x7fffffff, bestId = V.childList[s];
        for (int c = s; c < e; c++) {
            const int id = V.childList[c];
            const uint4 b0 = __ldg(V.desc + 2 * (size_t)id), b1 = __ldg(V.desc + 2 * (size_t)id + 1);
            const int d = hamming256(a0, a1, b0, b1);
            if (d < best) { best = d; bestId = id; }
        }
        fin = bestId;
        if (level == nidLevel) nid = fin;
    } while (V.childStart[fin + 1] > V.childStart[fin]);
    const size_t o = (size_t)f * stride + i;
    word[o] = V.wordId[fin]; leaf[o] = fin; node[o] = V.weight[fin] > 0 ? nid : -1;   // stopped words (weight 0) join neither vector
}

// keys: word << 12 | feature index (index < 4096, word < 2^20)
__global__ void __launch_bounds__(256) k_bow_vector(VocDev V, const int32_t* __restrict__ n, int stride, int n2, const int32_t* __restrict__ word, const int32_t* __restrict__ leaf,
                                                    const int32_t* __restrict__ node, int32_t* __restrict__ bowWord, double* __restrict__ bowVal, int32_t* __restrict__ bowCount) {
    extern __shared__ uint32_t key[];           // n2 keys, then n2 flags / ranks
    uint32_t* rank = key + n2;
    __shared__ uint32_t wsum[8], carry;
    __shared__ double norm;
    const int f = blockIdx.x, tid = threadIdx.x, nf = min(n[f], stride);
    const size_t o = (size_t)f * stride;
    for (int i = tid; i < n2; i += 256) key[i] = (i < nf && node[o + i] >= 0) ? ((uint32_t)word[o + i] << 12) | (uint32_t)i : 0xffffffffu;
    __syncthreads();
    block_bitonic_sort(key, n2);
    // segment starts -> output rank (exclusive scan of the start flags)
    if (tid == 0) carry = 0;
    __syncthreads();
    for (int base = 0; base < n2; base += 256) {
        const int p = base + tid;
        const uint32_t x = (p < n2 && key[p] != 0xffffffffu && (p == 0 || (key[p - 1] >> 12) != (key[p] >> 12))) ? 1u : 0u;
        uint32_t s = x;
#pragma unroll
        for (int sh = 1; sh < 32; sh <<= 1) { const uint32_t t = __shfl_up_sync(0xffffffffu, s, sh); if ((tid & 31) >= sh) s += t; }
        if ((tid & 31) == 31) wsum[tid >> 5] = s;
        __syncthreads();
        uint32_t pre = carry;
        for (int w = 0; w < (tid >> 5); w++) pre += wsum[w];
        if (p < n2) rank[p] = x ? pre + s - 1 : 0xffffffffu;
        __syncthreads();
        if (tid == 255) carry = pre + s;
        __syncthreads();
    }
    const int nWords = (int)carry;
    // in-order segment sums: v[word] += weight, feature by feature (BowVector::addWeight)
    for (int p = tid; p < n2; p += 256) {
        if (rank[p] == 0xffffffffu) continue;
        const uint32_t w = key[p] >> 12;
        double s = 0;
        for (int q = p; q < n2 && key[q] != 0xffffffffu && (key[q] >> 12) == w; q++) s += V.weight[leaf[o + (key[q] & 0xfff)]];
        bowWord[o + rank[p]] = (int32_t)w; bowVal[o + rank[p]] = s;
    }
    __syncthreads();
    if (tid == 0) {   // BowVector::normalize(L1): norm += fabs(value) in word order
        double s = 0;
        for (int i = 0; i < nWords; i++) s += fabs(bowVal[o + i]);
        norm = s; bowCount[f] = nWords;
    }
    __syncthreads();
    if (norm > 0.0) for (int i = tid; i < nWords; i += 256) bowVal[o + i] = bowVal[o + i] / norm;
}

// exclusive scan of the segment starts of the sorted keys (segment = key >> FV_IDX_BITS; all-ones keys are dead and sort last): rank[p] = output
// slot of the segment starting at p, all-ones elsewhere. Returns the number of segments. blockDim.x = 1024.
constexpr int FV_IDX_BITS = 14;
constexpr unsigned long long FV_DEAD = ~0ull;
__device__ int fv_segment_ranks(const unsigned long long* key, uint32_t* rank, int n2, uint32_t* wsum, uint32_t& carry) {
    const int tid = threadIdx.x;
    if (tid == 0) carry = 0;
    __syncthreads();
    for (int base = 0; base < n2; base += 1024) {
        const int p = base + tid;
        const uint32_t x = (p < n2 && key[p] != FV_DEAD && (p == 0 || (key[p - 1] >> FV_IDX_BITS) != (key[p] >> FV_IDX_BITS))) ? 1u : 0u;
        uint32_t s = x;
#pragma unroll
        for (int sh = 1; sh < 32; sh <<= 1) { const uint32_t t = __shfl_up_sync(0xffffffffu, s, sh); if ((tid & 31) >= sh) s += t; }
        if ((tid & 31) == 31) wsum[tid >> 5] = s;
        __syncthreads();
        uint32_t pre = carry;
        for (int w = 0; w < (tid >> 5); w++) pre += wsum[w];
        if (p < n2) rank[p] = x ? pre + s - 1 : 0xffffffffu;
        __syncthreads();
        if (tid == 1023) carry = pre + s;
        __syncthreads();
    }
    return (int)carry;
}

// BowVector + FeatureVector of frames of up to 16384 features from k_bow_descend's word / leaf / node. Per frame f: bow_word / bow_val at
// f*stride (bowCount[f] entries), fv_node at f*stride (fvCount[f] nodes), fv_start at f*(stride+1) (fvCount[f] + 1 offsets into fv_feat),
// fv_feat at f*stride (the live features, grouped by node).
__global__ void __launch_bounds__(1024) k_bow_vector_fv(VocDev V, const int32_t* __restrict__ n, int stride, int n2, const int32_t* __restrict__ word,
                                                        const int32_t* __restrict__ leaf, const int32_t* __restrict__ node, int32_t* __restrict__ bowWord,
                                                        double* __restrict__ bowVal, int32_t* __restrict__ bowCount, int32_t* __restrict__ fvNode,
                                                        int32_t* __restrict__ fvStart, int32_t* __restrict__ fvFeat, int32_t* __restrict__ fvCount) {
    extern __shared__ unsigned long long key64[];   // n2 keys, then n2 ranks
    uint32_t* rank = reinterpret_cast<uint32_t*>(key64 + n2);
    __shared__ uint32_t wsum[32], carry;
    __shared__ double norm;
    const int f = blockIdx.x, tid = threadIdx.x, nf = min(n[f], stride);
    const size_t o = (size_t)f * stride, os = (size_t)f * (stride + 1);
    // 1. BowVector: sort by (word, index); stopped words (node -1) are dead keys
    for (int i = tid; i < n2; i += 1024)
        key64[i] = (i < nf && node[o + i] >= 0) ? ((unsigned long long)(uint32_t)word[o + i] << FV_IDX_BITS) | (unsigned)i : FV_DEAD;
    __syncthreads();
    block_bitonic_sort(key64, n2);
    const int nWords = fv_segment_ranks(key64, rank, n2, wsum, carry);
    // in-order segment sums, feature by feature (BowVector::addWeight); a word is one leaf, so every addend of a segment is that leaf's weight
    for (int p = tid; p < n2; p += 1024) {
        if (rank[p] == 0xffffffffu) continue;
        const unsigned long long w = key64[p] >> FV_IDX_BITS;
        const double wt = V.weight[leaf[o + (key64[p] & ((1u << FV_IDX_BITS) - 1))]];
        double s = 0;
        for (int q = p; q < n2 && key64[q] != FV_DEAD && (key64[q] >> FV_IDX_BITS) == w; q++) s += wt;
        bowWord[o + rank[p]] = (int32_t)w; bowVal[o + rank[p]] = s;
    }
    __syncthreads();
    if (tid == 0) {   // BowVector::normalize(L1): norm += fabs(value) in word order
        double s = 0;
        for (int i = 0; i < nWords; i++) s += fabs(bowVal[o + i]);
        norm = s; bowCount[f] = nWords;
    }
    __syncthreads();
    if (norm > 0.0) for (int i = tid; i < nWords; i += 1024) bowVal[o + i] = bowVal[o + i] / norm;
    // 2. FeatureVector: the same live features sorted by (node, index) -> CSR
    for (int i = tid; i < n2; i += 1024)
        key64[i] = (i < nf && node[o + i] >= 0) ? ((unsigned long long)(uint32_t)node[o + i] << FV_IDX_BITS) | (unsigned)i : FV_DEAD;
    __syncthreads();
    block_bitonic_sort(key64, n2);
    const int nNodes = fv_segment_ranks(key64, rank, n2, wsum, carry);
    for (int p = tid; p < n2; p += 1024) {
        const unsigned long long kp = key64[p];
        if (kp == FV_DEAD) continue;
        fvFeat[o + p] = (int32_t)(kp & ((1u << FV_IDX_BITS) - 1));
        if (rank[p] != 0xffffffffu) { fvNode[o + rank[p]] = (int32_t)(kp >> FV_IDX_BITS); fvStart[os + rank[p]] = p; }
        if (p + 1 == n2 || key64[p + 1] == FV_DEAD) fvStart[os + nNodes] = p + 1;   // the last live feature closes the last node
    }
    if (tid == 0) { fvCount[f] = nNodes; if (nNodes == 0) fvStart[os] = 0; }
}

}  // namespace cslam

using namespace cslam;

// arena: staging of cslam_bow_transform
struct cslam_vocabulary : cslam::Handle {
    VocDev V; int maxFrames = 0, maxFeat = 0;
};

extern "C" void cslam_vocabulary_destroy(cslam_vocabulary* v) { destroy_handle(v); }

// nodes 1..n_nodes in ORBvoc.txt's order (TemplatedVocabulary::loadFromTextFile :1337-1415): parent id, leaf flag, 32 descriptor bytes, weight
extern "C" int cslam_vocabulary_create(cslam_vocabulary** out, int device, int k, int L, int n_nodes, const int32_t* parent, const uint8_t* is_leaf, const uint8_t* desc,
                                       const double* weight, int max_frames, int max_features) {
    if (!out || k < 2 || L < 1 || n_nodes <= 0 || !parent || !is_leaf || !desc || !weight || max_frames <= 0 || max_features <= 0 || max_features > 4096) { set_error("cslam_vocabulary_create: bad argument"); return CSLAM_E_BADARG; }
    cslam_vocabulary* v = new cslam_vocabulary; v->maxFrames = max_frames; v->maxFeat = max_features;
    auto fail = [&](int code) { destroy_handle(v); return code; };
    // chunks: room for the descriptors, four int32 arrays and the double weights of a call at the handle's limits, at most 64 MB
    int rc = v->open(device, std::min<size_t>((size_t)64 << 20, (size_t)max_frames * max_features * (32 + 4 * 4 + 8) + (size_t)max_frames * 8), false);
    if (rc) return fail(rc);
    const int N = n_nodes + 1;
    std::vector<int> cnt(N + 1, 0), wordId(N, -1);
    int words = 0;
    for (int i = 0; i < n_nodes; i++) {
        if (parent[i] < 0 || parent[i] > i) { set_error("vocabulary node %d: parent %d must precede it", i + 1, parent[i]); return fail(CSLAM_E_BADARG); }
        cnt[parent[i] + 1]++;
        if (is_leaf[i]) wordId[i + 1] = words++;
    }
    if (words >= (1 << 20)) { set_error("vocabulary has %d words; the packed sort keys hold word ids < 2^20", words); return fail(CSLAM_E_BADARG); }
    for (int i = 0; i < N; i++) cnt[i + 1] += cnt[i];
    std::vector<int> start(cnt), fill(cnt.begin(), cnt.end() - 1), list(n_nodes);
    for (int i = 0; i < n_nodes; i++) list[fill[parent[i]]++] = i + 1;       // children in file order (push_back order)
    std::vector<uint8_t> d((size_t)N * 32, 0); std::vector<double> w(N, 0.0);
    std::memcpy(d.data() + 32, desc, (size_t)n_nodes * 32);
    std::memcpy(w.data() + 1, weight, (size_t)n_nodes * 8);
    int *dStart, *dList, *dWid; uint4* dDesc; double* dW;
    auto valloc = [&](auto** p, size_t n) { return dev_alloc(v->owned, p, n, false); };
    if ((rc = valloc(&dStart, N + 1)) || (rc = valloc(&dList, n_nodes)) || (rc = valloc(&dWid, N)) || (rc = valloc(&dDesc, (size_t)N * 2)) || (rc = valloc(&dW, N))) return fail(rc);
    if (cudaMemcpy(dStart, start.data(), (N + 1) * 4, cudaMemcpyHostToDevice) != cudaSuccess || cudaMemcpy(dList, list.data(), (size_t)n_nodes * 4, cudaMemcpyHostToDevice) != cudaSuccess ||
        cudaMemcpy(dWid, wordId.data(), N * 4, cudaMemcpyHostToDevice) != cudaSuccess || cudaMemcpy(dDesc, d.data(), (size_t)N * 32, cudaMemcpyHostToDevice) != cudaSuccess ||
        cudaMemcpy(dW, w.data(), (size_t)N * 8, cudaMemcpyHostToDevice) != cudaSuccess) { set_error("vocabulary upload failed"); return fail(CSLAM_E_CUDA); }
    v->V.k = k; v->V.L = L; v->V.nNodes = N; v->V.childStart = dStart; v->V.childList = dList; v->V.desc = dDesc; v->V.weight = dW; v->V.wordId = dWid;
    cudaFuncSetAttribute(k_bow_vector, cudaFuncAttributeMaxDynamicSharedMemorySize, 2 * 4096 * 4);
    cudaFuncSetAttribute(k_bow_vector_fv, cudaFuncAttributeMaxDynamicSharedMemorySize, CSLAM_BOW_FV_MAX_FEATURES * 12);
    *out = v;
    return CSLAM_OK;
}
extern "C" void* cslam_vocabulary_stream(const cslam_vocabulary* v) { return v ? (void*)v->stream : nullptr; }
extern "C" int cslam_vocabulary_sync(cslam_vocabulary* v) { return v ? v->sync() : CSLAM_E_BADARG; }

extern "C" int cslam_bow_transform_dev(cslam_vocabulary* v, const uint8_t* desc, const int32_t* n, int stride, int nframes, int levelsup, int32_t* word, int32_t* leaf, int32_t* node,
                                       int32_t* bow_word, double* bow_val, int32_t* bow_count) {
    if (!v || !desc || !n || !word || !leaf || !node || !bow_word || !bow_val || !bow_count || nframes <= 0 || stride <= 0 || stride > 4096) { set_error("cslam_bow_transform_dev: bad argument"); return CSLAM_E_BADARG; }
    CSLAM_CUDA(cudaSetDevice(v->device));
    k_bow_descend<<<dim3(cdiv(stride, 128), nframes), 128, 0, v->stream>>>(v->V, desc, n, stride, levelsup, word, leaf, node);
    const int n2 = pow2_at_least(stride);
    k_bow_vector<<<nframes, 256, (size_t)2 * n2 * 4, v->stream>>>(v->V, n, stride, n2, word, leaf, node, bow_word, bow_val, bow_count);
    v->launches += 2;
    CSLAM_CUDA(cudaGetLastError());
    return CSLAM_OK;
}

extern "C" int cslam_bow_transform(cslam_vocabulary* v, const uint8_t* desc, const int32_t* n, int stride, int nframes, int levelsup, int32_t* word, int32_t* node, int32_t* bow_word,
                                   double* bow_val, int32_t* bow_count) {
    if (!v || nframes <= 0 || nframes > v->maxFrames || stride <= 0 || stride > v->maxFeat) { set_error("cslam_bow_transform: sizes out of range"); return CSLAM_E_BADARG; }
    CSLAM_CUDA(cudaSetDevice(v->device));
    v->arena.reset();
    const size_t nf = (size_t)nframes * stride;
    const uint8_t* dFeat; const int32_t* dN; int32_t *dWord, *dLeaf, *dNode, *dBowWord, *dBowCount; double* dBowVal; int rc;
    if ((rc = v->arena.upload(&dFeat, desc, nf * 32)) || (rc = v->arena.upload(&dN, n, nframes)) || (rc = v->arena.take(&dWord, nf)) || (rc = v->arena.take(&dLeaf, nf)) ||
        (rc = v->arena.take(&dNode, nf)) || (rc = v->arena.take(&dBowWord, nf)) || (rc = v->arena.take(&dBowVal, nf)) || (rc = v->arena.take(&dBowCount, nframes)) ||
        (rc = cslam_bow_transform_dev(v, dFeat, dN, stride, nframes, levelsup, dWord, dLeaf, dNode, dBowWord, dBowVal, dBowCount))) return rc;
    if (word) CSLAM_CUDA(cudaMemcpyAsync(word, dWord, nf * 4, cudaMemcpyDeviceToHost, v->stream));
    CSLAM_CUDA(cudaMemcpyAsync(node, dNode, nf * 4, cudaMemcpyDeviceToHost, v->stream));
    CSLAM_CUDA(cudaMemcpyAsync(bow_word, dBowWord, nf * 4, cudaMemcpyDeviceToHost, v->stream));
    CSLAM_CUDA(cudaMemcpyAsync(bow_val, dBowVal, nf * 8, cudaMemcpyDeviceToHost, v->stream));
    CSLAM_CUDA(cudaMemcpyAsync(bow_count, dBowCount, (size_t)nframes * 4, cudaMemcpyDeviceToHost, v->stream));
    return v->sync();
}

extern "C" int cslam_bow_transform_fv_dev(cslam_vocabulary* v, const uint8_t* desc, const int32_t* n, int stride, int nframes, int levelsup, int32_t* word, int32_t* leaf,
                                          int32_t* node, int32_t* bow_word, double* bow_val, int32_t* bow_count, int32_t* fv_node, int32_t* fv_start, int32_t* fv_feat,
                                          int32_t* fv_count) {
    if (!v || !desc || !n || !word || !leaf || !node || !bow_word || !bow_val || !bow_count || !fv_node || !fv_start || !fv_feat || !fv_count || nframes <= 0 || stride <= 0 ||
        stride > CSLAM_BOW_FV_MAX_FEATURES) { set_error("cslam_bow_transform_fv_dev: bad argument (stride must be in [1, %d])", CSLAM_BOW_FV_MAX_FEATURES); return CSLAM_E_BADARG; }
    CSLAM_CUDA(cudaSetDevice(v->device));
    k_bow_descend<<<dim3(cdiv(stride, 128), nframes), 128, 0, v->stream>>>(v->V, desc, n, stride, levelsup, word, leaf, node);
    const int n2 = pow2_at_least(stride);
    k_bow_vector_fv<<<nframes, 1024, (size_t)n2 * 12, v->stream>>>(v->V, n, stride, n2, word, leaf, node, bow_word, bow_val, bow_count, fv_node, fv_start, fv_feat, fv_count);
    v->launches += 2;
    CSLAM_CUDA(cudaGetLastError());
    return CSLAM_OK;
}

extern "C" int cslam_bow_transform_fv(cslam_vocabulary* v, const uint8_t* desc, const int32_t* n, int stride, int nframes, int levelsup, int32_t* bow_word, double* bow_val,
                                      int32_t* bow_count, int32_t* fv_node, int32_t* fv_start, int32_t* fv_feat, int32_t* fv_count) {
    if (!v || !desc || !n || !bow_word || !bow_val || !bow_count || !fv_node || !fv_start || !fv_feat || !fv_count || nframes <= 0 || nframes > v->maxFrames || stride <= 0 ||
        stride > CSLAM_BOW_FV_MAX_FEATURES) {
        set_error("cslam_bow_transform_fv: bad argument (nframes must be in [1, max_frames], stride in [1, %d])", CSLAM_BOW_FV_MAX_FEATURES); return CSLAM_E_BADARG;
    }
    CSLAM_CUDA(cudaSetDevice(v->device));
    v->arena.reset();
    const size_t nf = (size_t)nframes * stride, ns = (size_t)nframes * (stride + 1);
    const uint8_t* dFeat; const int32_t* dN; int32_t *dWord, *dLeaf, *dNode, *dBowWord, *dBowCount, *dFvNode, *dFvStart, *dFvFeat, *dFvCount; double* dBowVal; int rc;
    if ((rc = v->arena.upload(&dFeat, desc, nf * 32)) || (rc = v->arena.upload(&dN, n, nframes)) || (rc = v->arena.take(&dWord, nf)) || (rc = v->arena.take(&dLeaf, nf)) ||
        (rc = v->arena.take(&dNode, nf)) || (rc = v->arena.take(&dBowWord, nf)) || (rc = v->arena.take(&dBowVal, nf)) || (rc = v->arena.take(&dBowCount, nframes)) ||
        (rc = v->arena.take(&dFvNode, nf)) || (rc = v->arena.take(&dFvStart, ns)) || (rc = v->arena.take(&dFvFeat, nf)) || (rc = v->arena.take(&dFvCount, nframes)) ||
        (rc = cslam_bow_transform_fv_dev(v, dFeat, dN, stride, nframes, levelsup, dWord, dLeaf, dNode, dBowWord, dBowVal, dBowCount, dFvNode, dFvStart, dFvFeat, dFvCount)))
        return rc;
    CSLAM_CUDA(cudaMemcpyAsync(bow_word, dBowWord, nf * 4, cudaMemcpyDeviceToHost, v->stream));
    CSLAM_CUDA(cudaMemcpyAsync(bow_val, dBowVal, nf * 8, cudaMemcpyDeviceToHost, v->stream));
    CSLAM_CUDA(cudaMemcpyAsync(bow_count, dBowCount, (size_t)nframes * 4, cudaMemcpyDeviceToHost, v->stream));
    CSLAM_CUDA(cudaMemcpyAsync(fv_node, dFvNode, nf * 4, cudaMemcpyDeviceToHost, v->stream));
    CSLAM_CUDA(cudaMemcpyAsync(fv_start, dFvStart, ns * 4, cudaMemcpyDeviceToHost, v->stream));
    CSLAM_CUDA(cudaMemcpyAsync(fv_feat, dFvFeat, nf * 4, cudaMemcpyDeviceToHost, v->stream));
    CSLAM_CUDA(cudaMemcpyAsync(fv_count, dFvCount, (size_t)nframes * 4, cudaMemcpyDeviceToHost, v->stream));
    return v->sync();
}

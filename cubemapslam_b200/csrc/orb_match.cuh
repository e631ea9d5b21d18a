// Device-side ORB-matching rules shared by the matcher kernels (match.cu, track.cu, mapping.cu, bow.cu): one definition each, so the
// reference's exact rounding and tie-breaking live in one place.
#pragma once
#include <algorithm>
#include <cstdint>
#include <vector>

namespace cslam {

static const int HISTO_BINS = 30;   // ceil(360 / HISTO_LENGTH), HISTO_LENGTH = 12 (src/ORBMatcher.cpp:44)

// ORBMatcher::DescriptorDistance src/ORBMatcher.cpp:951-967 (SWAR popcount of 8 x 32-bit XOR) = FORB::distance
// ThirdParty/DBoW2/DBoW2/FORB.cpp:81-101: 256-bit Hamming distance of two descriptors held as two uint4 each
__device__ __forceinline__ int hamming256(const uint4 a0, const uint4 a1, const uint4 b0, const uint4 b1) {
    return __popc(a0.x ^ b0.x) + __popc(a0.y ^ b0.y) + __popc(a0.z ^ b0.z) + __popc(a0.w ^ b0.w) + __popc(a1.x ^ b1.x) + __popc(a1.y ^ b1.y) + __popc(a1.z ^ b1.z) +
           __popc(a1.w ^ b1.w);
}

// Rotation-histogram bin of a match (e.g. src/ORBMatcher.cpp:488-493): rot = angle a - angle b, wrapped into [0, 360), times 1/12 in float,
// C round() (half away from zero); bin 30 is bin 0
__device__ __forceinline__ int rot_bin(float a, float b) {
    const float factor = 1.0f / 12.0f;
    float rot = __fsub_rn(a, b);
    if (rot < 0.0f) rot = __fadd_rn(rot, 360.0f);
    int bin = (int)roundf(__fmul_rn(rot, factor));
    if (bin == HISTO_BINS) bin = 0;
    return bin;
}

// ComputeThreeMaxima src/ORBMatcher.cpp:905-946 on bin counts (one thread); keep[] = 1 for the bins that survive. The first of equal
// counts wins, and the second / third maxima are dropped below 0.1 * max1 in float.
__device__ __forceinline__ void three_maxima(const int* hist, int* keep) {
    int max1 = 0, max2 = 0, max3 = 0, ind1 = -1, ind2 = -1, ind3 = -1;
    for (int i = 0; i < HISTO_BINS; i++) {
        const int s = hist[i];
        if (s > max1) { max3 = max2; max2 = max1; max1 = s; ind3 = ind2; ind2 = ind1; ind1 = i; }
        else if (s > max2) { max3 = max2; max2 = s; ind3 = ind2; ind2 = i; }
        else if (s > max3) { max3 = s; ind3 = i; }
    }
    if ((float)max2 < __fmul_rn(0.1f, (float)max1)) { ind2 = -1; ind3 = -1; }
    else if ((float)max3 < __fmul_rn(0.1f, (float)max1)) { ind3 = -1; }
    for (int i = 0; i < HISTO_BINS; i++) keep[i] = (i == ind1 || i == ind2 || i == ind3);
}

// Block-wide ascending bitonic sort of n2 unsigned keys (u32 or u64) in shared memory, n2 a power of two; every thread of the block calls it
template <class K>
__device__ inline void block_bitonic_sort(K* key, int n2) {
    for (int k = 2; k <= n2; k <<= 1)
        for (int j = k >> 1; j > 0; j >>= 1) {
            for (int t = threadIdx.x; t < n2; t += blockDim.x) {
                const int ixj = t ^ j;
                if (ixj > t) {
                    const K a = key[t], b = key[ixj];
                    const bool up = (t & k) == 0;
                    if ((a > b) == up) { key[t] = b; key[ixj] = a; }
                }
            }
            __syncthreads();
        }
}

// A FeatureVector (DBoW2 node -> feature indices in ascending order) rebuilt as sorted keys node << 12 | index: the first position of `node`
// among key[0, n), or the position where it would be
__device__ __forceinline__ int node_lower_bound(const uint32_t* key, int n, uint32_t node) {
    const uint32_t target = node << 12;
    int lo = 0, hi = n;
    while (lo < hi) { const int mid = (lo + hi) >> 1; if (key[mid] < target) lo = mid + 1; else hi = mid; }
    return lo;
}

// SearchByBoW's candidate scan (src/ORBMatcher.cpp:455-475): feature at list position p with distance d against the running (best1, best2,
// position of best1). Strict `<`, so of equal distances the first position scanned wins; a lane scans its positions in increasing order.
__device__ __forceinline__ void bow_take(int d, int p, int& best1, int& best2, int& bpos) {
    if (d < best1) { best2 = best1; best1 = d; bpos = p; }
    else if (d < best2) best2 = d;
}
// Merges the 32 lanes' partial scans: the winner is the smaller distance, ties go to the earlier list position. Every lane ends with the result.
__device__ __forceinline__ void bow_warp_merge(int& best1, int& best2, int& bpos) {
#pragma unroll
    for (int o = 16; o; o >>= 1) {
        const int ob1 = __shfl_xor_sync(0xffffffffu, best1, o), ob2 = __shfl_xor_sync(0xffffffffu, best2, o), op = __shfl_xor_sync(0xffffffffu, bpos, o);
        const bool otherWins = ob1 < best1 || (ob1 == best1 && op < bpos);
        if (otherWins) { best2 = min(best1, ob2); best1 = ob1; bpos = op; }
        else best2 = min(best2, ob1);
    }
}
// SearchByBoW's acceptance: TH_LOW = 50 with `<=` for (KeyFrame, Frame) (:477) and `<` for (KeyFrame, KeyFrame) (:619), then the ratio test in float
__device__ __forceinline__ bool bow_accept(int best1, int best2, float nnratio, bool strictThLow) {
    return (strictThLow ? best1 < 50 : best1 <= 50) && (float)best1 < __fmul_rn(nnratio, (float)best2);
}

// A FeatureVector given as a CSR (cslam_bow_transform_fv's layout: nodes strictly ascending): the position of `node` among node[0, count),
// or -1 when the FeatureVector does not hold it
__device__ __forceinline__ int fv_find(const int32_t* __restrict__ node, int count, int32_t target) {
    int lo = 0, hi = count;
    while (lo < hi) { const int mid = (lo + hi) >> 1; if (__ldg(node + mid) < target) lo = mid + 1; else hi = mid; }
    return lo < count && __ldg(node + lo) == target ? lo : -1;
}

// Host check of `npairs` FeatureVectors in that CSR layout, pair p at node / feat + p*stride, start + p*(stride+1), with n[p] features (clamped
// to stride) and count[p] nodes. Returns nullptr, or what is wrong with pair *bad. Each feature may sit in one node only: the searches treat
// the nodes as independent.
static inline const char* fv_csr_check(int npairs, int stride, const int32_t* n, const int32_t* node, const int32_t* start, const int32_t* feat,
                                       const int32_t* count, int* bad) {
    std::vector<uint8_t> seen(stride);
    for (int p = 0; p < npairs; p++) {
        *bad = p;
        if (n[p] < 0) return "negative feature count";
        const int nn = n[p] < stride ? n[p] : stride, c = count[p];
        if (c < 0 || c > stride) return "node count outside [0, stride]";
        const int32_t* st = start + (size_t)p * (stride + 1); const int32_t* nd = node + (size_t)p * stride; const int32_t* ft = feat + (size_t)p * stride;
        if (st[0] < 0) return "fv_start below 0";
        for (int j = 0; j < c; j++) if (st[j + 1] < st[j]) return "fv_start decreases";
        if (st[c] > nn) return "fv_start exceeds the feature count";
        if (c && nd[0] < 0) return "negative node id";
        for (int j = 0; j + 1 < c; j++) if (nd[j + 1] <= nd[j]) return "nodes not strictly ascending";
        std::fill(seen.begin(), seen.end(), 0);
        for (int k = st[0]; k < st[c]; k++) {
            if (ft[k] < 0 || ft[k] >= nn) return "feature index outside [0, feature count)";
            if (seen[ft[k]]++) return "feature listed twice";
        }
    }
    return nullptr;
}

// Node ids the keys hold apart: [-1, 2^20 - 1). -1 (a stopped word's feature, in no FeatureVector node) packs to group 0xfffff, which the
// searches skip; 2^20 - 1 would share that group, and anything else outside the range would alias another node through the 32-bit key.
static const int NODE_ID_END = (1 << 20) - 1;
static inline bool node_ids_ok(const int32_t* node, size_t n) {
    for (size_t i = 0; i < n; i++) if (node[i] < -1 || node[i] >= NODE_ID_END) return false;
    return true;
}

}  // namespace cslam

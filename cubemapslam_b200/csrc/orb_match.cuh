// Device-side ORB-matching rules shared by the matcher kernels (match.cu, track.cu, mapping.cu, bow.cu): one definition each, so the
// reference's exact rounding and tie-breaking live in one place.
#pragma once
#include <cstdint>

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

// Node ids the keys hold apart: [-1, 2^20 - 1). -1 (a stopped word's feature, in no FeatureVector node) packs to group 0xfffff, which the
// searches skip; 2^20 - 1 would share that group, and anything else outside the range would alias another node through the 32-bit key.
static const int NODE_ID_END = (1 << 20) - 1;
static inline bool node_ids_ok(const int32_t* node, size_t n) {
    for (size_t i = 0; i < n; i++) if (node[i] < -1 || node[i] >= NODE_ID_END) return false;
    return true;
}

}  // namespace cslam

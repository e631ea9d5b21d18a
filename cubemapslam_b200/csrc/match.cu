// 256-bit Hamming matching of libcubemap_b200.so, sm_90a.
//
// Reference (CPU): SearchByBoW(KeyFrame*,Frame&,...) src/ORBMatcher.cpp:409-539, thresholds :42-45; DescriptorDistance, the rotation bin
//   and ComputeThreeMaxima are restated once in orb_match.cuh.
// The all-pairs ("brute force") matcher of BASELINE config 3 has no reference function; DESIGN.md defines it as the
// SearchByBoW acceptance rule + rotation histogram applied to the best/second-best column of every row of A.
//
// k_match_bruteforce  binary tensor-core GEMM: dist(a, b) = popc(a) + popc(b) - 2 popc(a AND b), popc(a AND b) of a 16 x 8 tile of
//                     (A row, B row) pairs over the whole 256-bit descriptor is one BMMA (mma m16n8k256 .b1 .and.popc). A CTA owns
//                     256 rows of A (a warp keeps 4 m16 fragments in registers); B streams through shared memory in 128-descriptor
//                     tiles (cp.async, double-buffered, ldmatrix with a 16-byte-chunk XOR swizzle). Best / second best per row are
//                     exact integer minima of a key that packs (distance, column). The rows of a pair are split over CTAs; the
//                     rotation histogram and 3-maxima filter run in the CTA of the pair that arrives last. Bound by the min/max
//                     epilogue (4 integer instructions per distance) and the BMMA issue rate, not by HBM (192 KB per pair).
// k_search_by_bow     one CTA per pair; both FeatureVectors are rebuilt on the fly by an in-CTA bitonic sort of
//                     (node, index); one warp walks the KF features of a node in order (the reference's "already
//                     matched" skip makes that order matter), lanes scan the F features of the node.
#include <cstring>
#include <vector>
#include "common.cuh"
#include "orb_match.cuh"

namespace cslam {

static const int BF_WARPS = 4;
static const int BF_THREADS = 32 * BF_WARPS;
static const int BF_MT = 4;                          // m16 row fragments per warp
static const int BF_ROWS = BF_WARPS * BF_MT * 16;    // rows of A per CTA
static const int BF_TILE = 128;                      // descriptors of B per shared-memory stage (one per thread for the popcount)
static const int BF_COL_BITS = 12;                   // column field of a selection key: columns < 4096 (max_features)
static_assert(BF_TILE == BF_THREADS, "one thread per staged column");

// popc(a AND b) for a 16 x 8 tile of 256-bit rows: A fragment a[0..3] = words (t, t of row g+8, 4+t, 4+t of row g+8) of row g = lane / 4,
// t = lane % 4; B fragment b0 / b1 = words t / 4+t of column g; d[0..3] = (g, 2t), (g, 2t+1), (g+8, 2t), (g+8, 2t+1).
__device__ __forceinline__ void bmma_and_popc(int (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
    asm("mma.sync.aligned.m16n8k256.row.col.s32.b1.b1.s32.and.popc {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%10,%10,%10,%10};"
        : "=r"(d[0]), "=r"(d[1]), "=r"(d[2]), "=r"(d[3]) : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1), "r"(0));
}

__device__ __forceinline__ void cp_async16(uint32_t dst, const void* src, int bytes) {   // bytes < 16: the rest is zero-filled
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" :: "r"(dst), "l"(src), "r"(bytes) : "memory");
}

// Selection key of one distance: (popc(b) - 2 popc(a AND b)) << 12 | column; the row's popc(a) is added when the key is decoded. Smaller key =
// smaller distance, then lower column ("first column wins"). best1 / best2 are the two smallest keys of the row (keys are distinct, so a
// duplicate minimum distance gives dist(best2) == dist(best1)).
__device__ __forceinline__ void bf_take(int& best1, int& best2, int key) {
    best2 = min(best2, max(best1, key));
    best1 = min(best1, key);
}
__device__ __forceinline__ void bf_merge(int& best1, int& best2, int o1, int o2) {
    best2 = min(max(best1, o1), min(best2, o2));
    best1 = min(best1, o1);
}
// Key -> distance (capped at 256, which also catches the key of a column past nB: its prefix is INT_MAX)
__device__ __forceinline__ int bf_dist(int popcA, int key) { return min(256, popcA + (key >> BF_COL_BITS)); }

// Layout: pair p reads rows [p*strideA, p*strideA + nA) of descA (and B likewise); angles are read with a stride of `angStride` floats
// (1 for a plain float array, 7 for cv::KeyPoint records, whose `angle` field the pointer then addresses); when nAarr / nBarr are given they
// hold per-pair row counts (the front end's n_out). Outputs are strided like A.
struct BfLayout { int strideA, strideB, angStride; const int32_t* nAarr; const int32_t* nBarr; };
__global__ void __launch_bounds__(BF_THREADS) k_match_bruteforce(const uint8_t* __restrict__ descA, const float* __restrict__ angA, int nA_,
                                                                 const uint8_t* __restrict__ descB, const float* __restrict__ angB, int nB_, float nnratio,
                                                                 int thLow, int checkOri, int32_t* __restrict__ match12, int32_t* __restrict__ dist12,
                                                                 int32_t* __restrict__ second12, int32_t* __restrict__ nmatches, BfLayout L, int* __restrict__ gHist) {
    // CTA (pair, part) owns rows [part * BF_ROWS, +BF_ROWS) of A; gridDim.y covers the largest row count the launch allows, CTAs past the pair's
    // own count exit at once. With more than one part the rotation histogram goes through gHist[pair][32] (30 bins, total, arrival counter;
    // zeroed by the launcher) and the CTA that arrives last applies the three-maxima filter to the whole pair.
    __shared__ __align__(128) uint4 sB[2][2 * BF_TILE];   // 32-byte rows; 16-byte chunk c of row r sits at chunk c ^ ((r >> 2) & 1)
    __shared__ __align__(16) int sPre[BF_TILE];           // popc(b) << 12 | column, INT_MAX past nB
    __shared__ int hist[HISTO_BINS], keep[HISTO_BINS], total;
    __shared__ bool lastCta;
    const int pair = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, g = lane >> 2, t = lane & 3;
    const int nA = L.nAarr ? min(L.nAarr[pair], L.strideA) : nA_, nB = L.nBarr ? min(L.nBarr[pair], L.strideB) : nB_;
    const int parts = max(1, (nA + BF_ROWS - 1) / BF_ROWS), part = blockIdx.y;
    if (part >= parts) return;
    const uint32_t* Aw = reinterpret_cast<const uint32_t*>(descA + (size_t)pair * L.strideA * 32);
    const uint4* B4 = reinterpret_cast<const uint4*>(descB + (size_t)pair * L.strideB * 32);
    const float* aA = angA + (size_t)pair * L.strideA * L.angStride;
    const float* aB = angB + (size_t)pair * L.strideB * L.angStride;
    int32_t* m12 = match12 + (size_t)pair * L.strideA;
    if (tid < HISTO_BINS) hist[tid] = 0;
    if (tid == 0) total = 0;

    // A fragments of this warp's 4 x 16 rows (zero past nA) and popc(a) of rows g / g+8 of each
    const int row0 = part * BF_ROWS + warp * BF_MT * 16;
    const int nmt = min(BF_MT, max(0, (nA - row0 + 15) >> 4));   // live m16 fragments of this warp
    uint32_t a[BF_MT][4];
    int popcA[BF_MT][2], best1[BF_MT][2], best2[BF_MT][2];
#pragma unroll
    for (int mt = 0; mt < BF_MT; mt++) {
        const int r = row0 + mt * 16 + g;
        a[mt][0] = r < nA ? __ldg(Aw + (size_t)r * 8 + t) : 0u;
        a[mt][1] = r + 8 < nA ? __ldg(Aw + (size_t)(r + 8) * 8 + t) : 0u;
        a[mt][2] = r < nA ? __ldg(Aw + (size_t)r * 8 + 4 + t) : 0u;
        a[mt][3] = r + 8 < nA ? __ldg(Aw + (size_t)(r + 8) * 8 + 4 + t) : 0u;
        int p0 = __popc(a[mt][0]) + __popc(a[mt][2]), p1 = __popc(a[mt][1]) + __popc(a[mt][3]);
        p0 += __shfl_xor_sync(0xffffffffu, p0, 1); p1 += __shfl_xor_sync(0xffffffffu, p1, 1);
        p0 += __shfl_xor_sync(0xffffffffu, p0, 2); p1 += __shfl_xor_sync(0xffffffffu, p1, 2);
        popcA[mt][0] = p0; popcA[mt][1] = p1;
        best1[mt][0] = best1[mt][1] = best2[mt][0] = best2[mt][1] = INT_MAX;
    }

    // B: stage k = descriptors [k * BF_TILE, +BF_TILE) into sB[k & 1]; rows past nB are zero-filled (their key prefix is INT_MAX anyway)
    const uint32_t sBase = (uint32_t)__cvta_generic_to_shared(&sB[0][0]);
    auto stage = [&](int k) {
        const uint32_t dst = sBase + (uint32_t)(k & 1) * (2 * BF_TILE * 16);
        for (int q = tid; q < 2 * BF_TILE; q += BF_THREADS) {
            const int r = q >> 1, c = q & 1, col = k * BF_TILE + r;
            const bool ok = col < nB;
            cp_async16(dst + (uint32_t)(r * 32 + ((c ^ ((r >> 2) & 1)) << 4)), ok ? (const void*)(B4 + 2 * col + c) : (const void*)B4, ok ? 16 : 0);
        }
        asm volatile("cp.async.commit_group;" ::: "memory");
    };
    // ldmatrix.x4 source row of this lane: matrices (cols 0-7, chunk 0), (0-7, 1), (8-15, 0), (8-15, 1) of a 16-column group -> b0, b1 of
    // two n8 tiles
    const int lr = ((lane >> 4) << 3) + (lane & 7), lc = (lane >> 3) & 1;
    const uint32_t ldOff = (uint32_t)(lr * 32 + ((lc ^ ((lr >> 2) & 1)) << 4));
    const int ntiles = (nB + BF_TILE - 1) / BF_TILE;
    if (ntiles) stage(0);
    __syncthreads();                         // hist / total are zeroed (nB may be 0)
    for (int kt = 0; kt < ntiles; kt++) {
        asm volatile("cp.async.wait_group 0;" ::: "memory");
        __syncthreads();                     // stage kt has landed; every warp is done with stage kt-1 and with sPre
        if (kt + 1 < ntiles) stage(kt + 1);  // overlaps with this stage's MMAs
        {
            const int col = kt * BF_TILE + tid;
            const uint4 u0 = sB[kt & 1][2 * tid], u1 = sB[kt & 1][2 * tid + 1];   // chunk order does not matter for the popcount
            const int pb = __popc(u0.x) + __popc(u0.y) + __popc(u0.z) + __popc(u0.w) + __popc(u1.x) + __popc(u1.y) + __popc(u1.z) + __popc(u1.w);
            sPre[tid] = col < nB ? (pb << BF_COL_BITS) | col : INT_MAX;
        }
        __syncthreads();
        if (nmt > 0) {
            const uint32_t sb = sBase + (uint32_t)(kt & 1) * (2 * BF_TILE * 16) + ldOff;
#pragma unroll 2
            for (int j = 0; j < BF_TILE / 16; j++) {
                uint32_t b[4];
                asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];"
                             : "=r"(b[0]), "=r"(b[1]), "=r"(b[2]), "=r"(b[3]) : "r"(sb + (uint32_t)j * 512));
                const int2 p0 = *reinterpret_cast<const int2*>(&sPre[16 * j + 2 * t]), p1 = *reinterpret_cast<const int2*>(&sPre[16 * j + 8 + 2 * t]);
#pragma unroll
                for (int mt = 0; mt < BF_MT; mt++) {
                    if (mt < nmt) {
                        int d[4], e[4];
                        bmma_and_popc(d, a[mt], b[0], b[1]);
                        bmma_and_popc(e, a[mt], b[2], b[3]);
                        bf_take(best1[mt][0], best2[mt][0], d[0] * -(2 << BF_COL_BITS) + p0.x);
                        bf_take(best1[mt][0], best2[mt][0], d[1] * -(2 << BF_COL_BITS) + p0.y);
                        bf_take(best1[mt][1], best2[mt][1], d[2] * -(2 << BF_COL_BITS) + p0.x);
                        bf_take(best1[mt][1], best2[mt][1], d[3] * -(2 << BF_COL_BITS) + p0.y);
                        bf_take(best1[mt][0], best2[mt][0], e[0] * -(2 << BF_COL_BITS) + p1.x);
                        bf_take(best1[mt][0], best2[mt][0], e[1] * -(2 << BF_COL_BITS) + p1.y);
                        bf_take(best1[mt][1], best2[mt][1], e[2] * -(2 << BF_COL_BITS) + p1.x);
                        bf_take(best1[mt][1], best2[mt][1], e[3] * -(2 << BF_COL_BITS) + p1.y);
                    }
                }
            }
        }
    }

    // merge the 4 lanes of a quad (columns 2t, 2t+1 of every n8 tile); lane t then finishes row-sets (mt, h) with (2 mt + h) % 4 == t
#pragma unroll
    for (int mt = 0; mt < BF_MT; mt++)
#pragma unroll
        for (int h = 0; h < 2; h++)
#pragma unroll
            for (int o = 1; o <= 2; o <<= 1)
                bf_merge(best1[mt][h], best2[mt][h], __shfl_xor_sync(0xffffffffu, best1[mt][h], o), __shfl_xor_sync(0xffffffffu, best2[mt][h], o));
#pragma unroll
    for (int mt = 0; mt < BF_MT; mt++)
#pragma unroll
        for (int h = 0; h < 2; h++) {
            const int i = row0 + mt * 16 + h * 8 + g;
            if (((2 * mt + h) & 3) != t || i >= nA) continue;
            const int d1 = bf_dist(popcA[mt][h], best1[mt][h]), d2 = bf_dist(popcA[mt][h], best2[mt][h]);
            const int bestIdx = d1 < 256 ? (best1[mt][h] & ((1 << BF_COL_BITS) - 1)) : -1;
            int m = -1;
            if (bestIdx >= 0 && d1 <= thLow && (float)d1 < __fmul_rn(nnratio, (float)d2)) {
                m = bestIdx;
                if (checkOri) atomicAdd(&hist[rot_bin(aA[(size_t)i * L.angStride], aB[(size_t)bestIdx * L.angStride])], 1);
                atomicAdd(&total, 1);
            }
            m12[i] = m;
            if (dist12) dist12[(size_t)pair * L.strideA + i] = d1;
            if (second12) second12[(size_t)pair * L.strideA + i] = d2;
        }
    __syncthreads();
    if (parts > 1) {
        int* g = gHist + (size_t)pair * 32;
        if (tid < HISTO_BINS && hist[tid]) atomicAdd(g + tid, hist[tid]);
        if (tid == 0 && total) atomicAdd(g + 30, total);
        __threadfence();
        __syncthreads();
        if (tid == 0) lastCta = atomicAdd(g + 31, 1) == parts - 1;
        __syncthreads();
        if (!lastCta) return;
        __threadfence();
        if (tid < HISTO_BINS) hist[tid] = __ldcg(g + tid);
        if (tid == 0) total = __ldcg(g + 30);
        __syncthreads();
    }
    if (checkOri) {
        if (tid == 0) three_maxima(hist, keep);
        __syncthreads();
        for (int i = tid; i < nA; i += BF_THREADS) {
            const int m = parts > 1 ? __ldcg(m12 + i) : m12[i];
            if (m >= 0 && !keep[rot_bin(aA[(size_t)i * L.angStride], aB[(size_t)m * L.angStride])]) { m12[i] = -1; atomicSub(&total, 1); }
        }
        __syncthreads();
    }
    if (tid == 0) nmatches[pair] = total;
}

// ------------------------------------------------------------------------------------------------- SearchByBoW
static const int BOW_THREADS = 256;

// keys: node << 12 | index (index < 4096, node in [-1, 2^20 - 1): node -1 = in no FeatureVector node, key group 0xfffff, never matched).
// Shared memory: keyKF[n2K], keyF[n2F], takenF[nF] bytes.
__global__ void __launch_bounds__(BOW_THREADS) k_search_by_bow(const uint8_t* __restrict__ descKF, const float* __restrict__ angKF,
                                                               const uint8_t* __restrict__ kfValid, const int32_t* __restrict__ nodeKF, int nKF,
                                                               const uint8_t* __restrict__ descF, const float* __restrict__ angF,
                                                               const int32_t* __restrict__ nodeF, int nF, int n2K, int n2F, float nnratio, int checkOri,
                                                               int32_t* __restrict__ matchF, int32_t* __restrict__ nmatches,
                                                               const uint8_t* __restrict__ fValid, int kfkfMode) {
    // kfkfMode = 0: SearchByBoW(KeyFrame*, Frame&)  (src/ORBMatcher.cpp:409-539), output per F feature.
    // kfkfMode = 1: SearchByBoW(KeyFrame*, KeyFrame*) (:541-674): F-side features need fValid, acceptance is strict (< TH_LOW),
    //               output per KF feature (index of the matched feature of the second key frame).
    extern __shared__ __align__(16) uint8_t smem[];
    uint32_t* keyKF = reinterpret_cast<uint32_t*>(smem);
    uint32_t* keyF = keyKF + n2K;
    int* mF = reinterpret_cast<int*>(keyF + n2F);   // match per F feature (KF index or -1), staged in shared memory
    __shared__ int hist[HISTO_BINS], keep[HISTO_BINS], total;
    const int pair = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nwarps = BOW_THREADS / 32;
    const uint4* K4 = reinterpret_cast<const uint4*>(descKF + (size_t)pair * nKF * 32);
    const uint4* F4 = reinterpret_cast<const uint4*>(descF + (size_t)pair * nF * 32);
    const float* aK = angKF + (size_t)pair * nKF;
    const float* aF = angF + (size_t)pair * nF;
    const uint8_t* val = kfValid + (size_t)pair * nKF;
    const int32_t* nK = nodeKF + (size_t)pair * nKF;
    const int32_t* nFd = nodeF + (size_t)pair * nF;
    for (int i = tid; i < n2K; i += BOW_THREADS) keyKF[i] = i < nKF ? ((uint32_t)nK[i] << 12) | (uint32_t)i : 0xffffffffu;
    for (int i = tid; i < n2F; i += BOW_THREADS) keyF[i] = i < nF ? ((uint32_t)nFd[i] << 12) | (uint32_t)i : 0xffffffffu;
    for (int i = tid; i < nF; i += BOW_THREADS) mF[i] = -1;
    if (tid < HISTO_BINS) hist[tid] = 0;
    if (tid == 0) total = 0;
    __syncthreads();
    block_bitonic_sort(keyKF, n2K);
    block_bitonic_sort(keyF, n2F);
    // one warp per KF node group: a group starts where the node id changes
    for (int s = warp; s < nKF; s += nwarps) {
        // warps take candidate group starts round-robin: position s is a start iff s==0 or node differs from s-1
        // (cheap: every warp scans its own positions; groups are independent of each other)
        const uint32_t node = keyKF[s] >> 12;
        if (node == 0xfffffu || (s > 0 && (keyKF[s - 1] >> 12) == node)) continue;   // 0xfffff: node -1, in no FeatureVector node
        // KF group [s, e)
        int e = s + 1;
        while (e < nKF && (keyKF[e] >> 12) == node) e++;
        // F group by binary search of node << 12
        const int fs = node_lower_bound(keyF, nF, node);
        int fe = fs;
        while (fe < nF && (keyF[fe] >> 12) == node) fe++;
        if (fe == fs) continue;
        for (int q = s; q < e; q++) {
            const int iK = keyKF[q] & 0xfff;
            if (!val[iK]) continue;
            const uint4 k0 = __ldg(K4 + 2 * iK), k1 = __ldg(K4 + 2 * iK + 1);
            // lanes scan the F features of the node in list order; (best1, pos, best2) with first-position ties
            int best1 = 256, best2 = 256, bpos = 0x7fffffff;
            for (int p = fs + lane; p < fe; p += 32) {
                const int iF = keyF[p] & 0xfff;
                if (mF[iF] >= 0) continue;
                if (kfkfMode && !fValid[(size_t)pair * nF + iF]) continue;
                const int d = hamming256(k0, k1, __ldg(F4 + 2 * iF), __ldg(F4 + 2 * iF + 1));
                if (d < best1) { best2 = best1; best1 = d; bpos = p; }
                else if (d < best2) best2 = d;
            }
#pragma unroll
            for (int o = 16; o; o >>= 1) {
                const int ob1 = __shfl_xor_sync(0xffffffffu, best1, o), ob2 = __shfl_xor_sync(0xffffffffu, best2, o), op = __shfl_xor_sync(0xffffffffu, bpos, o);
                // merge two partial scans: the winner is the smaller distance, ties go to the earlier list position
                const bool otherWins = ob1 < best1 || (ob1 == best1 && op < bpos);
                if (otherWins) { best2 = min(best1, ob2); best1 = ob1; bpos = op; }
                else best2 = min(best2, ob1);
            }
            if ((kfkfMode ? best1 < 50 : best1 <= 50) && (float)best1 < __fmul_rn(nnratio, (float)best2)) {
                const int iF = keyF[bpos] & 0xfff;
                if (lane == 0) {
                    mF[iF] = iK;
                    if (checkOri) atomicAdd(&hist[rot_bin(aK[iK], aF[iF])], 1);
                    atomicAdd(&total, 1);
                }
            }
            __syncwarp();
        }
    }
    __syncthreads();
    if (checkOri) {
        if (tid == 0) three_maxima(hist, keep);
        __syncthreads();
        for (int j = tid; j < nF; j += BOW_THREADS) {
            const int m = mF[j];
            if (m >= 0 && !keep[rot_bin(aK[m], aF[j])]) { mF[j] = -1; atomicSub(&total, 1); }
        }
        __syncthreads();
    }
    if (!kfkfMode) {
        int32_t* out = matchF + (size_t)pair * nF;
        for (int j = tid; j < nF; j += BOW_THREADS) out[j] = mF[j];
    } else {
        int32_t* out = matchF + (size_t)pair * nKF;
        for (int i = tid; i < nKF; i += BOW_THREADS) out[i] = -1;
        __syncthreads();
        for (int j = tid; j < nF; j += BOW_THREADS) if (mF[j] >= 0) out[mF[j]] = j;
    }
    if (tid == 0) nmatches[pair] = total;
}

__global__ void k_hamming(const uint8_t* __restrict__ a, const uint8_t* __restrict__ b, int n, int32_t* __restrict__ dist) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint4* A4 = reinterpret_cast<const uint4*>(a) + 2 * (size_t)i;
    const uint4* B4 = reinterpret_cast<const uint4*>(b) + 2 * (size_t)i;
    const uint4 a0 = __ldg(A4), a1 = __ldg(A4 + 1);
    dist[i] = hamming256(a0, a1, __ldg(B4), __ldg(B4 + 1));
}

}  // namespace cslam

using namespace cslam;

// arena: staging of the host entry points, the row-split histogram and the micro-benchmarks' output sink
struct cslam_matcher : cslam::Handle {
    int maxPairs = 0, maxFeat = 0;
};

extern "C" int cslam_matcher_create(cslam_matcher** out, int device, int max_pairs, int max_features) {
    if (!out || max_pairs <= 0 || max_features <= 0 || max_features > 4096) { set_error("cslam_matcher_create: bad argument (max_features <= 4096)"); return CSLAM_E_BADARG; }
    cslam_matcher* m = new cslam_matcher;
    m->maxPairs = max_pairs; m->maxFeat = max_features;
    // chunks: room for both descriptor sets, a flag and seven 4-byte arrays per feature at the handle's limits, at most 64 MB
    const int rc = m->open(device, std::min<size_t>((size_t)64 << 20, (size_t)max_pairs * max_features * (2 * 32 + 1 + 7 * 4) + (size_t)max_pairs * 4), false);
    if (rc) { destroy_handle(m); return rc; }
    cudaFuncSetAttribute(k_search_by_bow, cudaFuncAttributeMaxDynamicSharedMemorySize, 64 * 1024);
    *out = m;
    return CSLAM_OK;
}

extern "C" void cslam_matcher_destroy(cslam_matcher* m) { destroy_handle(m); }
extern "C" void* cslam_matcher_stream(const cslam_matcher* m) { return m ? (void*)m->stream : nullptr; }
extern "C" int64_t cslam_matcher_launches(const cslam_matcher* m) { return m ? m->launches : 0; }
extern "C" int cslam_matcher_sync(cslam_matcher* m) { return m ? m->sync() : CSLAM_E_BADARG; }

// The brute-force launch of every entry point: one CTA per BF_ROWS rows of the largest A a pair can have (L.strideA); with more than one, the
// per-pair rotation histogram is a zeroed arena piece.
static int bf_launch(cslam_matcher* m, int npairs, const uint8_t* descA, const float* angA, int nA, const uint8_t* descB, const float* angB, int nB, float nnratio,
                     int th_low, int check_ori, int32_t* match12, int32_t* dist12, int32_t* second12, int32_t* nmatches, const BfLayout& L) {
    const int parts = std::max(1, cdiv(L.strideA, BF_ROWS));
    int* gHist = nullptr;
    if (parts > 1) { const int rc = m->arena.take(&gHist, (size_t)npairs * 32, true); if (rc) return rc; }
    k_match_bruteforce<<<dim3(npairs, parts), BF_THREADS, 0, m->stream>>>(descA, angA, nA, descB, angB, nB, nnratio, th_low, check_ori, match12, dist12, second12, nmatches, L, gHist);
    m->launches++;
    CSLAM_CUDA(cudaGetLastError());
    return CSLAM_OK;
}
// frame f of a front-end batch (rows [f*kp_stride, f*kp_stride + n[f]) of kps / desc) against frame f+1, for f = 0 .. nframes-2
static int frames_launch(cslam_matcher* m, const cslam_keypoint* kps, const uint8_t* desc, const int32_t* n, int kp_stride, int nframes, float nnratio, int th_low,
                         int check_ori, int32_t* match12, int32_t* nmatches) {
    const float* ang = &kps[0].angle;
    const BfLayout L = {kp_stride, kp_stride, (int)(sizeof(cslam_keypoint) / sizeof(float)), n, n + 1};
    return bf_launch(m, nframes - 1, desc, ang, 0, desc + (size_t)kp_stride * 32, ang + (size_t)kp_stride * L.angStride, 0, nnratio, th_low, check_ori, match12, nullptr,
                     nullptr, nmatches, L);
}

static int check_sizes(cslam_matcher* m, int nA, int nB, int npairs) {
    if (!m || nA < 0 || nB < 0 || npairs <= 0 || npairs > m->maxPairs || nA > m->maxFeat || nB > m->maxFeat) {
        set_error("matcher: sizes out of range (pairs %d/%d, features %d,%d/%d)", npairs, m ? m->maxPairs : 0, nA, nB, m ? m->maxFeat : 0);
        return CSLAM_E_BADARG;
    }
    CSLAM_CUDA(cudaSetDevice(m->device));
    return 0;
}

extern "C" int cslam_match_bruteforce_dev(cslam_matcher* m, const uint8_t* descA, const float* angA, int nA, const uint8_t* descB, const float* angB, int nB,
                                          int npairs, float nnratio, int th_low, int check_ori, int32_t* match12, int32_t* dist12, int32_t* second12,
                                          int32_t* nmatches) {
    int rc = check_sizes(m, nA, nB, npairs);
    if (rc) return rc;
    if (nA == 0) { CSLAM_CUDA(cudaMemsetAsync(nmatches, 0, (size_t)npairs * 4, m->stream)); return CSLAM_OK; }
    m->arena.reset();
    return bf_launch(m, npairs, descA, angA, nA, descB, angB, nB, nnratio, th_low, check_ori, match12, dist12, second12, nmatches, {nA, nB, 1, nullptr, nullptr});
}

extern "C" int cslam_match_bruteforce(cslam_matcher* m, const uint8_t* descA, const float* angA, int nA, const uint8_t* descB, const float* angB, int nB, int npairs,
                                      float nnratio, int th_low, int check_ori, int32_t* match12, int32_t* dist12, int32_t* second12, int32_t* nmatches) {
    int rc = check_sizes(m, nA, nB, npairs);
    if (rc) return rc;
    m->arena.reset();
    const size_t na = (size_t)npairs * nA, nb = (size_t)npairs * nB;
    const uint8_t *dA, *dB; const float *aA, *aB; int32_t *dMatch, *dDist, *dSecond, *dN;
    if ((rc = m->arena.upload(&dA, descA, na * 32)) || (rc = m->arena.upload(&aA, angA, na)) || (rc = m->arena.upload(&dB, descB, nb * 32)) || (rc = m->arena.upload(&aB, angB, nb)) ||
        (rc = m->arena.take(&dMatch, na)) || (rc = m->arena.take(&dDist, na)) || (rc = m->arena.take(&dSecond, na)) || (rc = m->arena.take(&dN, npairs))) return rc;
    if (nA == 0) CSLAM_CUDA(cudaMemsetAsync(dN, 0, (size_t)npairs * 4, m->stream));
    else if ((rc = bf_launch(m, npairs, dA, aA, nA, dB, aB, nB, nnratio, th_low, check_ori, dMatch, dDist, dSecond, dN, {nA, nB, 1, nullptr, nullptr}))) return rc;
    if (na) {
        CSLAM_CUDA(cudaMemcpyAsync(match12, dMatch, na * 4, cudaMemcpyDeviceToHost, m->stream));
        if (dist12) CSLAM_CUDA(cudaMemcpyAsync(dist12, dDist, na * 4, cudaMemcpyDeviceToHost, m->stream));
        if (second12) CSLAM_CUDA(cudaMemcpyAsync(second12, dSecond, na * 4, cudaMemcpyDeviceToHost, m->stream));
    }
    CSLAM_CUDA(cudaMemcpyAsync(nmatches, dN, (size_t)npairs * 4, cudaMemcpyDeviceToHost, m->stream));
    return m->sync();
}

// All-pairs matcher between consecutive frames of a front-end batch, straight from cslam_frontend_run_dev's output layout: frame f (rows
// [f*kp_stride, f*kp_stride + n[f]) of kps / desc) is matched against frame f+1 for f = 0 .. nframes-2. match12: (nframes-1) x kp_stride.
extern "C" int cslam_match_frames_dev(cslam_matcher* m, const cslam_keypoint* kps, const uint8_t* desc, const int32_t* n, int kp_stride, int nframes, float nnratio, int th_low,
                                      int check_ori, int32_t* match12, int32_t* nmatches) {
    if (!m || !kps || !desc || !n || !match12 || !nmatches || nframes < 2 || nframes - 1 > m->maxPairs || kp_stride <= 0 || kp_stride > m->maxFeat) {
        set_error("cslam_match_frames_dev: bad argument (frames %d, pairs <= %d, stride %d <= %d)", nframes, m ? m->maxPairs : 0, kp_stride, m ? m->maxFeat : 0);
        return CSLAM_E_BADARG;
    }
    CSLAM_CUDA(cudaSetDevice(m->device));
    m->arena.reset();
    return frames_launch(m, kps, desc, n, kp_stride, nframes, nnratio, th_low, check_ori, match12, nmatches);
}

// host buffers in / out (copies inside, synchronous): kps / desc / n as cslam_frontend_run returns them
extern "C" int cslam_match_frames(cslam_matcher* m, const cslam_keypoint* kps, const uint8_t* desc, const int32_t* n, int kp_stride, int nframes, float nnratio, int th_low,
                                  int check_ori, int32_t* match12, int32_t* nmatches) {
    if (!m || nframes < 2 || nframes > m->maxPairs || kp_stride <= 0 || kp_stride > m->maxFeat) { set_error("cslam_match_frames: sizes out of range (frames %d/%d, stride %d/%d)", nframes, m ? m->maxPairs : 0, kp_stride, m ? m->maxFeat : 0); return CSLAM_E_BADARG; }
    CSLAM_CUDA(cudaSetDevice(m->device));
    m->arena.reset();
    const size_t nf = (size_t)nframes * kp_stride, nm = (size_t)(nframes - 1) * kp_stride;
    const cslam_keypoint* dK; const uint8_t* dD; const int32_t* dN; int32_t *dMatch, *dNm; int rc;
    if ((rc = m->arena.upload(&dK, kps, nf)) || (rc = m->arena.upload(&dD, desc, nf * 32)) || (rc = m->arena.upload(&dN, n, nframes)) || (rc = m->arena.take(&dMatch, nm)) ||
        (rc = m->arena.take(&dNm, nframes - 1)) || (rc = frames_launch(m, dK, dD, dN, kp_stride, nframes, nnratio, th_low, check_ori, dMatch, dNm))) return rc;
    CSLAM_CUDA(cudaMemcpyAsync(match12, dMatch, nm * 4, cudaMemcpyDeviceToHost, m->stream));
    CSLAM_CUDA(cudaMemcpyAsync(nmatches, dNm, (size_t)(nframes - 1) * 4, cudaMemcpyDeviceToHost, m->stream));
    return m->sync();
}

// Harness of the register-only issue-rate micro-benchmarks below: 8 CTAs per SM, a warm-up launch of 100 iterations, then the timed
// launch of `iters`. launch(blocks, iters, out) enqueues the kernel on m->stream; *blocks is the grid it was given, *ms the timed launch.
template <class Launch>
static int time_ubench(cslam_matcher* m, int iters, Launch launch, int* blocks, float* ms) {
    int sms = 132;
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, m->device);
    *blocks = sms * 8;
    uint32_t* out;
    const int rc = m->arena.take(&out, 1);
    if (rc) return rc;
    cudaEvent_t e0, e1;
    CSLAM_CUDA(cudaEventCreate(&e0)); CSLAM_CUDA(cudaEventCreate(&e1));
    launch(*blocks, 100, out);   // warm-up
    CSLAM_CUDA(cudaEventRecord(e0, m->stream));
    launch(*blocks, iters, out);
    CSLAM_CUDA(cudaEventRecord(e1, m->stream));
    CSLAM_CUDA(cudaStreamSynchronize(m->stream));
    CSLAM_CUDA(cudaEventElapsedTime(ms, e0, e1));
    cudaEventDestroy(e0); cudaEventDestroy(e1);
    m->launches += 2;
    return CSLAM_OK;
}

// POPC issue-rate micro-benchmark (SURVEY 8d: "measure the real rate with a micro-benchmark on the box before quoting a fraction"): every thread
// runs `iters` rounds of 8 independent XOR+POPC+ADD chains on registers - the exact instruction mix of hamming256 (orb_match.cuh) without any memory traffic.
__global__ void __launch_bounds__(256) k_ubench_popc(uint32_t* out, int iters, uint32_t seed) {
    uint32_t a[8], acc[8];
#pragma unroll
    for (int k = 0; k < 8; k++) { a[k] = seed * (threadIdx.x + 1) + k * 0x9e3779b9u + blockIdx.x; acc[k] = 0; }
    for (int i = 0; i < iters; i++) {
#pragma unroll
        for (int k = 0; k < 8; k++) { acc[k] += __popc(a[k] ^ acc[(k + 1) & 7]); }
    }
    uint32_t s = 0;
#pragma unroll
    for (int k = 0; k < 8; k++) s += acc[k];
    if (s == 0xdeadbeefu) out[0] = s;   // keeps the chains alive
}
extern "C" int cslam_ubench_popc(cslam_matcher* m, double* popc32_per_s) {
    if (!m || !popc32_per_s) return CSLAM_E_BADARG;
    CSLAM_CUDA(cudaSetDevice(m->device));
    m->arena.reset();
    const int iters = 20000;
    int blocks; float ms;
    const int rc = time_ubench(m, iters, [&](int b, int it, uint32_t* out) { k_ubench_popc<<<b, 256, 0, m->stream>>>(out, it, 1u); }, &blocks, &ms);
    if (rc) return rc;
    *popc32_per_s = (double)blocks * 256.0 * iters * 8.0 / (ms * 1e-3);
    return CSLAM_OK;
}

// Tensor-core issue-rate micro-benchmark: every warp runs `iters` rounds of 8 independent accumulator chains of one MMA shape on registers.
// BINARY: m16n8k256 .b1 AND.POPC (the matcher's BMMA); else m16n8k32 s8 IMMA (the same distance from +-1 int8 expansions of the bits).
template <bool BINARY>
__global__ void __launch_bounds__(256) k_ubench_mma(uint32_t* out, int iters, uint32_t seed) {
    uint32_t a[4], b[2];
#pragma unroll
    for (int k = 0; k < 4; k++) a[k] = seed * (threadIdx.x + 1) + k * 0x9e3779b9u + blockIdx.x;
    b[0] = a[0] ^ 0x5bd1e995u; b[1] = a[3] * 0x27d4eb2fu;
    int acc[8][4];
#pragma unroll
    for (int c = 0; c < 8; c++) acc[c][0] = acc[c][1] = acc[c][2] = acc[c][3] = c;
    for (int i = 0; i < iters; i++) {
#pragma unroll
        for (int c = 0; c < 8; c++) {
            if (BINARY)
                asm volatile("mma.sync.aligned.m16n8k256.row.col.s32.b1.b1.s32.and.popc {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                             : "+r"(acc[c][0]), "+r"(acc[c][1]), "+r"(acc[c][2]), "+r"(acc[c][3]) : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[0]), "r"(b[1]));
            else
                asm volatile("mma.sync.aligned.m16n8k32.row.col.s32.s8.s8.s32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                             : "+r"(acc[c][0]), "+r"(acc[c][1]), "+r"(acc[c][2]), "+r"(acc[c][3]) : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[0]), "r"(b[1]));
        }
    }
    int s = 0;
#pragma unroll
    for (int c = 0; c < 8; c++) s += acc[c][0] + acc[c][1] + acc[c][2] + acc[c][3];
    if (s == 0x7eadbeef) out[0] = (uint32_t)s;   // keeps the chains alive
}
extern "C" int cslam_ubench_bmma(cslam_matcher* m, double* bmma_products_per_s, double* imma_products_per_s) {
    if (!m || !bmma_products_per_s || !imma_products_per_s) return CSLAM_E_BADARG;
    CSLAM_CUDA(cudaSetDevice(m->device));
    m->arena.reset();
    const int iters = 4000;
    int blocks; float ms;
    int rc = time_ubench(m, iters, [&](int b, int it, uint32_t* out) { k_ubench_mma<true><<<b, 256, 0, m->stream>>>(out, it, 1u); }, &blocks, &ms);
    if (rc) return rc;
    const double n = (double)blocks * 8.0 * iters * 8.0;     // warp-level MMA instructions
    *bmma_products_per_s = n * 128.0 / (ms * 1e-3);          // 16 x 8 256-bit products per BMMA
    rc = time_ubench(m, iters, [&](int b, int it, uint32_t* out) { k_ubench_mma<false><<<b, 256, 0, m->stream>>>(out, it, 1u); }, &blocks, &ms);
    if (rc) return rc;
    *imma_products_per_s = n * 128.0 / 8.0 / (ms * 1e-3);    // 16 x 8 dot products of 32 bytes; a 256-bit product is 8 of them
    return CSLAM_OK;
}

// The front end's k_fast is bound by the issue rate of 3-input u16x2 min / max (VIMNMX3.U16x2, 80 of them per pixel pair): the same kind of
// register-only chain measurement gives the denominator of its roofline.
__global__ void __launch_bounds__(256) k_ubench_minmax3(uint32_t* out, int iters, uint32_t seed) {
    uint32_t a[8], acc[8];
#pragma unroll
    for (int k = 0; k < 8; k++) { a[k] = (seed * (threadIdx.x + 1) + k * 0x9e3779b9u + blockIdx.x) & 0x00ff00ffu; acc[k] = a[k] ^ 0x00550055u; }
    for (int i = 0; i < iters; i += 2) {
#pragma unroll
        for (int k = 0; k < 8; k++) acc[k] = __vimin3_u16x2(acc[k] + 0x00010001u * (i & 1), a[k], acc[(k + 1) & 7]);
#pragma unroll
        for (int k = 0; k < 8; k++) acc[k] = __vimax3_u16x2(acc[k], a[(k + 3) & 7], acc[(k + 5) & 7]);
    }
    uint32_t s = 0;
#pragma unroll
    for (int k = 0; k < 8; k++) s += acc[k];
    if (s == 0xdeadbeefu) out[0] = s;
}
extern "C" int cslam_ubench_minmax3(cslam_matcher* m, double* ops_per_s) {
    if (!m || !ops_per_s) return CSLAM_E_BADARG;
    CSLAM_CUDA(cudaSetDevice(m->device));
    m->arena.reset();
    const int iters = 20000;
    int blocks; float ms;
    const int rc = time_ubench(m, iters, [&](int b, int it, uint32_t* out) { k_ubench_minmax3<<<b, 256, 0, m->stream>>>(out, it, 1u); }, &blocks, &ms);
    if (rc) return rc;
    *ops_per_s = (double)blocks * 256.0 * iters * 8.0 / (ms * 1e-3);   // warp-lane u16x2 3-input min/max per second
    return CSLAM_OK;
}

// SearchByBoW launch of both forms. valid_f == nullptr: (KeyFrame, Frame), output per F feature; else (KeyFrame, KeyFrame) with the second
// key frame's valid flags, output per KF feature.
static int bow_launch(cslam_matcher* m, const uint8_t* descKF, const float* angKF, const uint8_t* kf_valid, const int32_t* node_kf, int nKF, const uint8_t* descF,
                      const float* angF, const int32_t* node_f, int nF, const uint8_t* valid_f, int npairs, float nnratio, int check_ori, int32_t* match, int32_t* nmatches) {
    const int n2K = pow2_at_least(nKF), n2F = pow2_at_least(nF);
    const size_t smem = (size_t)(n2K + n2F + nF) * 4;
    k_search_by_bow<<<npairs, BOW_THREADS, smem, m->stream>>>(descKF, angKF, kf_valid, node_kf, nKF, descF, angF, node_f, nF, n2K, n2F, nnratio, check_ori, match, nmatches,
                                                              valid_f, valid_f ? 1 : 0);
    m->launches++;
    CSLAM_CUDA(cudaGetLastError());
    return CSLAM_OK;
}

extern "C" int cslam_search_by_bow_dev(cslam_matcher* m, const uint8_t* descKF, const float* angKF, const uint8_t* kf_valid, const int32_t* node_kf, int nKF,
                                       const uint8_t* descF, const float* angF, const int32_t* node_f, int nF, int npairs, float nnratio, int check_ori,
                                       int32_t* match_f, int32_t* nmatches) {
    int rc = check_sizes(m, nKF, nF, npairs);
    if (rc) return rc;
    if (nF == 0 || nKF == 0) {
        CSLAM_CUDA(cudaMemsetAsync(nmatches, 0, (size_t)npairs * 4, m->stream));
        if (nF) CSLAM_CUDA(cudaMemsetAsync(match_f, 0xff, (size_t)npairs * nF * 4, m->stream));
        return CSLAM_OK;
    }
    return bow_launch(m, descKF, angKF, kf_valid, node_kf, nKF, descF, angF, node_f, nF, nullptr, npairs, nnratio, check_ori, match_f, nmatches);
}

extern "C" int cslam_search_by_bow(cslam_matcher* m, const uint8_t* descKF, const float* angKF, const uint8_t* kf_valid, const int32_t* node_kf, int nKF,
                                   const uint8_t* descF, const float* angF, const int32_t* node_f, int nF, int npairs, float nnratio, int check_ori, int32_t* match_f,
                                   int32_t* nmatches) {
    int rc = check_sizes(m, nKF, nF, npairs);
    if (rc) return rc;
    const size_t nk = (size_t)npairs * nKF, nf = (size_t)npairs * nF;
    if (!node_ids_ok(node_kf, nk) || !node_ids_ok(node_f, nf)) { set_error("cslam_search_by_bow: node ids must be in [-1, 2^20 - 1)"); return CSLAM_E_BADARG; }
    m->arena.reset();
    const uint8_t *dK, *dValid, *dF; const float *aK, *aF; const int32_t *nodeK, *nodeF; int32_t *dMatch, *dN;
    if ((rc = m->arena.upload(&dK, descKF, nk * 32)) || (rc = m->arena.upload(&aK, angKF, nk)) || (rc = m->arena.upload(&dValid, kf_valid, nk)) ||
        (rc = m->arena.upload(&nodeK, node_kf, nk)) || (rc = m->arena.upload(&dF, descF, nf * 32)) || (rc = m->arena.upload(&aF, angF, nf)) ||
        (rc = m->arena.upload(&nodeF, node_f, nf)) || (rc = m->arena.take(&dMatch, nf)) || (rc = m->arena.take(&dN, npairs)) ||
        (rc = cslam_search_by_bow_dev(m, dK, aK, dValid, nodeK, nKF, dF, aF, nodeF, nF, npairs, nnratio, check_ori, dMatch, dN))) return rc;
    if (nf) CSLAM_CUDA(cudaMemcpyAsync(match_f, dMatch, nf * 4, cudaMemcpyDeviceToHost, m->stream));
    CSLAM_CUDA(cudaMemcpyAsync(nmatches, dN, (size_t)npairs * 4, cudaMemcpyDeviceToHost, m->stream));
    return m->sync();
}

extern "C" int cslam_hamming(cslam_matcher* m, const uint8_t* a, const uint8_t* b, int n, int32_t* dist) {
    if (!m || n < 0 || (size_t)n > (size_t)m->maxPairs * m->maxFeat) { set_error("cslam_hamming: n out of range"); return CSLAM_E_BADARG; }
    if (n == 0) return CSLAM_OK;
    CSLAM_CUDA(cudaSetDevice(m->device));
    m->arena.reset();
    const uint8_t *dA, *dB; int32_t* dDist; int rc;
    if ((rc = m->arena.upload(&dA, a, (size_t)n * 32)) || (rc = m->arena.upload(&dB, b, (size_t)n * 32)) || (rc = m->arena.take(&dDist, n))) return rc;
    k_hamming<<<cdiv(n, 256), 256, 0, m->stream>>>(dA, dB, n, dDist);
    m->launches++;
    CSLAM_CUDA(cudaMemcpyAsync(dist, dDist, (size_t)n * 4, cudaMemcpyDeviceToHost, m->stream));
    return m->sync();
}

// ORBMatcher::SearchByBoW(KeyFrame*, KeyFrame*, vector<MapPoint*>&)  (reference src/ORBMatcher.cpp:541-674), host buffers.
extern "C" int cslam_search_by_bow_kf(cslam_matcher* m, const uint8_t* desc1, const float* ang1, const uint8_t* valid1, const int32_t* node1, int n1,
                                      const uint8_t* desc2, const float* ang2, const uint8_t* valid2, const int32_t* node2, int n2, int npairs, float nnratio,
                                      int check_ori, int32_t* match12, int32_t* nmatches) {
    int rc = check_sizes(m, n1, n2, npairs);
    if (rc) return rc;
    if (!node_ids_ok(node1, (size_t)npairs * n1) || !node_ids_ok(node2, (size_t)npairs * n2)) {
        set_error("cslam_search_by_bow_kf: node ids must be in [-1, 2^20 - 1)"); return CSLAM_E_BADARG;
    }
    if (n1 == 0 || n2 == 0) { for (size_t i = 0; i < (size_t)npairs * n1; i++) match12[i] = -1; for (int p = 0; p < npairs; p++) nmatches[p] = 0; return CSLAM_OK; }
    m->arena.reset();
    const size_t k1 = (size_t)npairs * n1, k2 = (size_t)npairs * n2;
    const uint8_t *dD1, *dV1, *dD2, *dV2; const float *dA1, *dA2; const int32_t *dN1, *dN2; int32_t *dMatch, *dNm;
    if ((rc = m->arena.upload(&dD1, desc1, k1 * 32)) || (rc = m->arena.upload(&dA1, ang1, k1)) || (rc = m->arena.upload(&dV1, valid1, k1)) ||
        (rc = m->arena.upload(&dN1, node1, k1)) || (rc = m->arena.upload(&dD2, desc2, k2 * 32)) || (rc = m->arena.upload(&dA2, ang2, k2)) ||
        (rc = m->arena.upload(&dN2, node2, k2)) || (rc = m->arena.upload(&dV2, valid2, k2)) || (rc = m->arena.take(&dMatch, k1)) || (rc = m->arena.take(&dNm, npairs)) ||
        (rc = bow_launch(m, dD1, dA1, dV1, dN1, n1, dD2, dA2, dN2, n2, dV2, npairs, nnratio, check_ori, dMatch, dNm))) return rc;
    CSLAM_CUDA(cudaMemcpyAsync(match12, dMatch, k1 * 4, cudaMemcpyDeviceToHost, m->stream));
    CSLAM_CUDA(cudaMemcpyAsync(nmatches, dNm, (size_t)npairs * 4, cudaMemcpyDeviceToHost, m->stream));
    return m->sync();
}

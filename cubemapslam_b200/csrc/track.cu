// Per-frame indexing and projection matching of libcubemap_b200.so (the matcher on the steady-state frame path), sm_90a.
//
// Reference (CPU):
//   Frame::ComputeKeyPointRays  src/Frame.cpp:746-760 -> CamModelGeneral::TransformCubemapToRays include/CamModelGeneral.h:494-513
//   Frame::AssignFeaturesToGrid src/Frame.cpp:158-176 (5 x 50 x 50 cells)          -> k_frame_index (one CTA per frame)
//   Frame::GetFeaturesInArea    src/Frame.cpp:251-716 (cube-face wrap-around)      -> area_table.cuh, walked through cube_geom.cuh's area_cells
//   ORBMatcher::SearchByProjection(Frame&, const Frame&, th, mono)   src/ORBMatcher.cpp:130-251 (Tracking::TrackWithMotionModel :634)
//   ORBMatcher::SearchByProjection(Frame&, vector<MapPoint*>&, th)   src/ORBMatcher.cpp:51-128  (Tracking::SearchLocalPoints :841)
//
// k_search_by_projection: one CTA per (frame pair / frame + local map). The reference's loop over MapPoints is sequential - a feature taken by
// an earlier MapPoint (with observations) is invisible to later ones - so the kernel works in rounds of 8 MapPoints: (A) each warp projects
// its MapPoint, walks the window's cells in the reference's visiting order and stores the (feature, Hamming distance) candidates in shared
// memory; (B) one thread commits the 8 MapPoints in order with the reference's scalar best / second-best rule against the `taken` flags.
// Distances dominate the work and stay parallel; the commit touches a few dozen shorts per MapPoint. Hamming distance, rotation bin and
// three-maxima filter: orb_match.cuh.
#include <climits>
#include <cstring>
#include <vector>
#include "area_table.cuh"
#include "common.cuh"
#include "cube_geom.cuh"
#include "orb_match.cuh"

namespace cslam {

static const AreaRect h_area[5][9][3] = AREA_TABLE_INIT;

static const int NCELLS = 5 * GRID_G * GRID_G;
static const int TRK_WARPS = 8;
static const int TRK_CAND = 256;          // candidate capacity per MapPoint (window cells are walked until it is full -> CSLAM_E_CAPACITY)

// ------------------------------------------------------------------------------------------------- k_frame_index
// rays: n x 3 float; cellStart: NCELLS+1 u16 (CSR over cells in (face, col, row) order); cellIdx: n u16, ascending inside a cell
__global__ void __launch_bounds__(256) k_frame_index(const cslam_keypoint* __restrict__ kps, const int32_t* __restrict__ nIn, int kpStride, int W, int H,
                                                     float* __restrict__ rays, uint16_t* __restrict__ cellStart, uint16_t* __restrict__ cellIdx) {
    extern __shared__ uint32_t cnt[];   // NCELLS counters, then scan scratch
    __shared__ uint32_t wsum[8], carry;
    const int f = blockIdx.x, tid = threadIdx.x;
    const int n = min(nIn[f], kpStride);
    const cslam_keypoint* K = kps + (size_t)f * kpStride;
    float* R = rays ? rays + (size_t)f * kpStride * 3 : nullptr;
    uint16_t* CS = cellStart + (size_t)f * (NCELLS + 1);
    uint16_t* CI = cellIdx + (size_t)f * kpStride;
    for (int c = tid; c < NCELLS; c += 256) cnt[c] = 0;
    __syncthreads();
    const float inv = __fdiv_rn((float)(3 * GRID_G), (float)(3 * W));   // mfGridElementLengthInv
    for (int i = tid; i < n; i += 256) {
        const float px = K[i].x, py = K[i].y;
        const int face = face_of_pixel_f(px, py, W, H);
        if (R) {   // TransformCubemapToRays
            float r0 = 0, r1 = 0, r2 = 0;
            if (face >= 0) {
                const double fx = W / 2.0, fy = H / 2.0;
                double di = (double)px, dj = (double)py;
                di = di - (double)((int)(di / W) * W); dj = dj - (double)((int)(dj / H) * H);
                const float lx = (float)((di - fx) * 1.0 / fx), ly = (float)((dj - fy) * 1.0 / fy), lz = 1.0f;
                float p0, p1, p2;
                switch (face) {
                    case FACE_FRONT: p0 = lx; p1 = ly; p2 = lz; break;
                    case FACE_LEFT: p0 = -lz; p1 = ly; p2 = lx; break;
                    case FACE_RIGHT: p0 = lz; p1 = ly; p2 = -lx; break;
                    case FACE_LOWER: p0 = lx; p1 = lz; p2 = -ly; break;
                    default: p0 = lx; p1 = -lz; p2 = ly; break;
                }
                const double nrm = sqrt(__dadd_rn(__dadd_rn(__dmul_rn((double)p0, (double)p0), __dmul_rn((double)p1, (double)p1)), __dmul_rn((double)p2, (double)p2)));
                const double s = nrm > 0 ? 1. / nrm : 0.;
                r0 = (float)((double)p0 * s); r1 = (float)((double)p1 * s); r2 = (float)((double)p2 * s);
            }
            R[3 * i] = r0; R[3 * i + 1] = r1; R[3 * i + 2] = r2;
        }
        if (face >= 0) {   // PosInGrid (src/Frame.cpp:728-744)
            const int posX = (int)__fmul_rn(px, inv) % GRID_G, posY = (int)__fmul_rn(py, inv) % GRID_G;
            atomicAdd(&cnt[(face * GRID_G + posX) * GRID_G + posY], 1u);
        }
    }
    __syncthreads();
    // exclusive scan of the cell counts (block-wide, 256 per pass)
    if (tid == 0) carry = 0;
    __syncthreads();
    for (int base = 0; base < NCELLS; base += 256) {
        const int c = base + tid;
        const uint32_t x = c < NCELLS ? cnt[c] : 0;
        uint32_t s = x;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) { const uint32_t t = __shfl_up_sync(0xffffffffu, s, o); if ((tid & 31) >= o) s += t; }
        if ((tid & 31) == 31) wsum[tid >> 5] = s;
        __syncthreads();
        uint32_t pre = carry;
        for (int w = 0; w < (tid >> 5); w++) pre += wsum[w];
        const uint32_t excl = pre + s - x;
        __syncthreads();
        if (c < NCELLS) { CS[c] = (uint16_t)excl; cnt[c] = excl; }   // cnt becomes the running fill cursor
        if (tid == 255) carry = excl + x;
        __syncthreads();
    }
    if (tid == 0) CS[NCELLS] = (uint16_t)carry;
    __syncthreads();
    for (int i = tid; i < n; i += 256) {
        const float px = K[i].x, py = K[i].y;
        const int face = face_of_pixel_f(px, py, W, H);
        if (face < 0) continue;
        const int posX = (int)__fmul_rn(px, inv) % GRID_G, posY = (int)__fmul_rn(py, inv) % GRID_G;
        CI[atomicAdd(&cnt[(face * GRID_G + posX) * GRID_G + posY], 1u)] = (uint16_t)i;
    }
    __syncthreads();
    // ascending feature index inside every cell (the reference pushes i = 0..N-1); cells hold a handful of entries
    for (int c = tid; c < NCELLS; c += 256) {
        const int s = CS[c], e = (c + 1 < NCELLS) ? CS[c + 1] : (int)carry;
        for (int a = s + 1; a < e; a++) { const uint16_t v = CI[a]; int b = a - 1; while (b >= s && CI[b] > v) { CI[b + 1] = CI[b]; b--; } CI[b + 1] = v; }
    }
}

// ------------------------------------------------------------------------------------------------- projection matchers
struct TrackArgs {
    // current frame (the one searched)
    const cslam_keypoint* kCur; const uint8_t* dCur; const int32_t* nCur; const uint16_t* cellStart; const uint16_t* cellIdx; const uint8_t* curTaken; int curStride;
    // query side: LastFrame features (mode 0) or local MapPoints (mode 1)
    const int32_t* nQ; int qStride;
    const uint8_t* qValid;      // mode 0: has a MapPoint that is not an outlier; mode 1: mbTrackInView && !isBad
    const uint8_t* qDesc;       // MapPoint descriptors
    const uint8_t* qObs;        // Observations() > 0
    const float* qXw; const cslam_keypoint* kLast; const float* TcwCur;   // mode 0
    const float* qProj; const int32_t* qLevel; const float* qViewCos;     // mode 1
    int mode, W, H, checkOri; float th, nnratio, cosFovTh; float scale[16];
    int32_t* match; int32_t* nmatches; int* errFlag;
    uint32_t* lmList; uint16_t* lmCount;   // k_local_candidates -> k_local_commit: LM_K packed entries and the candidate count per (frame, MapPoint)
};

// Mode 1's window of the MapPoint in row `row` (scale: A.scale or a copy): RadiusByViewingCos (src/ORBMatcher.cpp:380-386), times th unless th == 1, times the scale of
// the predicted level; levels [level - 1, level]
__device__ __forceinline__ void local_window(const TrackArgs& A, const float* scale, size_t row, float& u, float& v, float& radius, int& minL, int& maxL) {
    u = A.qProj[row * 2]; v = A.qProj[row * 2 + 1];
    const int lvl = A.qLevel[row];
    float r = A.qViewCos[row] > 0.998 ? 2.5f : 4.0f;   // float compared with the double literal 0.998
    if (A.th != 1.0f) r = __fmul_rn(r, A.th);
    radius = __fmul_rn(r, scale[lvl]); minL = lvl - 1; maxL = lvl;
}

// Frame::GetFeaturesInArea for one query, walked by the calling warp: the window's cells in the reference's visiting order (area_cells; entries
// ascending inside a cell), the level and radius gates, and the Hamming distance to the query's descriptor qd. The candidates go to cIdx / cDist
// in visiting order; returns their number (warp-uniform). More than TRK_CAND candidates, or more than 16 in one cell, sets CSLAM_E_CAPACITY.
__device__ __forceinline__ int window_candidates(const cslam_keypoint* kC, const uint4* dC, const uint16_t* CS, const uint16_t* CI, float u, float v, float radius, int minL,
                                                 int maxL, int W, int H, float inv, const uint4* qd, uint16_t* cIdx, uint16_t* cDist, int* errFlag) {
    const int lane = threadIdx.x & 31;
    int ncand = 0;
    AreaQuery aq;
    if (!area_query(u, v, radius, W, H, inv, aq)) return 0;
    const bool checkLevels = (minL > 0) || (maxL >= 0);
    const uint4 a0 = __ldg(qd), a1 = __ldg(qd + 1);
    for (int k = 0; k < 3; k++) {
        AreaCells rc;
        if (!area_cells(aq, k, rc)) break;
        for (int cb = 0; cb < rc.n; cb += 32) {   // lanes = consecutive cells (ix major, iy minor), entries kept in cell order
            const int ci = cb + lane;
            int s = 0, e = 0;
            if (ci < rc.n) { const int cell = rc.cell(ci); s = CS[cell]; e = CS[cell + 1]; }
            // walk the (few) entries of the 32 cells in order
            const int maxLen = __reduce_max_sync(0xffffffffu, e - s);
            if (maxLen == 0) continue;
            // per lane: filter its cell's entries, then order-preserving append
            int myKeep = 0; uint16_t keepIdx[16];   // a 13-px cell with more than 16 passing key points is reported, never truncated silently
            bool slow = false;
            for (int a = s; a < e; a++) {
                const int idx = CI[a];
                const cslam_keypoint kp = kC[idx];
                if (checkLevels) { if (kp.octave < minL) continue; if (maxL >= 0 && kp.octave > maxL) continue; }
                if (fabsf(__fsub_rn(kp.x, u)) < radius && fabsf(__fsub_rn(kp.y, v)) < radius) { if (myKeep < 16) keepIdx[myKeep] = (uint16_t)idx; else slow = true; myKeep++; }
            }
            if (__any_sync(0xffffffffu, slow)) { if (lane == 0) *errFlag = CSLAM_E_CAPACITY; myKeep = min(myKeep, 16); }
            int off = myKeep;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) { const int t = __shfl_up_sync(0xffffffffu, off, o); if (lane >= o) off += t; }
            const int tot = __shfl_sync(0xffffffffu, off, 31);
            off -= myKeep;
            for (int j = 0; j < myKeep; j++) {
                const int pos = ncand + off + j;
                if (pos < TRK_CAND) {
                    const int idx = keepIdx[j];
                    cIdx[pos] = (uint16_t)idx;
                    cDist[pos] = (uint16_t)hamming256(a0, a1, __ldg(dC + 2 * idx), __ldg(dC + 2 * idx + 1));
                } else *errFlag = CSLAM_E_CAPACITY;
            }
            ncand = min(ncand + tot, TRK_CAND);
        }
    }
    return ncand;
}

// The reference's scalar scan over one query's candidates in visiting order, skipping taken slots: `dist < bestDist` shifts the best to
// second place; with `second` (mode 1) `else if (dist < bestDist2)` replaces the second. No candidate: dist 256, level -1.
struct Best { int dist, level, dist2, level2, idx; };
__device__ __forceinline__ Best best_two(const uint16_t* cIdx, const uint16_t* cDist, int nc, const uint8_t* slotObs, const cslam_keypoint* kC, bool second) {
    Best b = {256, -1, 256, -1, -1};
    for (int c = 0; c < nc; c++) {
        const int idx = cIdx[c];
        if (slotObs[idx]) continue;
        const int dist = cDist[c];
        if (dist < b.dist) { b.dist2 = b.dist; b.dist = dist; b.level2 = b.level; b.level = kC[idx].octave; b.idx = idx; }
        else if (second && dist < b.dist2) { b.level2 = kC[idx].octave; b.dist2 = dist; }
    }
    return b;
}
// mode 1's ratio test (src/ORBMatcher.cpp:111-112): only when the best and the second best are at the same level
__device__ __forceinline__ bool ratio_ok(const Best& b, float nnratio) { return !(b.level == b.level2 && (float)b.dist > __fmul_rn(nnratio, (float)b.dist2)); }

__global__ void __launch_bounds__(TRK_WARPS * 32) k_search_by_projection(TrackArgs A) {
    __shared__ uint16_t candIdx[TRK_WARPS][TRK_CAND];
    __shared__ uint16_t candDist[TRK_WARPS][TRK_CAND];
    __shared__ int candN[TRK_WARPS];
    __shared__ uint8_t slotObs[4096];
    __shared__ int hist[HISTO_BINS], keep[HISTO_BINS], total, logN;
    __shared__ uint16_t logIdx[4096];   // mode 0: every accepted assignment (current slot, rotation bin), replayed by the orientation filter
    __shared__ uint8_t logBin[4096];
    const int p = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int nCur = min(A.nCur[p], A.curStride), nQ = min(A.nQ[p], A.qStride);
    const cslam_keypoint* kC = A.kCur + (size_t)p * A.curStride;
    const uint4* dC = reinterpret_cast<const uint4*>(A.dCur + (size_t)p * A.curStride * 32);
    const uint16_t* CS = A.cellStart + (size_t)p * (NCELLS + 1);
    const uint16_t* CI = A.cellIdx + (size_t)p * A.curStride;
    const uint4* dQ = reinterpret_cast<const uint4*>(A.qDesc + (size_t)p * A.qStride * 32);
    int32_t* M = A.match + (size_t)p * A.curStride;
    for (int i = tid; i < nCur; i += blockDim.x) { M[i] = -1; slotObs[i] = A.curTaken ? A.curTaken[(size_t)p * A.curStride + i] : 0; }
    if (tid < HISTO_BINS) hist[tid] = 0;
    if (tid == 0) { total = 0; logN = 0; }
    __syncthreads();
    const float inv = __fdiv_rn((float)(3 * GRID_G), (float)(3 * A.W));
    float Tc[12];
    if (A.mode == 0) for (int i = 0; i < 12; i++) Tc[i] = A.TcwCur[(size_t)p * 16 + i];
    for (int q0 = 0; q0 < nQ; q0 += TRK_WARPS) {
        // ---- (A) candidates of MapPoint q = q0 + warp, in the reference's visiting order
        const int q = q0 + warp;
        int ncand = 0;
        if (q < nQ && A.qValid[(size_t)p * A.qStride + q]) {
            float u = 0, v = 0, radius = 0; int minL = 0, maxL = 0; bool ok = true;
            if (A.mode == 0) {
                float xc[3];
                transform_cw(Tc, A.qXw + ((size_t)p * A.qStride + q) * 3, xc);   // `Rcw*x3Dw+tcw`
                if (xc[2] < A.cosFovTh) ok = false;
                if (ok) ok = ray_to_cubemap(xc[0], xc[1], xc[2], A.W, A.H, u, v);
                const int oct = A.kLast[(size_t)p * A.qStride + q].octave;
                radius = __fmul_rn(A.th, A.scale[oct]); minL = oct - 1; maxL = oct + 1;
            } else local_window(A, A.scale, (size_t)p * A.qStride + q, u, v, radius, minL, maxL);
            if (ok) ncand = window_candidates(kC, dC, CS, CI, u, v, radius, minL, maxL, A.W, A.H, inv, dQ + 2 * q, candIdx[warp], candDist[warp], A.errFlag);
        }
        if (lane == 0) candN[warp] = ncand;
        __syncthreads();
        // ---- (B) commit in MapPoint order (one thread; the reference's scalar rules)
        if (tid == 0) {
            for (int w = 0; w < TRK_WARPS; w++) {
                const int qq = q0 + w, nc = candN[w];
                if (qq >= nQ || nc == 0) continue;
                const Best b = best_two(candIdx[w], candDist[w], nc, slotObs, kC, A.mode == 1);
                if (b.dist > 100) continue;   // TH_HIGH
                if (A.mode == 1 && !ratio_ok(b, A.nnratio)) continue;
                const int bestIdx = b.idx;
                M[bestIdx] = qq; slotObs[bestIdx] = A.qObs[(size_t)p * A.qStride + qq];
                total++;
                if (A.mode == 0 && A.checkOri) {
                    const int bin = rot_bin(A.kLast[(size_t)p * A.qStride + qq].angle, kC[bestIdx].angle);
                    hist[bin]++;
                    if (logN < 4096) { logIdx[logN] = (uint16_t)bestIdx; logBin[logN] = (uint8_t)bin; logN++; } else *A.errFlag = CSLAM_E_CAPACITY;
                }
            }
        }
        __syncthreads();
    }
    if (A.mode == 0 && A.checkOri) {
        // the reference keeps per-bin lists of CURRENT feature indices (a slot overwritten by a later, observation-less MapPoint is listed twice)
        // and clears every slot listed in a non-dominant bin, decrementing nmatches per list entry: the assignment log is replayed.
        if (tid == 0) three_maxima(hist, keep);
        __syncthreads();
        for (int i = tid; i < logN; i += blockDim.x)
            if (!keep[logBin[i]]) { M[logIdx[i]] = -2; atomicSub(&total, 1); }   // -2: assigned, then cleared (the reference NULLs the slot)
        __syncthreads();
    }
    if (tid == 0) A.nmatches[p] = total;
}

// ------------------------------------------------------------------------------------------------- local maps past 4096 MapPoints
// cslam_search_by_projection_local_large in two launches (DESIGN.md, "Local maps past 4096 MapPoints"):
//   k_local_candidates: one warp per (frame, MapPoint) over the whole device walks the window (window_candidates) and keeps the first LM_K
//     candidates in (distance, visiting position) order, packed, plus the full candidate count.
//   k_local_commit: one CTA per frame applies the reference's rules in MapPoint order. The first two untaken entries of that order are the
//     scan's best and second best, so a MapPoint needs nothing else unless fewer than two of its stored entries are untaken while it has more
//     than LM_K candidates: then the committing warp walks the window again and runs the scan itself (best_two).
static const int LM_K = 8;        // stored entries per MapPoint: a performance choice, the answer does not depend on it
static const int LM_CHUNK = 256;  // MapPoints per staged chunk of the commit

// entry = feature (12 bits) | distance << 12 (9 bits) | octave << 21 (a signed byte)
__device__ __forceinline__ uint32_t lm_pack(int idx, int dist, int octave) { return (uint32_t)idx | (uint32_t)dist << 12 | (uint32_t)(octave & 0xff) << 21; }

__global__ void __launch_bounds__(TRK_WARPS * 32) k_local_candidates(TrackArgs A, int nframes) {
    __shared__ uint16_t candIdx[TRK_WARPS][TRK_CAND];
    __shared__ uint16_t candDist[TRK_WARPS][TRK_CAND];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int q = blockIdx.x * TRK_WARPS + warp;
    const float inv = __fdiv_rn((float)(3 * GRID_G), (float)(3 * A.W));
    uint16_t* cI = candIdx[warp]; uint16_t* cD = candDist[warp];
    for (int p = blockIdx.y; p < nframes; p += gridDim.y) {
        if (q >= min(A.nQ[p], A.qStride)) continue;
        const size_t row = (size_t)p * A.qStride + q;
        const cslam_keypoint* kC = A.kCur + (size_t)p * A.curStride;
        int nc = 0;
        __syncwarp();   // the previous frame's reads of cI / cD are done
        if (A.qValid[row]) {
            float u, v, radius; int minL, maxL;
            local_window(A, A.scale, row, u, v, radius, minL, maxL);
            nc = window_candidates(kC, reinterpret_cast<const uint4*>(A.dCur + (size_t)p * A.curStride * 32), A.cellStart + (size_t)p * (NCELLS + 1),
                                   A.cellIdx + (size_t)p * A.curStride, u, v, radius, minL, maxL, A.W, A.H, inv, reinterpret_cast<const uint4*>(A.qDesc) + 2 * row, cI, cD,
                                   A.errFlag);
        }
        __syncwarp();
        // selection by key = distance << 8 | position (unique), LM_K rounds of a warp minimum above the previous round's key
        int last = -1;
        for (int j = 0; j < min(nc, LM_K); j++) {
            unsigned mn = 0xffffffffu;
            for (int c = lane; c < nc; c += 32) { const unsigned key = (unsigned)cD[c] << 8 | (unsigned)c; if ((int)key > last && key < mn) mn = key; }
            mn = __reduce_min_sync(0xffffffffu, mn);
            last = (int)mn;
            if (lane == 0) { const int pos = mn & 0xff, idx = cI[pos]; A.lmList[row * LM_K + j] = lm_pack(idx, cD[pos], kC[idx].octave); }
        }
        if (lane == 0) A.lmCount[row] = (uint16_t)nc;
    }
}

// chunk c of a frame's MapPoints (rows row0 + c * LM_CHUNK ...) into one buffer of the commit, by threads t0, t0 + nt, ...
__device__ __forceinline__ void lm_stage(const TrackArgs& A, size_t row0, int nQ, int c, int t0, int nt, uint32_t* list, uint16_t* cnt, uint8_t* obs) {
    const int q0 = c * LM_CHUNK, n = min(LM_CHUNK, nQ - q0);
    for (int i = t0; i < n * LM_K; i += nt) list[i] = A.lmList[(row0 + q0) * LM_K + i];
    for (int i = t0; i < n; i += nt) { cnt[i] = A.lmCount[row0 + q0 + i]; obs[i] = A.qObs[row0 + q0 + i]; }
}

// The reference's scan over the whole window of the MapPoint in row `row` of frame p, walked again by the calling warp. scale: A.scale in
// shared memory (indexed by level, a kernel parameter array would be copied to local memory)
__device__ __forceinline__ Best lm_rewalk(const TrackArgs& A, const float* scale, int p, size_t row, const uint8_t* slotObs, uint16_t* candIdx, uint16_t* candDist) {
    const cslam_keypoint* kC = A.kCur + (size_t)p * A.curStride;
    float u, v, radius; int minL, maxL;
    local_window(A, scale, row, u, v, radius, minL, maxL);
    const int nc = window_candidates(kC, reinterpret_cast<const uint4*>(A.dCur + (size_t)p * A.curStride * 32), A.cellStart + (size_t)p * (NCELLS + 1),
                                     A.cellIdx + (size_t)p * A.curStride, u, v, radius, minL, maxL, A.W, A.H, __fdiv_rn((float)(3 * GRID_G), (float)(3 * A.W)),
                                     reinterpret_cast<const uint4*>(A.qDesc) + 2 * row, candIdx, candDist, A.errFlag);
    __syncwarp();
    return best_two(candIdx, candDist, nc, slotObs, kC, true);
}

__global__ void __launch_bounds__(TRK_WARPS * 32, 1) k_local_commit(TrackArgs A) {
    __shared__ uint32_t list[2][LM_CHUNK * LM_K];   // double-buffered: warp 0 commits one chunk while the other warps stage the next
    __shared__ uint16_t cnt[2][LM_CHUNK];
    __shared__ uint8_t obs[2][LM_CHUNK];
    __shared__ uint8_t slotObs[4096];
    __shared__ uint16_t candIdx[TRK_CAND], candDist[TRK_CAND];   // warp 0's window walk when the stored entries run out
    __shared__ float sScale[16];
    const int p = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int nCur = min(A.nCur[p], A.curStride), nQ = max(0, min(A.nQ[p], A.qStride)), nChunks = (nQ + LM_CHUNK - 1) / LM_CHUNK;
    const cslam_keypoint* kC = A.kCur + (size_t)p * A.curStride;
    int32_t* M = A.match + (size_t)p * A.curStride;
    const size_t row0 = (size_t)p * A.qStride;
    for (int i = tid; i < A.curStride; i += blockDim.x) { M[i] = -1; if (i < nCur) slotObs[i] = A.curTaken[(size_t)p * A.curStride + i]; }
    if (tid < 16) sScale[tid] = A.scale[tid];
    if (nChunks > 0) lm_stage(A, row0, nQ, 0, tid, blockDim.x, list[0], cnt[0], obs[0]);
    __syncthreads();
    int total = 0;   // warp 0
    for (int c = 0; c < nChunks; c++) {
        const int b = c & 1, q0 = c * LM_CHUNK, n = min(LM_CHUNK, nQ - q0);
        if (warp != 0) {
            if (c + 1 < nChunks) lm_stage(A, row0, nQ, c + 1, tid - 32, blockDim.x - 32, list[b ^ 1], cnt[b ^ 1], obs[b ^ 1]);
        } else {
            for (int j = 0; j < n; j++) {
                const int nc = cnt[b][j];
                if (nc == 0) continue;
                const int ns = min(nc, LM_K);
                const uint32_t e = lane < ns ? list[b][j * LM_K + lane] : 0u;
                const unsigned fr = __ballot_sync(0xffffffffu, lane < ns && !slotObs[e & 0xfff]);
                Best best = {256, -1, 256, -1, -1};
                if (__popc(fr) < 2 && nc > LM_K) {   // the untaken entries may lie past the stored ones: the reference's scan over the whole window
                    best = lm_rewalk(A, sScale, p, row0 + q0 + j, slotObs, candIdx, candDist);
                    __syncwarp();   // every lane has read candIdx / candDist before the next walk overwrites them
                } else if (fr) {
                    const uint32_t e1 = __shfl_sync(0xffffffffu, e, __ffs(fr) - 1);
                    best.idx = e1 & 0xfff; best.dist = (e1 >> 12) & 0x1ff; best.level = (int8_t)(e1 >> 21);
                    const unsigned rest = fr & (fr - 1);
                    if (rest) { const uint32_t e2 = __shfl_sync(0xffffffffu, e, __ffs(rest) - 1); best.dist2 = (e2 >> 12) & 0x1ff; best.level2 = (int8_t)(e2 >> 21); }
                }
                if (best.dist > 100 || !ratio_ok(best, A.nnratio)) continue;   // TH_HIGH, ratio test
                if (lane == 0) { M[best.idx] = q0 + j; slotObs[best.idx] = obs[b][j]; }
                total++;
                __syncwarp();   // the slot's new state is visible to every lane before the next MapPoint
            }
        }
        __syncthreads();
    }
    if (tid == 0) A.nmatches[p] = total;
}

// ------------------------------------------------------------------------------------------------- SearchForInitialization
// cslam_search_for_initialization in four launches after F2's frame index (DESIGN.md, "SearchForInitialization"):
//   k_init_candidates (count): one warp per F1 key point counts its window's candidates (level-0 F2 key points inside the strict |dx|, |dy| < r gate);
//   k_init_scan: the counts become list offsets; the host reads the total and takes exactly that much scratch from the arena;
//   k_init_candidates (fill): the same walk stores every candidate as (F2 index, Hamming distance) in visiting order - no window or cell cap;
//   k_init_commit: one CTA applies the reference's rules in i1 order over the stored lists, then the rotation-consistency filter.
static const int INIT_WARPS = 8;
static const int INIT_CHUNK = 64;        // queries per staged chunk of the commit
static const int INIT_STAGE = 8192;      // entries staged per chunk; a list past them is read from global memory (the answer does not depend on it)

// entry = F2 index (14 bits) | distance << 14 (9 bits); the position in the list is the visiting position
__device__ __forceinline__ uint32_t init_pack(int idx, int dist) { return (uint32_t)idx | (uint32_t)dist << 14; }

// The window of query i1 walked by the calling warp (area_query / area_cells, the reference's visiting order, entries ascending inside a cell),
// with the level and radius gates of window_candidates. list == nullptr: returns the number of candidates (warp-uniform). Otherwise writes them
// to list[0, count) in visiting order. Lanes take consecutive cells; each lane counts its cell's passing entries, a warp scan places them, and
// the lane walks its cell again to write: nothing is held per lane, so no cell or window size is too large.
__device__ int init_window(const cslam_keypoint* kC, const uint4* dC, const uint16_t* CS, const uint16_t* CI, float u, float v, float radius, int minL, int maxL,
                           int W, int H, float inv, const uint4* qd, uint32_t* list) {
    const int lane = threadIdx.x & 31;
    int ncand = 0;
    AreaQuery aq;
    if (!area_query(u, v, radius, W, H, inv, aq)) return 0;
    const bool checkLevels = (minL > 0) || (maxL >= 0);
    uint4 a0 = make_uint4(0, 0, 0, 0), a1 = a0;
    if (list) { a0 = __ldg(qd); a1 = __ldg(qd + 1); }
    for (int k = 0; k < 3; k++) {
        AreaCells rc;
        if (!area_cells(aq, k, rc)) break;
        for (int cb = 0; cb < rc.n; cb += 32) {
            const int ci = cb + lane;
            int s = 0, e = 0;
            if (ci < rc.n) { const int cell = rc.cell(ci); s = CS[cell]; e = CS[cell + 1]; }
            if (__reduce_max_sync(0xffffffffu, e - s) == 0) continue;
            int mine = 0;
            for (int pass = 0; pass < (list ? 2 : 1); pass++) {
                int off = 0, tot = 0;
                if (pass == 1) {
                    off = mine;
#pragma unroll
                    for (int o = 1; o < 32; o <<= 1) { const int t = __shfl_up_sync(0xffffffffu, off, o); if (lane >= o) off += t; }
                    off -= mine;
                }
                for (int a = s; a < e; a++) {
                    const int idx = CI[a];
                    const cslam_keypoint kp = kC[idx];
                    if (checkLevels) { if (kp.octave < minL) continue; if (maxL >= 0 && kp.octave > maxL) continue; }
                    if (!(fabsf(__fsub_rn(kp.x, u)) < radius && fabsf(__fsub_rn(kp.y, v)) < radius)) continue;
                    if (pass == 0) mine++;
                    else list[ncand + off + tot++] = init_pack(idx, hamming256(a0, a1, __ldg(dC + 2 * idx), __ldg(dC + 2 * idx + 1)));
                }
            }
            ncand += __reduce_add_sync(0xffffffffu, (unsigned)mine);
        }
    }
    return ncand;
}

// count pass (list == nullptr): cnt[i1] = candidates of query i1; fill pass: list + off[i1] gets them. Only level-0 F1 key points search
// (`if (level1 > 0) continue`; the host rejects negative octaves), in F2's level-0 key points (GetFeaturesInArea(.., level1, level1)).
__global__ void __launch_bounds__(INIT_WARPS * 32) k_init_candidates(const cslam_keypoint* __restrict__ k1, const uint8_t* __restrict__ d1, const float* __restrict__ pos,
                                                                     int n1, const cslam_keypoint* __restrict__ k2, const uint8_t* __restrict__ d2, const uint16_t* __restrict__ CS,
                                                                     const uint16_t* __restrict__ CI, int W, int H, float radius, uint32_t* __restrict__ cnt,
                                                                     const uint32_t* __restrict__ off, uint32_t* __restrict__ list) {
    const int i1 = blockIdx.x * INIT_WARPS + (threadIdx.x >> 5);
    if (i1 >= n1) return;
    int nc = 0;
    if (k1[i1].octave == 0) {
        const float inv = __fdiv_rn((float)(3 * GRID_G), (float)(3 * W));
        nc = init_window(k2, reinterpret_cast<const uint4*>(d2), CS, CI, pos[2 * i1], pos[2 * i1 + 1], radius, 0, 0, W, H, inv,
                         reinterpret_cast<const uint4*>(d1) + 2 * i1, list ? list + off[i1] : nullptr);
    }
    if (!list && (threadIdx.x & 31) == 0) cnt[i1] = (uint32_t)nc;
}

// exclusive scan of cnt[0, n) in place into off[0, n]; one CTA of 1024 threads, n <= CSLAM_BOW_FV_MAX_FEATURES
__global__ void __launch_bounds__(1024) k_init_scan(uint32_t* __restrict__ off, int n) {
    __shared__ uint32_t wsum[32];
    const int tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
    const int per = (n + 1023) / 1024, b = tid * per, e = min(n, b + per);
    uint32_t s = 0;
    for (int i = b; i < e; i++) s += off[i];
    uint32_t x = s;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const uint32_t t = __shfl_up_sync(0xffffffffu, x, o); if (lane >= o) x += t; }
    if (lane == 31) wsum[w] = x;
    __syncthreads();
    uint32_t pre = x - s;
    for (int ww = 0; ww < w; ww++) pre += wsum[ww];
    for (int i = b; i < e; i++) { const uint32_t c = off[i]; off[i] = pre; pre += c; }
    if (tid == 1023) off[n] = pre;
}

// staging of chunk c (queries c*INIT_CHUNK ...) by threads t0, t0 + nt, ...: its offsets, and its first INIT_STAGE entries
__device__ __forceinline__ void init_stage(const uint32_t* off, const uint32_t* list, int n1, int c, int t0, int nt, uint32_t* sOff, uint32_t* sList) {
    const int q0 = c * INIT_CHUNK, nq = min(INIT_CHUNK, n1 - q0);
    for (int i = t0; i <= nq; i += nt) sOff[i] = off[q0 + i];
    const uint32_t e0 = off[q0], ne = umin(off[q0 + nq] - e0, (uint32_t)INIT_STAGE);
    for (uint32_t i = t0; i < ne; i += nt) sList[i] = list[e0 + i];
}

// Shared memory of k_init_commit: vMatchedDistance (u16, 0xffff = INT_MAX) and vnMatches21 (i16) per F2 key point, vnMatches12 (i16) and the
// rotation bin (u8, 0xff: never pushed) per F1 key point, then two staging buffers of offsets and entries
static const size_t INIT_SMEM = (size_t)CSLAM_BOW_FV_MAX_FEATURES * (2 + 2 + 2 + 1) + 2 * (INIT_CHUNK + 1) * 4 + 2 * INIT_STAGE * 4;

// The reference's scan of query i1 ends with best and second best = the first two eligible entries (vMatchedDistance[i2] > dist) in (distance,
// visiting position) order: both comparisons are strict, and the eligibility of an entry cannot change while i1 is scanned. Warp 0 takes them
// as two warp minima of the key distance << 16 | position, applies the acceptance rules of orb_match.cuh and commits, query after query.
__global__ void __launch_bounds__(INIT_WARPS * 32, 1) k_init_commit(const cslam_keypoint* __restrict__ k1, int n1, const cslam_keypoint* __restrict__ k2, int n2,
                                                                    const uint32_t* __restrict__ off, const uint32_t* __restrict__ list, float nnratio, int checkOri,
                                                                    int32_t* __restrict__ match12, int32_t* __restrict__ nmatches) {
    extern __shared__ __align__(16) uint8_t smem[];
    uint32_t* sList = reinterpret_cast<uint32_t*>(smem);                           // [2][INIT_STAGE]
    uint32_t* sOff = sList + 2 * INIT_STAGE;                                          // [2][INIT_CHUNK + 1]
    uint16_t* mdist = reinterpret_cast<uint16_t*>(sOff + 2 * (INIT_CHUNK + 1));      // [n2]
    int16_t* owner = reinterpret_cast<int16_t*>(mdist + CSLAM_BOW_FV_MAX_FEATURES);   // [n2]
    int16_t* m12 = owner + CSLAM_BOW_FV_MAX_FEATURES;                                  // [n1]
    uint8_t* bin = reinterpret_cast<uint8_t*>(m12 + CSLAM_BOW_FV_MAX_FEATURES);       // [n1]
    __shared__ int hist[HISTO_BINS], keep[HISTO_BINS], total;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nChunks = (n1 + INIT_CHUNK - 1) / INIT_CHUNK;
    for (int i = tid; i < n2; i += blockDim.x) { mdist[i] = 0xffff; owner[i] = -1; }
    for (int i = tid; i < n1; i += blockDim.x) { m12[i] = -1; bin[i] = 0xff; }
    if (tid < HISTO_BINS) hist[tid] = 0;
    if (tid == 0) total = 0;
    if (nChunks > 0) init_stage(off, list, n1, 0, tid, blockDim.x, sOff, sList);
    __syncthreads();
    for (int c = 0; c < nChunks; c++) {
        const int b = c & 1, q0 = c * INIT_CHUNK, nq = min(INIT_CHUNK, n1 - q0);
        if (warp != 0) {
            if (c + 1 < nChunks) init_stage(off, list, n1, c + 1, tid - 32, blockDim.x - 32, sOff + (b ^ 1) * (INIT_CHUNK + 1), sList + (b ^ 1) * INIT_STAGE);
        } else {
            const uint32_t* so = sOff + b * (INIT_CHUNK + 1); const uint32_t* sl = sList + b * INIT_STAGE;
            for (int j = 0; j < nq; j++) {
                const uint32_t s = so[j] - so[0], n = so[j + 1] - so[j];
                if (n == 0) continue;
                const uint32_t* L = s + n <= (uint32_t)INIT_STAGE ? sl + s : list + so[j];
                uint32_t m1 = 0xffffffffu, m2 = 0xffffffffu;   // this lane's two smallest eligible keys
                for (uint32_t p = lane; p < n; p += 32) {
                    const uint32_t e = L[p], dist = e >> 14;
                    if (mdist[e & 0x3fff] <= dist) continue;   // `if (vMatchedDistance[i2] <= dist) continue`
                    const uint32_t key = dist << 16 | p;
                    if (key < m1) { m2 = m1; m1 = key; } else if (key < m2) m2 = key;
                }
                const uint32_t best = __reduce_min_sync(0xffffffffu, m1);
                const uint32_t second = __reduce_min_sync(0xffffffffu, m1 == best ? m2 : m1);
                const int bestDist = best == 0xffffffffu ? INT_MAX : (int)(best >> 16), bestDist2 = second == 0xffffffffu ? INT_MAX : (int)(second >> 16);
                if (!bow_accept(bestDist, bestDist2, nnratio, false)) continue;   // bestDist <= TH_LOW, bestDist < (float)bestDist2 * mfNNratio
                if (lane == 0) {
                    const int i1 = q0 + j, i2 = L[best & 0xffff] & 0x3fff;
                    const int prev = owner[i2];
                    if (prev >= 0) { m12[prev] = -1; total--; }
                    m12[i1] = (int16_t)i2; owner[i2] = (int16_t)i1; mdist[i2] = (uint16_t)bestDist; total++;
                    if (checkOri) bin[i1] = (uint8_t)rot_bin(k1[i1].angle, k2[i2].angle);
                }
                __syncwarp();   // the new vMatchedDistance is visible to every lane before the next query
            }
        }
        __syncthreads();
    }
    if (checkOri) {
        // ComputeThreeMaxima over the bin sizes: an i1 whose F2 key point a later i1 took stays in its bin and counts
        for (int i = tid; i < n1; i += blockDim.x) if (bin[i] != 0xff) atomicAdd(&hist[bin[i]], 1);
        __syncthreads();
        if (tid == 0) three_maxima(hist, keep);
        __syncthreads();
        for (int i = tid; i < n1; i += blockDim.x) if (bin[i] != 0xff && !keep[bin[i]] && m12[i] >= 0) { m12[i] = -1; atomicSub(&total, 1); }
        __syncthreads();
    }
    for (int i = tid; i < n1; i += blockDim.x) match12[i] = m12[i];
    if (tid == 0) *nmatches = total;
}

// What Tracking does between SearchByProjection and PoseOptimization (src/Optimizer.cpp:80-131 reads mvpMapPoints / mvKeys / mvKeyRays):
// the matched slots of a frame, in slot order, become the (world point, key point, 1/sigma^2) correspondences of the pose-only BA.
__global__ void __launch_bounds__(256) k_gather_pose_inputs(const int32_t* __restrict__ match, const cslam_keypoint* __restrict__ kCur, const int32_t* __restrict__ nCur, int curStride,
                                                            const float* __restrict__ rays, float cosFovTh, const float* __restrict__ XwLast, int lastStride, const float* invSigma2,
                                                            float* __restrict__ XwOut, float* __restrict__ kpOut, float* __restrict__ wOut, int32_t* __restrict__ count) {
    __shared__ int wcnt[8], base;
    const int p = blockIdx.x, tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
    const int n = min(nCur[p], curStride);
    if (tid == 0) base = 0;
    __syncthreads();
    for (int i0 = 0; i0 < n; i0 += 256) {
        const int i = i0 + tid;
        int m = -1;
        if (i < n) { m = match[(size_t)p * curStride + i]; if (m >= 0 && rays && rays[((size_t)p * curStride + i) * 3 + 2] < cosFovTh) m = -1; }
        const unsigned ball = __ballot_sync(0xffffffffu, m >= 0);
        if (lane == 0) wcnt[w] = __popc(ball);
        __syncthreads();
        int pre = base;
        for (int ww = 0; ww < w; ww++) pre += wcnt[ww];
        if (m >= 0) {
            const size_t o = (size_t)p * curStride + pre + __popc(ball & ((1u << lane) - 1));
            const cslam_keypoint kp = kCur[(size_t)p * curStride + i];
            const float* X = XwLast + ((size_t)p * lastStride + m) * 3;
            XwOut[3 * o] = X[0]; XwOut[3 * o + 1] = X[1]; XwOut[3 * o + 2] = X[2];
            kpOut[2 * o] = kp.x; kpOut[2 * o + 1] = kp.y; wOut[o] = invSigma2[kp.octave];
        }
        __syncthreads();
        if (tid == 0) { int t = 0; for (int ww = 0; ww < 8; ww++) t += wcnt[ww]; base += t; }
        __syncthreads();
    }
    if (tid == 0) count[p] = base;
}

}  // namespace cslam

using namespace cslam;

extern "C" int cslam_tracker_gather_pose_inputs_dev(cslam_tracker* t, int npairs, const int32_t* match_cur, const cslam_keypoint* k_cur, const int32_t* n_cur, int cur_stride,
                                                    const float* rays_cur, float cos_fov_th, const float* Xw_last, int last_stride, const float* inv_sigma2_levels_dev,
                                                    float* Xw_out, float* kp_xy_out, float* inv_sigma2_out, int32_t* count_out);

// ---- host utility (no device needed): the cell rectangles Frame::GetFeaturesInArea visits, for callers that keep the grid on the host
extern "C" int cslam_area_rects(float x, float y, float r, int face_w, int face_h, int32_t* rects /* 3 x 5: face, x0, x1, y0, y1 (unclamped) */) {
    AreaQuery q;
    const float inv = (float)(3 * GRID_G) / (float)(3 * face_w);
    if (!area_query(x, y, r, face_w, face_h, inv, q)) return 0;
    int n = 0;
    for (int k = 0; k < 3; k++) {
        const AreaRect rc = h_area[q.face][q.caseRow][k];
        if (rc.face == FACE_NONE) break;
        rects[5 * n] = rc.face; rects[5 * n + 1] = area_sym(q, rc.x0); rects[5 * n + 2] = area_sym(q, rc.x1); rects[5 * n + 3] = area_sym(q, rc.y0); rects[5 * n + 4] = area_sym(q, rc.y1);
        n++;
    }
    return n;
}

// error flag: CSLAM_E_CAPACITY once a search window overflowed
struct cslam_tracker : cslam::Handle {
    int maxFrames = 0, maxFeat = 0;
};

extern "C" int cslam_tracker_create(cslam_tracker** out, int device, int max_frames, int max_features) {
    if (!out || max_frames <= 0 || max_features <= 0 || max_features > 4096) { set_error("cslam_tracker_create: bad argument (max_features <= 4096)"); return CSLAM_E_BADARG; }
    cslam_tracker* t = new cslam_tracker; t->maxFrames = max_frames; t->maxFeat = max_features;
    // chunks: room for every array the host calls stage at the handle's limits, at most 64 MB
    const size_t perFeature = 2 * sizeof(cslam_keypoint) + 2 * 32 + 3 + 2 * 4 + 3 * 4 + 2 * 4 + 4 + 3 * 4 + 2, perFrame = 3 * 4 + 16 * 4 + (NCELLS + 1) * 2;
    int rc;
    if ((rc = t->open(device, std::min<size_t>((size_t)64 << 20, (size_t)max_frames * max_features * perFeature + (size_t)max_frames * perFrame), true)) ||
        (rc = prepare_frame_index())) { destroy_handle(t); return rc; }
    *out = t;
    return CSLAM_OK;
}
extern "C" void cslam_tracker_destroy(cslam_tracker* t) { destroy_handle(t); }
extern "C" void* cslam_tracker_stream(const cslam_tracker* t) { return t ? (void*)t->stream : nullptr; }
extern "C" int64_t cslam_tracker_launches(const cslam_tracker* t) { return t ? t->launches : 0; }
extern "C" int cslam_tracker_sync(cslam_tracker* t) { return t ? t->sync("tracker: a search window held more candidates than the fixed capacity") : CSLAM_E_BADARG; }

extern "C" int cslam_tracker_gather_pose_inputs_dev(cslam_tracker* t, int npairs, const int32_t* match_cur, const cslam_keypoint* k_cur, const int32_t* n_cur, int cur_stride,
                                                    const float* rays_cur, float cos_fov_th, const float* Xw_last, int last_stride, const float* inv_sigma2_levels_dev,
                                                    float* Xw_out, float* kp_xy_out, float* inv_sigma2_out, int32_t* count_out) {
    if (!t || npairs <= 0 || !match_cur || !k_cur || !n_cur || !Xw_last || !inv_sigma2_levels_dev || !Xw_out || !kp_xy_out || !inv_sigma2_out || !count_out) { set_error("cslam_tracker_gather_pose_inputs_dev: bad argument"); return CSLAM_E_BADARG; }
    CSLAM_CUDA(cudaSetDevice(t->device));
    k_gather_pose_inputs<<<npairs, 256, 0, t->stream>>>(match_cur, k_cur, n_cur, cur_stride, rays_cur, cos_fov_th, Xw_last, last_stride, inv_sigma2_levels_dev, Xw_out, kp_xy_out,
                                                       inv_sigma2_out, count_out);
    t->launches++;
    CSLAM_CUDA(cudaGetLastError());
    return CSLAM_OK;
}

int cslam::prepare_frame_index() {
    CSLAM_CUDA(cudaFuncSetAttribute(k_frame_index, cudaFuncAttributeMaxDynamicSharedMemorySize, NCELLS * 4));
    return CSLAM_OK;
}
int cslam::frame_index(cudaStream_t stream, int64_t& launches, const cslam_keypoint* kps, const int32_t* n, int nframes, int kpStride, int faceW, int faceH, float* rays,
                       uint16_t* cellStart, uint16_t* cellIdx, int maxStride) {
    if (!kps || !n || !cellStart || !cellIdx || nframes <= 0 || kpStride <= 0 || kpStride > maxStride || faceW <= 0 || faceW != faceH) { set_error("cslam_frame_index: bad argument"); return CSLAM_E_BADARG; }
    k_frame_index<<<nframes, 256, NCELLS * 4, stream>>>(kps, n, kpStride, faceW, faceH, rays, cellStart, cellIdx); launches++;
    CSLAM_CUDA(cudaGetLastError());
    return CSLAM_OK;
}

extern "C" int cslam_frame_index_dev(cslam_tracker* t, const cslam_keypoint* kps, const int32_t* n, int nframes, int kp_stride, int face_w, int face_h, float* rays,
                                     uint16_t* cell_start, uint16_t* cell_idx) {
    if (!t) { set_error("cslam_frame_index: bad argument"); return CSLAM_E_BADARG; }
    CSLAM_CUDA(cudaSetDevice(t->device));
    return frame_index(t->stream, t->launches, kps, n, nframes, kp_stride, face_w, face_h, rays, cell_start, cell_idx);
}
extern "C" int cslam_frame_index(cslam_tracker* t, const cslam_keypoint* kps, const int32_t* n, int nframes, int kp_stride, int face_w, int face_h, float* rays, uint16_t* cell_start,
                                 uint16_t* cell_idx) {
    if (!t || nframes <= 0 || nframes > t->maxFrames || kp_stride > t->maxFeat) { set_error("cslam_frame_index: sizes out of range"); return CSLAM_E_BADARG; }
    CSLAM_CUDA(cudaSetDevice(t->device));
    t->arena.reset();
    const size_t nf = (size_t)nframes * kp_stride;
    const cslam_keypoint* dK; const int32_t* dN; float* dR; uint16_t *dCS, *dCI; int rc;
    if ((rc = t->arena.upload(&dK, kps, nf)) || (rc = t->arena.upload(&dN, n, nframes)) || (rc = t->arena.take(&dR, nf * 3)) ||
        (rc = t->arena.take(&dCS, (size_t)nframes * (NCELLS + 1))) || (rc = t->arena.take(&dCI, nf)) ||
        (rc = cslam_frame_index_dev(t, dK, dN, nframes, kp_stride, face_w, face_h, dR, dCS, dCI))) return rc;
    if (rays) CSLAM_CUDA(cudaMemcpyAsync(rays, dR, nf * 12, cudaMemcpyDeviceToHost, t->stream));
    CSLAM_CUDA(cudaMemcpyAsync(cell_start, dCS, (size_t)nframes * (NCELLS + 1) * 2, cudaMemcpyDeviceToHost, t->stream));
    CSLAM_CUDA(cudaMemcpyAsync(cell_idx, dCI, nf * 2, cudaMemcpyDeviceToHost, t->stream));
    return cslam_tracker_sync(t);
}

static void fill_scales(TrackArgs& A, float scale_factor, int nlevels) {
    A.scale[0] = 1.0f;
    for (int i = 1; i < 16; i++) A.scale[i] = i < nlevels ? A.scale[i - 1] * scale_factor : A.scale[i - 1];
}

extern "C" int cslam_search_by_projection_last_dev(cslam_tracker* t, int npairs, const cslam_keypoint* k_cur, const uint8_t* d_cur, const int32_t* n_cur, int cur_stride,
                                                   const uint16_t* cell_start, const uint16_t* cell_idx, const uint8_t* cur_taken, const float* Tcw_cur,
                                                   const cslam_keypoint* k_last, const int32_t* n_last, int last_stride, const uint8_t* has_mp, const float* Xw, const uint8_t* d_mp,
                                                   const uint8_t* mp_obs, int face_w, int face_h, float cos_fov_th, float th, int check_ori, float scale_factor, int nlevels,
                                                   int32_t* match_cur, int32_t* nmatches) {
    if (!t || npairs <= 0 || cur_stride <= 0 || cur_stride > 4096 || last_stride <= 0 || face_w != face_h || nlevels < 1 || nlevels > 16) { set_error("cslam_search_by_projection_last: bad argument"); return CSLAM_E_BADARG; }
    CSLAM_CUDA(cudaSetDevice(t->device));
    TrackArgs A; std::memset(&A, 0, sizeof(A));
    A.kCur = k_cur; A.dCur = d_cur; A.nCur = n_cur; A.cellStart = cell_start; A.cellIdx = cell_idx; A.curTaken = cur_taken; A.curStride = cur_stride;
    A.nQ = n_last; A.qStride = last_stride; A.qValid = has_mp; A.qDesc = d_mp; A.qObs = mp_obs; A.qXw = Xw; A.kLast = k_last; A.TcwCur = Tcw_cur;
    A.mode = 0; A.W = face_w; A.H = face_h; A.checkOri = check_ori; A.th = th; A.nnratio = 0; A.cosFovTh = cos_fov_th; fill_scales(A, scale_factor, nlevels);
    A.match = match_cur; A.nmatches = nmatches; A.errFlag = t->errFlag;
    k_search_by_projection<<<npairs, TRK_WARPS * 32, 0, t->stream>>>(A); t->launches++;
    CSLAM_CUDA(cudaGetLastError());
    return CSLAM_OK;
}

extern "C" int cslam_search_by_projection_local_dev(cslam_tracker* t, int nframes, const cslam_keypoint* k_f, const uint8_t* d_f, const int32_t* n_f, int f_stride,
                                                    const uint16_t* cell_start, const uint16_t* cell_idx, const uint8_t* f_taken, const int32_t* n_mp, int mp_stride,
                                                    const uint8_t* in_view, const float* proj_xy, const int32_t* level, const float* view_cos, const uint8_t* d_mp,
                                                    const uint8_t* mp_obs, int face_w, int face_h, float th, float nnratio, float scale_factor, int nlevels, int32_t* match_f,
                                                    int32_t* nmatches) {
    if (!t || nframes <= 0 || f_stride <= 0 || f_stride > 4096 || mp_stride <= 0 || face_w != face_h || nlevels < 1 || nlevels > 16) { set_error("cslam_search_by_projection_local: bad argument"); return CSLAM_E_BADARG; }
    CSLAM_CUDA(cudaSetDevice(t->device));
    TrackArgs A; std::memset(&A, 0, sizeof(A));
    A.kCur = k_f; A.dCur = d_f; A.nCur = n_f; A.cellStart = cell_start; A.cellIdx = cell_idx; A.curTaken = f_taken; A.curStride = f_stride;
    A.nQ = n_mp; A.qStride = mp_stride; A.qValid = in_view; A.qDesc = d_mp; A.qObs = mp_obs; A.qProj = proj_xy; A.qLevel = level; A.qViewCos = view_cos;
    A.mode = 1; A.W = face_w; A.H = face_h; A.checkOri = 0; A.th = th; A.nnratio = nnratio; fill_scales(A, scale_factor, nlevels);
    A.match = match_f; A.nmatches = nmatches; A.errFlag = t->errFlag;
    k_search_by_projection<<<nframes, TRK_WARPS * 32, 0, t->stream>>>(A); t->launches++;
    CSLAM_CUDA(cudaGetLastError());
    return CSLAM_OK;
}

// host entry points (one pair / frame per call batch; staging inside): what the drop-in ORBMatcher::SearchByProjection definitions call. Every
// array is uploaded at its exact size: the kernels read no row past a frame's count.
extern "C" int cslam_search_by_projection_last(cslam_tracker* t, int npairs, const cslam_keypoint* k_cur, const uint8_t* d_cur, const int32_t* n_cur, int cur_stride,
                                               const uint8_t* cur_taken, const float* Tcw_cur, const cslam_keypoint* k_last, const int32_t* n_last, int last_stride,
                                               const uint8_t* has_mp, const float* Xw, const uint8_t* d_mp, const uint8_t* mp_obs, int face_w, int face_h, float cos_fov_th, float th,
                                               int check_ori, float scale_factor, int nlevels, int32_t* match_cur, int32_t* nmatches) {
    if (!t || npairs <= 0 || npairs > t->maxFrames || cur_stride > t->maxFeat || last_stride > t->maxFeat) { set_error("cslam_search_by_projection_last: sizes out of range"); return CSLAM_E_BADARG; }
    CSLAM_CUDA(cudaSetDevice(t->device));
    t->arena.reset();
    const size_t nc = (size_t)npairs * cur_stride, nl = (size_t)npairs * last_stride;
    DevArena& a = t->arena;
    const cslam_keypoint *kC, *kL; const uint8_t *dC, *taken, *valid, *dQ, *obs; const int32_t *nC, *nL; const float *Tcw, *dXw; uint16_t *cs, *ci; int32_t *match, *nm; int rc;
    if ((rc = a.upload(&kC, k_cur, nc)) || (rc = a.upload(&dC, d_cur, nc * 32)) || (rc = a.upload(&nC, n_cur, npairs)) || (rc = a.upload(&taken, cur_taken, nc)) ||
        (rc = a.upload(&Tcw, Tcw_cur, (size_t)npairs * 16)) || (rc = a.upload(&kL, k_last, nl)) || (rc = a.upload(&nL, n_last, npairs)) || (rc = a.upload(&valid, has_mp, nl)) ||
        (rc = a.upload(&dXw, Xw, nl * 3)) || (rc = a.upload(&dQ, d_mp, nl * 32)) || (rc = a.upload(&obs, mp_obs, nl)) || (rc = a.take(&cs, (size_t)npairs * (NCELLS + 1))) ||
        (rc = a.take(&ci, nc)) || (rc = a.take(&match, nc)) || (rc = a.take(&nm, npairs)) ||
        (rc = cslam_frame_index_dev(t, kC, nC, npairs, cur_stride, face_w, face_h, nullptr, cs, ci)) ||
        (rc = cslam_search_by_projection_last_dev(t, npairs, kC, dC, nC, cur_stride, cs, ci, taken, Tcw, kL, nL, last_stride, valid, dXw, dQ, obs, face_w, face_h, cos_fov_th, th,
                                                  check_ori, scale_factor, nlevels, match, nm))) return rc;
    CSLAM_CUDA(cudaMemcpyAsync(match_cur, match, nc * 4, cudaMemcpyDeviceToHost, t->stream)); CSLAM_CUDA(cudaMemcpyAsync(nmatches, nm, npairs * 4, cudaMemcpyDeviceToHost, t->stream));
    return cslam_tracker_sync(t);
}

extern "C" int cslam_search_by_projection_local(cslam_tracker* t, int nframes, const cslam_keypoint* k_f, const uint8_t* d_f, const int32_t* n_f, int f_stride, const uint8_t* f_taken,
                                                const int32_t* n_mp, int mp_stride, const uint8_t* in_view, const float* proj_xy, const int32_t* level, const float* view_cos,
                                                const uint8_t* d_mp, const uint8_t* mp_obs, int face_w, int face_h, float th, float nnratio, float scale_factor, int nlevels,
                                                int32_t* match_f, int32_t* nmatches) {
    if (!t || nframes <= 0 || nframes > t->maxFrames || f_stride > t->maxFeat || mp_stride > t->maxFeat) { set_error("cslam_search_by_projection_local: sizes out of range"); return CSLAM_E_BADARG; }
    CSLAM_CUDA(cudaSetDevice(t->device));
    t->arena.reset();
    const size_t nc = (size_t)nframes * f_stride, nm = (size_t)nframes * mp_stride;
    DevArena& a = t->arena;
    const cslam_keypoint* kF; const uint8_t *dF, *taken, *valid, *dQ, *obs; const int32_t *nF, *nQ, *lvl; const float *proj, *vcos; uint16_t *cs, *ci; int32_t *match, *nmOut; int rc;
    if ((rc = a.upload(&kF, k_f, nc)) || (rc = a.upload(&dF, d_f, nc * 32)) || (rc = a.upload(&nF, n_f, nframes)) || (rc = a.upload(&taken, f_taken, nc)) ||
        (rc = a.upload(&nQ, n_mp, nframes)) || (rc = a.upload(&valid, in_view, nm)) || (rc = a.upload(&proj, proj_xy, nm * 2)) || (rc = a.upload(&lvl, level, nm)) ||
        (rc = a.upload(&vcos, view_cos, nm)) || (rc = a.upload(&dQ, d_mp, nm * 32)) || (rc = a.upload(&obs, mp_obs, nm)) || (rc = a.take(&cs, (size_t)nframes * (NCELLS + 1))) ||
        (rc = a.take(&ci, nc)) || (rc = a.take(&match, nc)) || (rc = a.take(&nmOut, nframes)) ||
        (rc = cslam_frame_index_dev(t, kF, nF, nframes, f_stride, face_w, face_h, nullptr, cs, ci)) ||
        (rc = cslam_search_by_projection_local_dev(t, nframes, kF, dF, nF, f_stride, cs, ci, taken, nQ, mp_stride, valid, proj, lvl, vcos, dQ, obs, face_w, face_h, th, nnratio,
                                                   scale_factor, nlevels, match, nmOut))) return rc;
    CSLAM_CUDA(cudaMemcpyAsync(match_f, match, nc * 4, cudaMemcpyDeviceToHost, t->stream)); CSLAM_CUDA(cudaMemcpyAsync(nmatches, nmOut, nframes * 4, cudaMemcpyDeviceToHost, t->stream));
    return cslam_tracker_sync(t);
}

// Local maps of up to CSLAM_LOCAL_MAP_MAX_POINTS MapPoints per frame, whatever the handle's max_features (frames stay <= max_features): the
// arguments and outputs of cslam_search_by_projection_local, with -1 in every slot row past a frame's count. Every argument is checked before
// anything is enqueued; the per-call scratch (LM_K + 1/2 words per MapPoint row) comes from the handle's arena.
extern "C" int cslam_search_by_projection_local_large(cslam_tracker* t, int nframes, const cslam_keypoint* k_f, const uint8_t* d_f, const int32_t* n_f, int f_stride,
                                                      const uint8_t* f_taken, const int32_t* n_mp, int mp_stride, const uint8_t* in_view, const float* proj_xy,
                                                      const int32_t* level, const float* view_cos, const uint8_t* d_mp, const uint8_t* mp_obs, int face_w, int face_h,
                                                      float th, float nnratio, float scale_factor, int nlevels, int32_t* match_f, int32_t* nmatches) {
    static const char* fn = "cslam_search_by_projection_local_large";
    if (!t || nframes <= 0 || nframes > t->maxFrames || f_stride <= 0 || f_stride > t->maxFeat || mp_stride <= 0 || mp_stride > CSLAM_LOCAL_MAP_MAX_POINTS ||
        face_w <= 0 || face_w != face_h || nlevels < 1 || nlevels > 16 || !k_f || !d_f || !n_f || !f_taken || !n_mp || !in_view || !proj_xy || !level || !view_cos ||
        !d_mp || !mp_obs || !match_f || !nmatches) {
        set_error("%s: bad argument (frames in [1, %d], f_stride in [1, %d], mp_stride in [1, %d], nlevels in [1, 16], square faces)", fn, t ? t->maxFrames : 0,
                  t ? t->maxFeat : 0, CSLAM_LOCAL_MAP_MAX_POINTS);
        return CSLAM_E_BADARG;
    }
    for (int f = 0; f < nframes; f++)   // the window radius reads the scale of the predicted level
        for (int q = 0; q < std::min(n_mp[f], mp_stride); q++) {
            const size_t r = (size_t)f * mp_stride + q;
            if (in_view[r] && (level[r] < 0 || level[r] >= nlevels)) { set_error("%s: frame %d MapPoint %d: level %d outside [0, %d)", fn, f, q, level[r], nlevels); return CSLAM_E_BADARG; }
        }
    CSLAM_CUDA(cudaSetDevice(t->device));
    t->arena.reset();
    const size_t nc = (size_t)nframes * f_stride, nm = (size_t)nframes * mp_stride;
    DevArena& a = t->arena;
    const cslam_keypoint* kF; const uint8_t *dF, *taken, *valid, *dQ, *obs; const int32_t *nF, *nQ, *lvl; const float *proj, *vcos; uint16_t *cs, *ci, *lmCount;
    uint32_t* lmList; int32_t *match, *nmOut; int rc;
    if ((rc = a.upload(&kF, k_f, nc)) || (rc = a.upload(&dF, d_f, nc * 32)) || (rc = a.upload(&nF, n_f, nframes)) || (rc = a.upload(&taken, f_taken, nc)) ||
        (rc = a.upload(&nQ, n_mp, nframes)) || (rc = a.upload(&valid, in_view, nm)) || (rc = a.upload(&proj, proj_xy, nm * 2)) || (rc = a.upload(&lvl, level, nm)) ||
        (rc = a.upload(&vcos, view_cos, nm)) || (rc = a.upload(&dQ, d_mp, nm * 32)) || (rc = a.upload(&obs, mp_obs, nm)) || (rc = a.take(&cs, (size_t)nframes * (NCELLS + 1))) ||
        (rc = a.take(&ci, nc)) || (rc = a.take(&lmList, nm * LM_K)) || (rc = a.take(&lmCount, nm)) || (rc = a.take(&match, nc)) || (rc = a.take(&nmOut, nframes)) ||
        (rc = cslam_frame_index_dev(t, kF, nF, nframes, f_stride, face_w, face_h, nullptr, cs, ci))) return rc;
    TrackArgs A; std::memset(&A, 0, sizeof(A));
    A.kCur = kF; A.dCur = dF; A.nCur = nF; A.cellStart = cs; A.cellIdx = ci; A.curTaken = taken; A.curStride = f_stride;
    A.nQ = nQ; A.qStride = mp_stride; A.qValid = valid; A.qDesc = dQ; A.qObs = obs; A.qProj = proj; A.qLevel = lvl; A.qViewCos = vcos;
    A.mode = 1; A.W = face_w; A.H = face_h; A.th = th; A.nnratio = nnratio; fill_scales(A, scale_factor, nlevels);
    A.match = match; A.nmatches = nmOut; A.errFlag = t->errFlag; A.lmList = lmList; A.lmCount = lmCount;
    k_local_candidates<<<dim3(cdiv(mp_stride, TRK_WARPS), std::min(nframes, 65535)), TRK_WARPS * 32, 0, t->stream>>>(A, nframes); t->launches++;
    CSLAM_CUDA(cudaGetLastError());
    k_local_commit<<<nframes, TRK_WARPS * 32, 0, t->stream>>>(A); t->launches++;
    CSLAM_CUDA(cudaGetLastError());
    CSLAM_CUDA(cudaMemcpyAsync(match_f, match, nc * 4, cudaMemcpyDeviceToHost, t->stream)); CSLAM_CUDA(cudaMemcpyAsync(nmatches, nmOut, nframes * 4, cudaMemcpyDeviceToHost, t->stream));
    return cslam_tracker_sync(t);
}

// One pair of frames of up to CSLAM_BOW_FV_MAX_FEATURES key points each, whatever the handle's max_features. Every argument is checked before
// anything is enqueued. The candidate lists are sized to the call: the count pass's total is read back (one stream synchronisation) and exactly
// that much scratch is taken from the handle's arena.
extern "C" int cslam_search_for_initialization(cslam_tracker* t, const cslam_keypoint* k1, const uint8_t* d1, int n1, const float* prev_xy, const cslam_keypoint* k2,
                                               const uint8_t* d2, int n2, int face_w, int face_h, int window_size, float nnratio, int check_ori, int32_t* match12,
                                               int32_t* nmatches) {
    static const char* fn = "cslam_search_for_initialization";
    if (!t || n1 < 0 || n1 > CSLAM_BOW_FV_MAX_FEATURES || n2 < 0 || n2 > CSLAM_BOW_FV_MAX_FEATURES || !nmatches || (n1 > 0 && (!k1 || !d1 || !prev_xy || !match12)) ||
        (n2 > 0 && (!k2 || !d2)) || face_w <= 0 || face_w != face_h || window_size <= 0 || 2 * window_size > face_w) {
        set_error("%s: bad argument (n1, n2 in [0, %d], square faces, window_size in (0, face_w / 2], no NULL buffer)", fn, CSLAM_BOW_FV_MAX_FEATURES);
        return CSLAM_E_BADARG;
    }
    for (int i = 0; i < n1; i++)   // a negative level would make GetFeaturesInArea search every level
        if (k1[i].octave < 0) { set_error("%s: F1 key point %d has octave %d", fn, i, k1[i].octave); return CSLAM_E_BADARG; }
    for (int i = 0; i < n1; i++) match12[i] = -1;
    *nmatches = 0;
    if (n1 == 0 || n2 == 0) return CSLAM_OK;
    CSLAM_CUDA(cudaSetDevice(t->device));
    t->arena.reset();
    DevArena& a = t->arena;
    const cslam_keypoint *dK1, *dK2; const uint8_t *dD1, *dD2; const float* dPos; const int32_t* dN2; uint16_t *cs, *ci; uint32_t *off, *list; int32_t *match, *nm; int rc;
    if ((rc = a.upload(&dK1, k1, n1)) || (rc = a.upload(&dD1, d1, (size_t)n1 * 32)) || (rc = a.upload(&dPos, prev_xy, (size_t)n1 * 2)) || (rc = a.upload(&dK2, k2, n2)) ||
        (rc = a.upload(&dD2, d2, (size_t)n2 * 32)) || (rc = a.upload(&dN2, &n2, 1)) || (rc = a.take(&cs, NCELLS + 1)) || (rc = a.take(&ci, n2)) ||
        (rc = a.take(&off, (size_t)n1 + 1)) || (rc = a.take(&match, n1)) || (rc = a.take(&nm, 1)) ||
        (rc = frame_index(t->stream, t->launches, dK2, dN2, 1, n2, face_w, face_h, nullptr, cs, ci, CSLAM_BOW_FV_MAX_FEATURES))) return rc;
    const float r = (float)window_size;
    const int blocks = cdiv(n1, INIT_WARPS);
    k_init_candidates<<<blocks, INIT_WARPS * 32, 0, t->stream>>>(dK1, dD1, dPos, n1, dK2, dD2, cs, ci, face_w, face_h, r, off, nullptr, nullptr); t->launches++;
    CSLAM_CUDA(cudaGetLastError());
    k_init_scan<<<1, 1024, 0, t->stream>>>(off, n1); t->launches++;
    CSLAM_CUDA(cudaGetLastError());
    uint32_t totalEntries = 0;
    CSLAM_CUDA(cudaMemcpyAsync(&totalEntries, off + n1, 4, cudaMemcpyDeviceToHost, t->stream));
    CSLAM_CUDA(cudaStreamSynchronize(t->stream));
    if ((rc = a.take(&list, totalEntries))) return rc;
    k_init_candidates<<<blocks, INIT_WARPS * 32, 0, t->stream>>>(dK1, dD1, dPos, n1, dK2, dD2, cs, ci, face_w, face_h, r, nullptr, off, list); t->launches++;
    CSLAM_CUDA(cudaGetLastError());
    CSLAM_CUDA(cudaFuncSetAttribute(k_init_commit, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)INIT_SMEM));
    k_init_commit<<<1, INIT_WARPS * 32, INIT_SMEM, t->stream>>>(dK1, n1, dK2, n2, off, list, nnratio, check_ori, match, nm); t->launches++;
    CSLAM_CUDA(cudaGetLastError());
    CSLAM_CUDA(cudaMemcpyAsync(match12, match, (size_t)n1 * 4, cudaMemcpyDeviceToHost, t->stream)); CSLAM_CUDA(cudaMemcpyAsync(nmatches, nm, 4, cudaMemcpyDeviceToHost, t->stream));
    return cslam_tracker_sync(t);
}

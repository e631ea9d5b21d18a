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
};

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
            } else {
                u = A.qProj[((size_t)p * A.qStride + q) * 2]; v = A.qProj[((size_t)p * A.qStride + q) * 2 + 1];
                const int lvl = A.qLevel[(size_t)p * A.qStride + q];
                float r = A.qViewCos[(size_t)p * A.qStride + q] > 0.998 ? 2.5f : 4.0f;   // float compared with the double literal 0.998
                if (A.th != 1.0f) r = __fmul_rn(r, A.th);
                radius = __fmul_rn(r, A.scale[lvl]); minL = lvl - 1; maxL = lvl;
            }
            AreaQuery aq;
            if (ok && area_query(u, v, radius, A.W, A.H, inv, aq)) {
                const bool checkLevels = (minL > 0) || (maxL >= 0);
                const uint4 a0 = __ldg(dQ + 2 * q), a1 = __ldg(dQ + 2 * q + 1);
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
                        if (__any_sync(0xffffffffu, slow)) { if (lane == 0) *A.errFlag = CSLAM_E_CAPACITY; myKeep = min(myKeep, 16); }
                        int off = myKeep;
#pragma unroll
                        for (int o = 1; o < 32; o <<= 1) { const int t = __shfl_up_sync(0xffffffffu, off, o); if (lane >= o) off += t; }
                        const int tot = __shfl_sync(0xffffffffu, off, 31);
                        off -= myKeep;
                        for (int j = 0; j < myKeep; j++) {
                            const int pos = ncand + off + j;
                            if (pos < TRK_CAND) {
                                const int idx = keepIdx[j];
                                candIdx[warp][pos] = (uint16_t)idx;
                                candDist[warp][pos] = (uint16_t)hamming256(a0, a1, __ldg(dC + 2 * idx), __ldg(dC + 2 * idx + 1));
                            } else *A.errFlag = CSLAM_E_CAPACITY;
                        }
                        ncand = min(ncand + tot, TRK_CAND);
                    }
                }
            }
        }
        if (lane == 0) candN[warp] = ncand;
        __syncthreads();
        // ---- (B) commit in MapPoint order (one thread; the reference's scalar rules)
        if (tid == 0) {
            for (int w = 0; w < TRK_WARPS; w++) {
                const int qq = q0 + w, nc = candN[w];
                if (qq >= nQ || nc == 0) continue;
                int bestDist = 256, bestLevel = -1, bestDist2 = 256, bestLevel2 = -1, bestIdx = -1;
                for (int c = 0; c < nc; c++) {
                    const int idx = candIdx[w][c];
                    if (slotObs[idx]) continue;
                    const int dist = candDist[w][c];
                    if (dist < bestDist) { bestDist2 = bestDist; bestDist = dist; bestLevel2 = bestLevel; bestLevel = kC[idx].octave; bestIdx = idx; }
                    else if (A.mode == 1 && dist < bestDist2) { bestLevel2 = kC[idx].octave; bestDist2 = dist; }
                }
                if (bestDist > 100) continue;   // TH_HIGH
                if (A.mode == 1 && bestLevel == bestLevel2 && (float)bestDist > __fmul_rn(A.nnratio, (float)bestDist2)) continue;
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

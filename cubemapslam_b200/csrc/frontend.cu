// Front end of libcubemap_b200.so: fisheye->cubemap warp + ORB extraction, batched, sm_90a.
//
// Reference path (CPU, one frame at a time):
//   System::CvtFisheyeToCubeMap_reverseQuery_withInterpolation   src/System.cpp:327-355   (5 x cv::remap)
//   ORBextractor::operator()                                      src/ORBExtractor.cpp:838-926
//     ComputePyramid :928-953, ComputeKeyPointsOctTree :739-827 (cv::FAST per 30-px cell, DistributeOctTree
//     :511-737, IC_Angle :48-75), cull :883-904, GaussianBlur :907-908, computeOrbDescriptor :79-118
//
// Kernels (byte work; k_describe's blur runs on the integer tensor cores):
//   k_warp        canvas face tiles <- bilinear gather of the fisheye frame through a pre-quantised map
//   k_pyramid     level l <- cv::resize(INTER_LINEAR) fixed-point model of level l-1
//   k_fast        per 30-px cell FAST-9/16 arc score, in-cell NMS, 20->7 threshold fallback, candidate append
//   k_distribute  the reference's quadtree, restated as data-parallel rounds over nodes (see DESIGN.md)
//   k_describe    IC angle + 7x7 Gaussian of the 43x43 neighbourhood (IMMA) + steered BRIEF, one warp per keypoint
#include <algorithm>
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <vector>
#include "area_table.cuh"
#include "common.cuh"

namespace cslam {

static const int PATCH_SIZE = 31, HALF_PATCH = 15, EDGE_THRESHOLD = 19;
static const int MAX_LEVELS = 16;
static const int CG = 4;            // cells per CTA (x) in k_fast
static const int CELL_MAX = 48;     // largest supported cell edge
static const int FAST_TS = 224;     // smem tile stride (bytes): whole 16-byte columns of CG*CELL_MAX+6 columns from a 16-byte column
static const int DESC_WARPS = 4;

// IC_Angle's disc by column: bit v of word 15 + u is set iff |u| <= umax[v] (ORBextractor's umax), built by cslam_frontend_create
__device__ uint32_t g_icRows[32];
// the BRIEF pattern as k_describe reads it: test k of lane (= output byte) `lane` as floats (x0, y0, x1, y1) at [k * 32 + lane] (coalesced;
// a byte-per-test table read per lane was an 8-way shared-memory bank conflict). Filled by cslam_frontend_create from the same table.
__device__ float4 g_pat[8 * 32];

struct LevelGeom {
    int w, h, pitch;          // image size, row pitch in bytes
    int minB, maxBX, maxBY;   // FAST region (EDGE_THRESHOLD-3 inset)
    int wCell, hCell, nColsEff, nRowsEff;
    int quota;                // mnFeaturesPerLevel
    int candCap;
    int liveCap;              // longest k_fast live list of one tile (DevLevels::live; 0 without warp geometry)
    float scale;              // mvScaleFactor
    float sizeF;              // (int)(PATCH_SIZE*scale)
};

struct DevLevels {
    LevelGeom g[MAX_LEVELS];
    uint8_t* img[MAX_LEVELS];          // batch-major: frame f at img + f*pitch*h
    uint32_t* cand[MAX_LEVELS];        // batch x candCap packed (x | y<<12 | resp<<24), minBorder-relative
    uint16_t* pnode[MAX_LEVELS];       // batch x candCap scratch for k_distribute
    const uint16_t* xofs[MAX_LEVELS];  // resize tables for building level l from l-1
    const uint32_t* xab[MAX_LEVELS];   // a0 | a1<<16
    const uint4* prows[MAX_LEVELS];    // per k_pyramid row block: source window descriptor (build_pyr_rows)
    const uint8_t* skip[MAX_LEVELS];   // per k_fast CTA: 1 = tile provably corner-free when level 0 came from k_warp (no live work item)
    const uint8_t* pskip[MAX_LEVELS];  // per k_pyramid warp (PYR_WX x PYR_RY dst px): 1 = every pixel provably 0 (black corner tiles); levels >= 1
    const uint16_t* live[MAX_LEVELS];     // k_fast phase-A work items that can score above 0 on the warp path: y<<6 | (wi - w0), per CTA tile
    const uint32_t* liveOff[MAX_LEVELS];  // per CTA tile [liveOff[t], liveOff[t+1]) into live
    const struct FastCols* fcols[MAX_LEVELS];   // per k_fast tile column: lane masks, cells and division magics (build_fast_cols)
    int nlevels;
};

// ------------------------------------------------------------------------------------------------- k_warp
// Map entry: sx | sy<<16 with sx=cvRound(u*32), sy=cvRound(v*32) (cv::remap's INTER_BITS=5 fixed point).
// Weights are exact integers: (32-fy)(32-fx)*32 etc. (= cvRound of the fp32 table products * 32768).
// k_warp computes v = ((t00(32-fx) + t01 fx)(32-fy) + (t10(32-fx) + t11 fx) fy) * 32, rounded >> 15: the factored form is the
// same integer as the four-weight sum, and (32 X + 2^14) >> 15 == (X + 2^9) >> 10.
__device__ __forceinline__ uint32_t bilerp5(uint32_t t00, uint32_t t01, uint32_t t10, uint32_t t11, uint32_t fx, uint32_t fy) {
    const uint32_t h0 = t00 * (32 - fx) + t01 * fx, h1 = t10 * (32 - fx) + t11 * fx;
    return (h0 * (32 - fy) + h1 * fy + 512) >> 10;
}
// one pixel straight from global memory (tiles too large to stage); ix,iy >= 0 always (maps are >= 0); each tap outside the source reads 0 (BORDER_CONSTANT)
__device__ __forceinline__ uint32_t gather_direct(const uint8_t* __restrict__ S, int Iw, int Ih, uint32_t m) {
    const int sx = m & 0xffff, sy = m >> 16;
    const int ix = sx >> 5, iy = sy >> 5;
    const bool x0ok = ix < Iw, x1ok = ix + 1 < Iw, y0ok = iy < Ih, y1ok = iy + 1 < Ih;
    const uint8_t* p = S + (size_t)iy * Iw + ix;
    const uint32_t t00 = (y0ok && x0ok) ? __ldg(p) : 0u, t01 = (y0ok && x1ok) ? __ldg(p + 1) : 0u;
    const uint32_t t10 = (y1ok && x0ok) ? __ldg(p + Iw) : 0u, t11 = (y1ok && x1ok) ? __ldg(p + Iw + 1) : 0u;
    return bilerp5(t00, t01, t10, t11, sx & 31, sy & 31);
}

// Tiled warp. The map is fixed at create time, so each output tile's source footprint is known: a CTA stages the bounding box of
// its tile's taps for WARP_FPT frames into shared memory with coalesced 4-byte cp.async (zero-filled outside the source = BORDER_CONSTANT;
// byte loads when source rows are not word-aligned), then gathers the 4 taps of each pixel from there. All WARP_FPT boxes are loaded
// before one barrier; several resident CTAs per SM overlap one CTA's loads with another's arithmetic. Tiles are WT_W canvas
// columns (aligned to WT_W in canvas coordinates, so every thread stores its 4 pixels as one aligned u32) x WT_H face rows;
// columns outside the face are masked, so only the five face ROIs are written. Table entry of a staged pixel: box offset | fx<<16 | fy<<21, or WE_ORIGIN for a pixel whose map is (0,0) (outside
// the image circle: cv::remap reads S(0,0) with zero fractions). A tile whose box exceeds WARP_BOX_MAX is `direct`: its entries are
// the raw map and its pixels gather from global memory.
static const int WT_W = 32, WT_H = 32;
static const int WARP_FPT = 8;   // frames per CTA
static const int WARP_BOX_MAX = 6144;
static const uint32_t WE_ORIGIN = 1u << 26;
struct WarpTile {
    int row0, xa;      // canvas row of the tile's first face row; canvas column of its first (aligned) column
    int cx0, cx1, nr;  // face columns [cx0, cx1) in canvas coordinates; face rows in this tile
    int bx0, by0;      // source box origin (bx0 a multiple of 4)
    int bw, bh;        // source box width (bytes, a multiple of 4) and height
    int direct;
};

__device__ __forceinline__ void cp_async4_zfill(void* smem, const void* gmem, int srcBytes) {
    const uint32_t s = (uint32_t)__cvta_generic_to_shared(smem);
    asm volatile("cp.async.ca.shared.global [%0], [%1], 4, %2;\n" ::"r"(s), "l"(gmem), "r"(srcBytes) : "memory");
}
__device__ __forceinline__ void cp_async16(void* smem, const void* gmem) {   // both 16-byte aligned
    const uint32_t s = (uint32_t)__cvta_generic_to_shared(smem);
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;\n" ::"r"(s), "l"(gmem) : "memory");
}

__global__ void __launch_bounds__(256) k_warp(const uint8_t* __restrict__ fisheye, int Iw, int Ih, const WarpTile* __restrict__ tiles,
                                              const uint32_t* __restrict__ ent, uint8_t* __restrict__ canvas, int cpitch, size_t cframe, int batch,
                                              int slot, int words) {
    extern __shared__ __align__(16) uint8_t wsm[];   // WARP_FPT boxes of `slot` bytes, then S(0,0) of each frame
    uint8_t* origin = wsm + WARP_FPT * slot;
    const WarpTile T = tiles[blockIdx.x];
    const int f0 = blockIdx.y * WARP_FPT, nf = min(WARP_FPT, batch - f0), tid = threadIdx.x;
    const size_t fsz = (size_t)Iw * Ih;
    const uint8_t* S0 = fisheye + (size_t)f0 * fsz;
    if (!T.direct) {
        if (words) {   // Iw % 4 == 0 and a word-aligned frame pointer: a word is all inside or all outside the source row
            const int bw4 = T.bw >> 2, nwords = bw4 * T.bh;
            for (int i = tid; i < nwords; i += 256) {
                const int r = i / bw4, x = T.bx0 + 4 * (i - r * bw4), y = T.by0 + r;
                const bool ok = y < Ih && x < Iw;
                const uint8_t* src = S0 + (ok ? (size_t)y * Iw + x : 0);
                for (int k = 0; k < nf; k++) cp_async4_zfill(wsm + k * slot + 4 * i, src + k * fsz, ok ? 4 : 0);
            }
        } else {       // any other source width: byte loads, still coalesced along box rows
            const int nb = T.bw * T.bh;
            for (int i = tid; i < nb; i += 256) {
                const int r = i / T.bw, x = T.bx0 + (i - r * T.bw), y = T.by0 + r;
                const bool ok = y < Ih && x < Iw;
                const uint8_t* src = S0 + (ok ? (size_t)y * Iw + x : 0);
                for (int k = 0; k < nf; k++) wsm[k * slot + i] = ok ? __ldg(src + k * fsz) : (uint8_t)0;
            }
        }
        asm volatile("cp.async.commit_group;\n" ::: "memory");
        if (tid < nf) origin[tid] = __ldg(S0 + tid * fsz);
        asm volatile("cp.async.wait_group 0;\n" ::: "memory");
        __syncthreads();
    }
    const int r = tid >> 3, c = (tid & 7) * 4, x = T.xa + c;
    if (r >= T.nr) return;
    uint32_t lm = 0;
#pragma unroll
    for (int j = 0; j < 4; j++) lm |= (x + j >= T.cx0 && x + j < T.cx1) ? 1u << j : 0u;
    if (!lm) return;
    const uint4 e4 = __ldg(reinterpret_cast<const uint4*>(ent) + (size_t)blockIdx.x * (WT_W * WT_H / 4) + tid);
    const uint32_t e[4] = {e4.x, e4.y, e4.z, e4.w};
    uint8_t* D = canvas + (size_t)f0 * cframe + (size_t)(T.row0 + r) * cpitch + x;
    const int bw = T.bw;
#pragma unroll
    for (int k = 0; k < WARP_FPT; k++) {
        if (k >= nf) break;
        uint32_t out = 0;
        if (T.direct) {
#pragma unroll
            for (int j = 0; j < 4; j++) out |= gather_direct(S0 + k * fsz, Iw, Ih, e[j]) << (8 * j);
        } else {
            const uint8_t* B = wsm + k * slot;
#pragma unroll
            for (int j = 0; j < 4; j++) {
                uint32_t v;
                if (e[j] & WE_ORIGIN) v = origin[k];
                else {
                    const uint8_t* p = B + (e[j] & 0xffff);
                    v = bilerp5(p[0], p[1], p[bw], p[bw + 1], (e[j] >> 16) & 31, (e[j] >> 21) & 31);
                }
                out |= v << (8 * j);
            }
        }
        uint8_t* d = D + k * cframe;
        if (lm == 0xfu) *reinterpret_cast<uint32_t*>(d) = out;
        else {
#pragma unroll
            for (int j = 0; j < 4; j++) if (lm & (1u << j)) d[j] = (uint8_t)(out >> (8 * j));
        }
    }
}

// ------------------------------------------------------------------------------------------------- k_pyramid
// cv::resize(src,dst,sz,0,0,INTER_LINEAR) 8U model: 11-bit coefficients, horizontal int pass H = S[s]*a0 + S[s+1]*a1,
// vertical (((b0*(H0>>4))>>16)+((b1*(H1>>4))>>16)+2)>>2.  One thread = 4 consecutive dst pixels x PYR_RY dst rows:
// the 8-byte source window of the 4 pixels is fetched with aligned 32-bit loads, the taps are gathered with PRMT and the
// horizontal pass is two-tap IDP.2A (coefficient pair a0|a1<<16 straight from the table).
// The source rows of a CTA's PYR_RY dst rows are one contiguous window (the scale factor is > 1, so consecutive dst rows have
// distinct top taps and every window row is the top tap of at most one dst row). Its descriptor (build_pyr_rows) is read once,
// every window row is loaded before the first arithmetic, and each window row's H is computed once; dst row k is emitted at the
// window row of its bottom tap. WIN bounds the window (PYR_WIN at scale factors up to about 1.4, PYR_WIN_MAX up to 2.0).
// `skip` (warp path only): one byte per warp-sized piece (128 dst px x PYR_RY rows), 1 = every pixel of the piece is provably 0
// (the black cubemap corners, DevLevels::pskip). The buffer already holds those zeros, so the warp exits without reading or writing.
static const int PYR_RY = 8;
static const int PYR_WX = 32 * 4;   // dst columns per warp
static const int PYR_WIN = 12, PYR_WIN_MAX = 20;   // window rows (and descriptor words) of the two k_pyramid instantiations
template <int WIN>
__global__ void __launch_bounds__(128) k_pyramid(const uint8_t* __restrict__ src, int sw, int sh, int spitch, uint8_t* __restrict__ dst, int dw, int dh,
                                                 int dpitch, const uint16_t* __restrict__ xofs, const uint32_t* __restrict__ xab,
                                                 const uint4* __restrict__ rows, const uint8_t* __restrict__ skip) {
    static_assert(WIN % 4 == 0 && WIN < 32, "descriptor = WIN / 4 uint4; nwin fits the top half of word 0");
    const int x4 = (blockIdx.x * blockDim.x + threadIdx.x) * 4;
    if (x4 >= dw) return;
    if (skip && skip[blockIdx.y * ((dw + PYR_WX - 1) / PYR_WX) + x4 / PYR_WX]) return;   // warp-uniform
    // row-block descriptor: word 0 = first source row | window rows << 16; word j >= 1 = b0 | b1 << 16 of the dst row whose bottom tap
    // is window row j, 0 for none (a real pair sums to 2048)
    uint32_t rd[WIN];
#pragma unroll
    for (int q = 0; q < WIN / 4; q++) {
        const uint4 v = __ldg(rows + (size_t)blockIdx.y * (WIN / 4) + q);
        rd[4 * q] = v.x; rd[4 * q + 1] = v.y; rd[4 * q + 2] = v.z; rd[4 * q + 3] = v.w;
    }
    const int src0 = rd[0] & 0xffff, nwin = rd[0] >> 16;
    const uint8_t* S = src + (size_t)blockIdx.z * spitch * sh;
    uint8_t* D = dst + ((size_t)blockIdx.z * dh + (size_t)blockIdx.y * PYR_RY) * dpitch + x4;
    int s0[4]; uint32_t ab[4];
#pragma unroll
    for (int k = 0; k < 4; k++) { const int x = min(x4 + k, dw - 1); s0[k] = xofs[x]; ab[k] = xab[x]; }
    const int base = s0[0], al = base & ~3, sh8 = (base & 3) * 8;
    // byte selectors into the 8-byte window starting at `base`: pair (left,right) per pixel; right = left when clamped at the last column
    uint32_t sel01 = 0, sel23 = 0;
#pragma unroll
    for (int k = 0; k < 4; k++) {
        const uint32_t dl = (uint32_t)(s0[k] - base), dr = (s0[k] + 1 <= sw - 1) ? dl + 1 : dl;
        const uint32_t pr = dl | (dr << 4);
        if (k < 2) sel01 |= pr << (8 * k); else sel23 |= pr << (8 * (k - 2));
    }
    // window row j is source row min(src0 + j, sh - 1): the clamp is cv::resize's bottom tap min(a + 1, sh - 1), and it keeps the rows past
    // nwin (loaded unconditionally, never used) inside the level. Words past the row's pitch are never selected; the last row's run into
    // the buffer's slack
    const uint8_t* R0 = S + (size_t)src0 * spitch + al;
    const uint32_t last = (uint32_t)(sh - 1 - src0);
    uint32_t w[WIN][3];
#pragma unroll
    for (int j = 0; j < WIN; j++) {
        const uint32_t* R = reinterpret_cast<const uint32_t*>(R0 + (size_t)min((uint32_t)j, last) * (uint32_t)spitch);
        w[j][0] = __ldg(R); w[j][1] = __ldg(R + 1); w[j][2] = __ldg(R + 2);
    }
    uint32_t Hp[4];
#pragma unroll
    for (int j = 0; j < WIN; j++) {
        if (j >= nwin) break;   // CTA-uniform
        const uint32_t lo = __funnelshift_r(w[j][0], w[j][1], sh8), hi = __funnelshift_r(w[j][1], w[j][2], sh8);
        const uint32_t p01 = __byte_perm(lo, hi, sel01), p23 = __byte_perm(lo, hi, sel23);
        uint32_t H[4];
        H[0] = __dp2a_lo(ab[0], p01, 0u) >> 4; H[1] = __dp2a_hi(ab[1], p01, 0u) >> 4;
        H[2] = __dp2a_lo(ab[2], p23, 0u) >> 4; H[3] = __dp2a_hi(ab[3], p23, 0u) >> 4;
        if (j > 0 && rd[j]) {   // CTA-uniform
            // (b * H) >> 16 == umulhi(b << 16, H). The sums are < 1024 (bytes <= 255 after >> 2, no clamp needed), so two of them
            // share a word and one shift; PRMT picks bytes 0 and 2 of each pair
            const uint32_t B0 = rd[j] << 16, B1 = rd[j] & 0xffff0000u;
            uint32_t s[4];
#pragma unroll
            for (int k = 0; k < 4; k++) s[k] = __umulhi(B0, Hp[k]) + __umulhi(B1, H[k]) + 2;
            const uint32_t s01 = s[0] | (s[1] << 16), s23 = s[2] | (s[3] << 16);
            *reinterpret_cast<uint32_t*>(D) = __byte_perm(s01 >> 2, s23 >> 2, 0x6420);   // pitch is a multiple of 128: padding absorbs the tail
            D += dpitch;
        }
#pragma unroll
        for (int k = 0; k < 4; k++) Hp[k] = H[k];
    }
}

// ------------------------------------------------------------------------------------------------- k_fast
// Arc score s(p) = max over the 16 arcs of 9 contiguous ring pixels of max(min(d), min(-d)), d = p - ring.
// corner(thr) <=> s > thr; OpenCV response = s-1. The reference runs cv::FAST per cell ROI [ini, ini+cell+6):
// detection areas of neighbouring cells tile the level without overlap, NMS only sees scores of the same cell,
// and the 20->7 fallback is decided per cell on "no keypoint survived NMS" (src/ORBExtractor.cpp:763-803).
// Exact arc score of 2 pixels at once in u16x2 lanes (sm_90a VIMNMX3.U16x2):
//   s = max(0, A - c, c - B),  A = max_k min(R[k..k+8]),  B = min_k max(R[k..k+8])   (R = ring intensities, c = centre)
// A and B take 32 min/max each, windows paired as described in the function. No data-dependent branch, no per-pixel early-out:
// on textured input almost every pixel passes the cheap antipodal tests, so the branch-free full score is cheaper
// than queueing.
// The intensities sit in the high bytes of the lanes, the low bytes hold anything (the neighbouring pixels of a raw image word): u16
// min/max orders by the high byte first, so the high byte of every min/max is the min/max of the high bytes. Only A, B and c are
// masked, before the subtractions. Returned per lane: (max(s, t) - t) << 8 for the threshold t, given as T = t << 8 in each lane, i.e.
// 0 where s <= t and order-preserving above it.
__device__ __forceinline__ uint32_t arc_score_x2(const uint32_t (&R)[16], uint32_t c, uint32_t T) {
    // Windows k and k+1 (k even) share ring pixels k+1..k+8. By distributivity max(min(R[k], s), min(s, R[k+9])) = min(s, max(R[k], R[k+9])),
    // so the pair's larger minimum is min(R[k+1..k+8], max(R[k], R[k+9])). For k = 4g and k = 4g + 2 the shared runs are P[k+1] + S[g] and
    // S[g] + P[k+9], with P[j] = min(R[j], R[j+1]) (j odd) and S[g] = R[4g+3..4g+8] = min3 of three P: 8 + 4 + 16 + 4 = 32 min/max per side
    // instead of 40 (B: the same with min and max swapped)
    uint32_t pn[8], px[8];   // P at index (j - 1) / 2
#pragma unroll
    for (int i = 0; i < 8; i++) {
        const int j = 2 * i + 1;
        pn[i] = __vminu2(R[j], R[(j + 1) & 15]);
        px[i] = __vmaxu2(R[j], R[(j + 1) & 15]);
    }
    uint32_t tA[8], tB[8];
#pragma unroll
    for (int g = 0; g < 4; g++) {
        const int k = 4 * g;
        const uint32_t sn = __vimin3_u16x2(pn[2 * g + 1], pn[(2 * g + 2) & 7], pn[(2 * g + 3) & 7]);
        const uint32_t sx = __vimax3_u16x2(px[2 * g + 1], px[(2 * g + 2) & 7], px[(2 * g + 3) & 7]);
        tA[2 * g] = __vimin3_u16x2(sn, pn[2 * g], __vmaxu2(R[k], R[(k + 9) & 15]));
        tB[2 * g] = __vimax3_u16x2(sx, px[2 * g], __vminu2(R[k], R[(k + 9) & 15]));
        tA[2 * g + 1] = __vimin3_u16x2(sn, pn[(2 * g + 4) & 7], __vmaxu2(R[k + 2], R[(k + 11) & 15]));
        tB[2 * g + 1] = __vimax3_u16x2(sx, px[(2 * g + 4) & 7], __vminu2(R[k + 2], R[(k + 11) & 15]));
    }
    uint32_t A = __vimax3_u16x2(__vimax3_u16x2(tA[0], tA[1], tA[2]), __vimax3_u16x2(tA[3], tA[4], tA[5]), __vmaxu2(tA[6], tA[7]));
    uint32_t Bm = __vimin3_u16x2(__vimin3_u16x2(tB[0], tB[1], tB[2]), __vimin3_u16x2(tB[3], tB[4], tB[5]), __vminu2(tB[6], tB[7]));
    const uint32_t HI = 0xff00ff00u;
    A &= HI; Bm &= HI; c &= HI;
    const uint32_t t1 = __vmaxu2(A, c) - c;      // lanes never borrow: max(A,c) >= c
    const uint32_t t2 = c - __vminu2(Bm, c);
    return __vimax3_u16x2(t1, t2, T) - T;
}

// Compass bound of the arc score of 2 pixels in u16x2 lanes, from ring pixels 0, 4, 8, 12 alone (same lane encoding as arc_score_x2).
// 9 contiguous ring pixels always hold two neighbouring compass points 4j and 4j+4, so A <= max_j min(R[4j], R[4j+4]), which by
// distributivity is min(max(R0, R8), max(R4, R12)); dually B >= max(min(R0, R8), min(R4, R12)). Only the centre is masked: with cl = c
// with low bytes 0 and ch = c with low bytes 0xff, max(A, cl) - cl and ch - min(B, ch) are d << 8 | (0..255) for the bright and dark
// margins d = max(A - c, 0), max(c - B, 0) of the high bytes, whatever the low bytes hold. Returned per lane: max(those, acc); with
// acc = T1 = t << 8 | 0xff (or a previous result) that is T1 exactly where neither margin exceeds t: where the arc score is provably <= t.
__device__ __forceinline__ uint32_t compass_x2(uint32_t r0, uint32_t r4, uint32_t r8, uint32_t r12, uint32_t c, uint32_t acc) {
    const uint32_t A = __vminu2(__vmaxu2(r0, r8), __vmaxu2(r4, r12));
    const uint32_t Bm = __vmaxu2(__vminu2(r0, r8), __vminu2(r4, r12));
    const uint32_t cl = c & 0xff00ff00u, ch = c | 0x00ff00ffu;
    return __vimax3_u16x2(__vmaxu2(A, cl) - cl, ch - __vminu2(Bm, ch), acc);   // lanes never borrow
}

// q = i / d for 0 <= i < 65536/..: d-uniform fast division (tile loops have i < 8192, d <= 64)
__device__ __forceinline__ int fdiv_small(int i, uint32_t magic) { return (int)(((uint32_t)i * magic) >> 20); }
__host__ __device__ inline uint32_t fdiv_magic(int d) { return ((1u << 20) + d - 1) / d; }

// Layout of one CTA: one tile column (CG cells wide) of FAST_R consecutive cell rows of one frame, walked tile by tile (a tile = CG cells of
// one cell row, exactly the reference's per-cell ROIs). Phases of each tile:
// The thresholds are mt = minTh and ti = max(iniTh, mt), each clamped to 1..255 (see below). A keypoint of cv::FAST at ti is exactly an NMS
// survivor at mt with s > ti: a suppressor needs s_n >= s, and a neighbour with s_n <= ti < s suppresses nothing at either threshold.
//  A0 compass pretest of every work item (4 pixels), at both thresholds from one bound (compass_x2): an item the bound cannot prove <= ti goes
//     to the tile's pass list, one it proves <= ti but not <= mt to the deferred list (one shared atomic per warp each). On the warp path
//     (`live` given) only the tile's live work items are tested: every other item's 7x7 windows hold one constant (DevLevels::live), so its
//     scores are 0
//  A  branch-free exact arc score of every pass-list item -> S (u16, (s - mt) << 8, 0 where s <= mt). An item left out scores 0, which the
//     zeroed S already holds. Each warp appends the items it scored non-zero to the tile's nzHi list (some score > ti) or nzLo list
//  B  round 1: 3x3 NMS at mt inside each cell, one work item (2 pair-words) per thread, over nzHi, keeping the survivors with s > ti: the
//     keypoints at ti, exactly (the deferred items, still 0 in S, are <= ti). A cell none of them lies in falls back to mt (the reference's
//     20->7 rule); if the tile has such cells (F), round 2 scores the deferred items with a pixel in F into S and, after a barrier, runs
//     the NMS at mt over every non-zero item with a pixel in F, keeping every survivor in F. S already holds the pass-list items' scores
//     at mt, so nothing is scored twice, and a cell whose pixels above ti all lose to equal neighbours (a plateau) falls back as it must
//  C  every NMS survivor appended to the strip's output buffer, one shared atomic per warp; the buffer is copied to the global candidate
//     list (one global atomic) at the end of the strip, or at the end of a tile after which it could not hold another tile's survivors
static const int FAST_R = 8;            // cell rows per k_fast CTA
static const int FAST_SW = FAST_TS / 2;   // pair-words per score row
static const int FAST_OUT = CG * ((CELL_MAX + 1) / 2) * ((CELL_MAX + 1) / 2);   // candidates the strip's output buffer holds: >= any kmax
static_assert(16 * ((15 + CG * CELL_MAX + 6 + 15) / 16) <= FAST_TS && FAST_TS / 16 <= 16,
              "a tile row is at most FAST_TS / 16 <= 16 columns of 16 bytes (k_fast stages a row with 16 lanes)");
static_assert((15 + CG * CELL_MAX + 6) / 4 < 64 && CELL_MAX < 1024, "a live work item packs y<<6 | (wi - w0) into 16 bits");
static_assert(CG <= 4, "FastItem packs a pixel's cell index into 2 bits");

// Column geometry of the k_fast CTA tile in tile column cx (blockIdx.x) of a level. The tile's rows start at a0 = tx0 & ~15 (16-byte
// loads); work item wi covers tile columns 4*wi..4*wi+3, and detection x = tile column - xoff.
struct FastTileX {
    int tx0, a0, nvec;     // first ROI column, first loaded column, loaded 16-byte columns per row
    int nx, xoff;          // detection width, tile column of detection x = 0
    int w0, w1;            // work items [w0, w1) cover the detection columns
    int q0, q1;            // uint4 columns [q0, q1) of an S2 row cover the pair-words phase B reads, [2*w0 - 1, 2*w1 + 1)
};
__host__ __device__ inline FastTileX fast_tile_x(const LevelGeom& g, int cx) {
    FastTileX t;
    const int j0 = cx * CG, ncell = min(CG, g.nColsEff - j0);
    t.tx0 = g.minB + j0 * g.wCell;
    const int tx1 = min(t.tx0 + ncell * g.wCell + 6, g.maxBX);
    t.a0 = t.tx0 & ~15; t.nvec = (tx1 - t.a0 + 15) >> 4;   // tx1 + 15 <= maxBX + 15 < w: the last column stays inside the row
    t.nx = tx1 - t.tx0 - 6; t.xoff = t.tx0 - t.a0 + 3;
    t.w0 = t.xoff >> 2; t.w1 = (t.xoff + t.nx + 3) >> 2;
    t.q0 = max(2 * t.w0 - 1, 0) >> 2; t.q1 = (t.w1 + 2) >> 1;
    return t;
}
// Per work item wi of a tile column: lane masks of pair-words 2*wi and 2*wi+1 (a lane is 0xffff or 0) and the cell of each pixel
struct FastItem {
    uint32_t valid[2];    // column inside the detection area
    uint32_t cells;       // cell index within the tile of pixel j (tile column 4*wi + j) in bits 2j..2j+1
    uint32_t cellMask;    // bit c: some pixel of the item inside the detection area lies in cell c
    uint32_t left[2], right[2];   // has a left / right neighbour in its cell
};
// Everything k_fast needs that depends on the tile column alone; built once per level at create time (build_fast_cols)
struct FastCols {
    uint32_t mgItems, mgZero, pad[2];   // fdiv_magic of w1 - w0 and q1 - q0
    FastItem item[FAST_SW / 2];
};

// Dynamic shared memory of a k_fast CTA (byte offsets), sized from the level's cell geometry; CELL_MAX bounds it (fast_smem_max)
struct FastSmem {
    int items;                 // the tile column's FastCols::item table
    int pass;                  // listCap u16 entries, encoded as the live list: from the front the current tile's pass list (items the compass
                               // bound cannot prove <= ti: phase A's work list), from the back its deferred list (provably <= ti, not <= mt:
                               // scored in round 2 only). An item enters at most one of them. Its own region, like the nz list
    int nz;                    // listCap u16 entries: from the front nzHi (items scored with a score > ti: round 1's work list), from the back
                               // nzLo (scored non-zero, no score > ti; round 2 appends the deferred items it scores non-zero). Its own
                               // region: warps append ahead of other warps' pass-list reads, and the other buffers hold the next tile
    int listCap;               // entries of each list region: >= the items of a tile that phase A0 tests
    int tile, tileBytes;     // tile buffer b at tile + b * tileBytes: 16 bytes in front (phase A reads the word left of row 0 unguarded),
                               // then hCell + 6 rows of FAST_TS
    int s2, klist;             // score map (hCell + 2 rows of FAST_SW pair-words); NMS survivors, kmax entries
    int live, liveBytes;       // live list buffer b (u16, staged in 16-byte pieces from an index that is a multiple of 8) at live + b * liveBytes
    int kmax, total;
};
__host__ __device__ inline FastSmem fast_smem(const LevelGeom& g) {
    FastSmem m;
    m.tileBytes = 16 + (g.hCell + 6) * FAST_TS; m.liveBytes = 16 * ((g.liveCap + 14) / 8);
    m.kmax = CG * ((g.wCell + 1) / 2) * ((g.hCell + 1) / 2);   // NMS survivors of a cell are pairwise non-adjacent
    // items of a tile: nw <= (nx + 6) / 4 (fast_tile_x, nx <= CG * wCell) per detection row, hCell rows at most
    m.listCap = 8 * ((max(g.liveCap, ((CG * g.wCell + 6) >> 2) * g.hCell) + 7) / 8);
    m.items = 0;
    m.nz = m.items + (int)sizeof(FastItem) * (FAST_SW / 2);   // a constant offset: no register holds its address
    m.pass = m.nz + 2 * m.listCap;
    m.tile = m.pass + 2 * m.listCap;
    m.s2 = m.tile + 2 * m.tileBytes;
    m.live = m.s2 + (g.hCell + 2) * FAST_SW * 4;
    m.klist = m.live + 2 * m.liveBytes;
    m.total = m.klist + 4 * m.kmax;
    return m;
}
static_assert(FAST_TS % 16 == 0 && sizeof(FastItem) % 16 == 0, "k_fast shared-memory regions stay 16-byte aligned");

// Neighbourhood maximum of pair-word `cur` over its 8 same-cell neighbours: a*, b*, c* = the pair-words left of, at and right of it in the
// row above (0), its own row (1) and the row below (2); ml / mr mask the lanes without a left / right neighbour in their cell. fl: a
// floor in both lanes (free in the last max), so that a lane survives only if it is above the floor too
__device__ __forceinline__ uint32_t nms_max(uint32_t a0, uint32_t b0, uint32_t c0, uint32_t a1, uint32_t cur, uint32_t c1, uint32_t a2, uint32_t b2,
                                            uint32_t c2, uint32_t ml, uint32_t mr, uint32_t fl) {
    const uint32_t upL = __funnelshift_r(a0, b0, 16) & ml, upR = __funnelshift_r(b0, c0, 16) & mr;
    const uint32_t cuL = __funnelshift_r(a1, cur, 16) & ml, cuR = __funnelshift_r(cur, c1, 16) & mr;
    const uint32_t dnL = __funnelshift_r(a2, b2, 16) & ml, dnR = __funnelshift_r(b2, c2, 16) & mr;
    return __vimax3_u16x2(__vimax3_u16x2(upL, b0, upR), __vimax3_u16x2(cuL, cuR, b2), __vimax3_u16x2(dnL, dnR, fl));
}

__global__ void __launch_bounds__(256, 4) k_fast(const uint8_t* __restrict__ img, LevelGeom g, int iniTh, int minTh, uint32_t* __restrict__ cand,
                                              uint32_t* __restrict__ candCount, int countStride, int* __restrict__ errFlag,
                                              const FastCols* __restrict__ cols, const uint8_t* __restrict__ skip,
                                              const uint16_t* __restrict__ live, const uint32_t* __restrict__ liveOff) {
    extern __shared__ __align__(16) uint8_t fsm[];   // FastSmem
    const FastSmem SM = fast_smem(g);
    // score map, one u16 per pixel as u16x2 pair-words: word 2*wi (+1) of row y+1 holds tile columns 4*wi..4*wi+1 (+2..+3)
    uint32_t* const S2 = reinterpret_cast<uint32_t*>(fsm + SM.s2);
    uint32_t* const klist = reinterpret_cast<uint32_t*>(fsm + SM.klist);   // x | y<<8 | s<<16
    const uint4* const items = reinterpret_cast<const uint4*>(fsm + SM.items);   // FastItem wi = items[2*wi], items[2*wi+1]
    uint16_t* const passS = reinterpret_cast<uint16_t*>(fsm + SM.pass);   // pass list from the front, deferred list from the back
    uint16_t* const nzS = reinterpret_cast<uint16_t*>(fsm + SM.nz);       // nzHi from the front, nzLo from the back
    __shared__ uint32_t rowLo[FAST_R], rowHi[FAST_R];   // live list of each strip row, [rowLo, rowHi)
    __shared__ int rowVisit[FAST_R];                    // the strip row's tile has work (not skipped, detection rows > 0)
    __shared__ uint32_t sout[FAST_OUT];   // the strip's selected candidates, packed as in cand
    __shared__ uint32_t hit;              // bit c: cell c of the tile has a keypoint at ti (round 1)
    __shared__ int nK, nPass, nDef, nHi, nLo, nOut, flushN;
    __shared__ uint32_t flushBase;
    const int frame = blockIdx.z, row0 = blockIdx.y * FAST_R, nr = min(FAST_R, g.nRowsEff - row0);
    const int tid = threadIdx.x, lane = tid & 31;
    // the tile column's geometry and division magics, read from shared memory after each barrier rather than held in registers across phase A
    __shared__ FastTileX X;
    __shared__ uint2 mg;   // FastCols::mgItems, mgZero
    const FastCols* C = cols + blockIdx.x;
    {
        const FastTileX t = fast_tile_x(g, blockIdx.x);
        if (t.nx <= 0) return;   // block-uniform: a ROI with fewer than 7 columns has no detection area (cv::FAST returns nothing)
        if (tid == 0) { X = t; mg = __ldg(reinterpret_cast<const uint2*>(C)); }
    }
    const uint8_t* I = img + (size_t)frame * g.pitch * g.h;
    for (int i = tid; i < nr; i += 256) {
        const int t = (row0 + i) * gridDim.x + blockIdx.x, iniY = g.minB + (row0 + i) * g.hCell;
        // a ROI with fewer than 7 rows has no detection area; a skipped tile is provably corner-free (no live work item)
        rowVisit[i] = min(iniY + g.hCell + 6, g.maxBY) - iniY > 6 && !(skip && skip[t]);
        if (live) { rowLo[i] = liveOff[t]; rowHi[i] = liveOff[t + 1]; }
    }
    if (tid == 0) nOut = 0;
    __syncthreads();
    int cur = 0;
    while (cur < nr && !rowVisit[cur]) cur++;
    if (cur == nr) return;
    // cv::FAST clamps its threshold to 0..255 and ranks corners by s - 1, with 0 for "no corner": at threshold 0 a corner with s = 1 ties
    // with its non-corner neighbours and never survives NMS, exactly as if the threshold were 1. An iniTh at or below minTh gives ti = mt:
    // every survivor at mt is then a keypoint at iniTh, as the fallback rule has it
    const int mt = min(max(minTh, 1), 255), ti = max(min(max(iniTh, 1), 255), mt);
    const uint32_t T = (uint32_t)mt * 0x01000100u;
    // ti in S's encoding, both lanes: a score is > ti iff its lane is > TH. Read from shared memory where it is used (after B1), which
    // keeps it out of the registers of phases A and B
    __shared__ uint32_t TH;
    if (tid == 0) TH = (uint32_t)(ti - mt) * 0x01000100u;
    // strip row i's tile rows and live list (from the multiple of 8 at or below rowLo) into buffer b, by 16-byte copies: a0 and the level
    // pitch are multiples of 16. Thread tid copies 16-byte column tid % 16 of tile rows tid / 16, tid / 16 + 16, ... (a row has at most 16)
    auto stage = [&](int i, int b) {
        const int iniY = g.minB + (row0 + i) * g.hCell, nrows = min(iniY + g.hCell + 6, g.maxBY) - iniY, vc = tid & 15;
        const uint8_t* base = I + (size_t)iniY * g.pitch + X.a0 + 16 * vc;
        uint8_t* tile = fsm + SM.tile + b * SM.tileBytes + 16 + 16 * vc;
        if (vc < X.nvec)
#pragma unroll 1
            for (int r = tid >> 4; r < nrows; r += 16) cp_async16(tile + r * FAST_TS, base + (size_t)r * g.pitch);
        if (live) {
            const uint32_t lo = rowLo[i] & ~7u, n = (rowHi[i] - lo + 7) >> 3;   // the list is padded to a multiple of 8 entries
            const uint4* src = reinterpret_cast<const uint4*>(live + lo);
            for (uint32_t k = tid; k < n; k += 256) cp_async16(fsm + SM.live + b * SM.liveBytes + 16 * k, src + k);
        }
        asm volatile("cp.async.commit_group;\n" ::: "memory");
    };
    for (int k = tid; k < (int)(sizeof(FastItem) / 16) * (FAST_SW / 2); k += 256) cp_async16(fsm + SM.items + 16 * k, reinterpret_cast<const uint4*>(C->item) + k);
    stage(cur, 0);   // same group as the item table
    // the strip's output buffer to the frame's candidate list. Called after a barrier that follows every append to it (block-uniform); the
    // next appends come after at least one more barrier, which also publishes nOut = 0. The count grows past candCap like the list would.
    auto flush = [&]() {
        if (tid == 0) { const int n = nOut; flushN = n; flushBase = atomicAdd(candCount + (size_t)frame * countStride, (uint32_t)n); }
        __syncthreads();
        if (tid == 0) nOut = 0;
        const int n = flushN;
        uint32_t* out = cand + (size_t)frame * g.candCap;
        for (int i = tid; i < n; i += 256) {
            const uint32_t pos = flushBase + i;
            if (pos < (uint32_t)g.candCap) out[pos] = sout[i];
            else *errFlag = CSLAM_E_CAPACITY;
        }
    };
    // Barriers of one tile (buffer b = tile parity in the strip):
    //  top   S2 cleared, nK / nPass / nDef / nHi / nLo / hit reset: the previous tile's phases A, B and C are done with them (its end
    //        barrier), or it ended at BP with empty pass and deferred lists and read nothing else after B1
    //  wait  this thread's copies of the tile landed; B1 (__syncthreads_or) makes every thread's copies visible
    //  after B1: the next visited tile is staged into buffer b^1, which the previous tile last read in phase A or round 2, before its end
    //  barrier
    //  A0 (reads the live list of b; appends to the pass and deferred lists, nPass, nDef) -> BP -> A (pass list, nPass; appends to nzHi
    //  and nzLo, nHi, nLo) -> B2 -> round 1 (S2, item table, nzHi, nHi; appends to klist, nK, hit) -> B3 -> only if the tile has a cell
    //  in F (hit, block-uniform): round 2 scoring (deferred list, nDef; S2, appends to nzLo, nLo) -> B4 -> round 2 NMS (S2, nzHi, nzLo;
    //  appends to klist, nK) -> B5 -> C (klist, nK; appends to the output buffer) -> end barrier
    //  a tile whose pass and deferred lists are empty has no corner: after BP it goes on to the next tile as the !any path does after B1
    //  after the end barrier: flush when the buffer could not hold another tile's kmax entries, and at the end of the strip (one barrier
    //  more; the next appends follow the next tile's B1)
    for (int b = 0;; b ^= 1) {
        const int iniY = g.minB + (row0 + cur) * g.hCell, maxY = min(iniY + g.hCell + 6, g.maxBY);
        const int nrows = maxY - iniY, ny = nrows - 6;   // detection rows
        const uint8_t* const tile = fsm + SM.tile + b * SM.tileBytes + 16;
        const uint16_t* const liveS = reinterpret_cast<const uint16_t*>(fsm + SM.live + b * SM.liveBytes) + (rowLo[cur] & 7u);
        const uint32_t nLive = live ? rowHi[cur] - rowLo[cur] : 0u;
        // S2 must read 0 around the scored area (rows 0 and ny+1, the pair-words left/right of [2*w0, 2*w1)) and wherever phase A skips an item
        {
            const int q0 = X.q0, nq = X.q1 - X.q0; const uint32_t mgZero = mg.y;
            for (int i = tid; i < (ny + 2) * nq; i += 256) {
                const int r = fdiv_small(i, mgZero);
                reinterpret_cast<uint4*>(S2 + r * FAST_SW)[q0 + i - r * nq] = make_uint4(0u, 0u, 0u, 0u);
            }
        }
        if (tid == 0) { nK = 0; nPass = 0; nDef = 0; nHi = 0; nLo = 0; hit = 0u; }
        asm volatile("cp.async.wait_group 0;\n" ::: "memory");
        // caller canvases: an all-zero tile has no corners at any threshold (OR of the columns this thread staged)
        uint32_t acc = live ? 1u : 0u;
        if (!live && (tid & 15) < X.nvec)
            for (int r = tid >> 4; r < nrows; r += 16) {
                const uint4 v = *reinterpret_cast<const uint4*>(tile + r * FAST_TS + 16 * (tid & 15));
                acc |= v.x | v.y | v.z | v.w;
            }
        const int any = __syncthreads_or(acc);   // B1
        int next = cur + 1;
        while (next < nr && !rowVisit[next]) next++;
        if (next < nr) stage(next, b ^ 1);
        if (!any) {   // nothing reads S2, the counters or buffer b after B1 (the output buffer is as the last end barrier left it)
            if (next == nr) break;
            cur = next;
            continue;
        }
        // ---- A0: the compass words of score_item (rows 0, 3 and 6 of the item: ring 0, 4 / 12 and centre, 8) and their bound.
        // compass_x2 ignores the low bytes, so the words of centres 0 and 2 need not be funnel shifts: a word shifted left by 8 bits puts
        // its bytes 0 and 2 in the high bytes of its lanes (a multiply by 256, on the FMA pipe rather than the integer pipe). Ring 0 / 8
        // of centres 0, 2 are bytes 0, 2 of the row-0 / row-6 word, ring 4 the same of ring 4's word of centres 1, 3 (V4), ring 12 bytes 1, 3
        // of the word left of the centre row (m), and the centres bytes 0, 2 of the centre word.
        {
            const int w0 = X.w0;
            const uint32_t T1 = T | 0x00ff00ffu, T1i = (uint32_t)ti * 0x01000100u | 0x00ff00ffu;
            // the bound of item e (encoded as the live list) at mt: T1 where it proves all 4 scores <= mt; above T1i where it cannot prove
            // them <= ti (T1i >= T1, and a lane's bound exceeds t << 8 | 0xff exactly where its margin exceeds t)
            auto bound = [&](int e) {
                const uint32_t* r0 = reinterpret_cast<const uint32_t*>(tile + (e >> 6) * FAST_TS + 4 * (w0 + (e & 63)));
                const int RS = FAST_TS / 4;
                const uint32_t* r3 = r0 + 3 * RS; const uint32_t* r6 = r0 + 6 * RS;
                const uint32_t uc = r0[0], m = r3[-1], c = r3[0], p = r3[1], dc = r6[0];
                const uint32_t V4 = __funnelshift_r(c, p, 24);
                const uint32_t b02 = compass_x2(uc * 256u, V4 * 256u, dc * 256u, m, c * 256u, T1);
                return compass_x2(uc, V4, dc, __funnelshift_r(m, c, 8), c, b02);
            };
            // items that can score above ti go to the pass list, the others that can score above mt to the deferred list, in the same
            // encoding (ptxas aggregates each atomic: one ATOMS per warp)
            auto append = [&](int e) {
                const uint32_t v = bound(e);
                if (__vmaxu2(v, T1i) != T1i) passS[atomicAdd(&nPass, 1)] = (uint16_t)e;
                else if (v != T1) passS[SM.listCap - 1 - atomicAdd(&nDef, 1)] = (uint16_t)e;
            };
            if (live) {
                for (uint32_t it = tid; it < nLive; it += 256) append(liveS[it]);
            } else {
                const int nw = X.w1 - w0; const uint32_t mgItems = mg.x;
                for (int it = tid; it < nw * ny; it += 256) {
                    const int y = fdiv_small(it, mgItems);
                    append(y << 6 | (it - y * nw));
                }
            }
        }
        __syncthreads();   // BP
        const int npass = nPass;
        if (npass == 0 && nDef == 0) {   // no item can score: nothing reads S2, the lists, the counters or buffer b after BP
            if (next == nr) break;
            cur = next;
            continue;
        }
        // Exact arc scores of item wi of detection row y into S2 (nothing is stored for an all-zero item: S2 already reads 0 there). Returns
        // 0 for an all-zero item, 2 if some lane is above ti (> TH), else 1
        auto score_item = [&](int y, int wi) {
            const int to = y * FAST_TS + 4 * wi;   // byte offset of the item in tile row y, the row 3 above its centres
            const uint32_t* r0 = reinterpret_cast<const uint32_t*>(tile + to);
            const int RS = FAST_TS / 4;
            // The word left of the item (m) feeds only centres 0..2 of item 0, which lie left of the detection area when w0 = 0 (xoff >= 3),
            // so it is read unguarded. Read as u16x2, a word starting dx pixels right of the item holds ring pixel dx of centres 1 and 3 in the high bytes of its
            // lanes (V), and the word one pixel further left holds those of centres 0 and 2 (U). ring k: (dx, dy) of the FAST-16 circle.
            // arc_score_x2 reads only the high bytes, so where U[k] is no loaded word it is V[k] shifted left by 8 bits (V[k]'s low
            // bytes are U's pixels): a multiply by 256 on the FMA pipe instead of a funnel shift on the integer pipe
            uint32_t V[16], U[16], Cv, Cu;
            {   // dy=-3: ring 15 (dx-1), 0 (dx 0), 1 (dx+1)
                const uint32_t m = r0[-1], c = r0[0], p = r0[1];
                V[15] = __funnelshift_r(m, c, 24); V[0] = c; V[1] = __funnelshift_r(c, p, 8);
                U[15] = V[15] * 256u; U[0] = V[15]; U[1] = c;
            }
            {   // dy=-2: ring 14 (dx-2), 2 (dx+2)
                const uint32_t* r = r0 + RS; const uint32_t m = r[-1], c = r[0], p = r[1];
                V[14] = __funnelshift_r(m, c, 16); V[2] = __funnelshift_r(c, p, 16);
                U[14] = V[14] * 256u; U[2] = V[2] * 256u;
            }
            {   // dy=-1: ring 13 (dx-3), 3 (dx+3)
                const uint32_t* r = r0 + 2 * RS; const uint32_t m = r[-1], c = r[0], p = r[1];
                V[13] = __funnelshift_r(m, c, 8); V[3] = __funnelshift_r(c, p, 24);
                U[13] = m; U[3] = V[3] * 256u;
            }
            {   // dy=0: ring 12 (dx-3), 4 (dx+3), centre
                const uint32_t* r = r0 + 3 * RS; const uint32_t m = r[-1], c = r[0], p = r[1];
                V[12] = __funnelshift_r(m, c, 8); V[4] = __funnelshift_r(c, p, 24); Cv = c;
                U[12] = m; U[4] = V[4] * 256u; Cu = c * 256u;
            }
            {   // dy=+1: ring 11 (dx-3), 5 (dx+3)
                const uint32_t* r = r0 + 4 * RS; const uint32_t m = r[-1], c = r[0], p = r[1];
                V[11] = __funnelshift_r(m, c, 8); V[5] = __funnelshift_r(c, p, 24);
                U[11] = m; U[5] = V[5] * 256u;
            }
            {   // dy=+2: ring 10 (dx-2), 6 (dx+2)
                const uint32_t* r = r0 + 5 * RS; const uint32_t m = r[-1], c = r[0], p = r[1];
                V[10] = __funnelshift_r(m, c, 16); V[6] = __funnelshift_r(c, p, 16);
                U[10] = V[10] * 256u; U[6] = V[6] * 256u;
            }
            {   // dy=+3: ring 9 (dx-1), 8 (dx 0), 7 (dx+1)
                const uint32_t* r = r0 + 6 * RS; const uint32_t m = r[-1], c = r[0], p = r[1];
                V[9] = __funnelshift_r(m, c, 24); V[8] = c; V[7] = __funnelshift_r(c, p, 8);
                U[9] = V[9] * 256u; U[8] = V[9]; U[7] = c;
            }
            const uint32_t s13 = arc_score_x2(V, Cv, T), s02 = arc_score_x2(U, Cu, T);
            // back to pair-word order (pixels 0,1) (2,3). Lanes outside the detection area keep what they scored: phase B masks them
            // (S2 row y+1 holds tile row y's 4 pixels of an item in 8 bytes at twice the tile offset)
            const uint32_t mx = __vmaxu2(s02, s13);
            if (mx != 0u)
                *reinterpret_cast<uint2*>(reinterpret_cast<uint8_t*>(S2) + 4 * FAST_SW + 2 * to) =
                    make_uint2(__byte_perm(s02, s13, 0x5410), __byte_perm(s02, s13, 0x7632));
            if (mx == 0u) return 0;
            const uint32_t th = TH;
            return __vmaxu2(mx, th) != th ? 2 : 1;
        };
        // ---- A: items scored non-zero go to nzHi or nzLo, in the same encoding. ptxas aggregates each atomic: one ATOMS per warp
        // (tools/kfast_sass.py). The entry is read again after the score rather than held across it (register pressure)
        {
            const int w0 = X.w0;
            for (int it = tid; it < npass; it += 256) {
                const int e = passS[it];
                const int k = score_item(e >> 6, w0 + (e & 63));
                if (k == 2) nzS[atomicAdd(&nHi, 1)] = passS[it];
                else if (k == 1) nzS[SM.listCap - 1 - atomicAdd(&nLo, 1)] = passS[it];
            }
        }
        __syncthreads();   // B2
        // ---- B: NMS at mt in u16x2 lanes: keep s iff every same-cell neighbour is < s (all stored scores are > mt). A pair-word can be
        // non-zero only inside an item phase A (or round 2) scored non-zero, so B walks the nz lists; one thread reads the item's 3 x 4
        // pair-word neighbourhood once.
        // Lanes outside the detection area hold scores of pixels outside it: the current pair-words are masked to the valid lanes, and a valid
        // lane's neighbours are valid or masked by the left / right masks (the rows above and below are the same columns, or the zeroed rows).
        // Round 1 (fb = false) keeps the survivors above ti (the floor TH) and marks their cells in `hit`; round 2 (fb = true) skips the items
        // without a pixel in the cells of fm and keeps every survivor in those cells
        auto nms_item = [&](int y, int wi, bool fb, uint32_t fm) {
            const uint4 hd = items[2 * wi];
            if (fb && !(hd.w & fm)) return;
            const uint32_t* r1 = S2 + (y + 1) * FAST_SW + 2 * wi;
            uint2 cu = *reinterpret_cast<const uint2*>(r1);
            cu.x &= hd.x; cu.y &= hd.y;
            if ((cu.x | cu.y) == 0) return;
            const uint32_t* r0 = r1 - FAST_SW; const uint32_t* r2 = r1 + FAST_SW;
            const uint2 up = *reinterpret_cast<const uint2*>(r0), dn = *reinterpret_cast<const uint2*>(r2);
            const uint32_t uL = wi > 0 ? r0[-1] : 0u, cL = wi > 0 ? r1[-1] : 0u, dL = wi > 0 ? r2[-1] : 0u;
            const uint32_t uR = r0[2], cR = r1[2], dR = r2[2];
            const uint4 lr = items[2 * wi + 1];
            const uint32_t fl = fb ? 0u : TH;
            const uint32_t M0 = nms_max(uL, up.x, up.y, cL, cu.x, cu.y, dL, dn.x, dn.y, lr.x, lr.z, fl);
            const uint32_t M1 = nms_max(up.x, up.y, uR, cu.x, cu.y, cR, dn.x, dn.y, dR, lr.y, lr.w, fl);
            // survivors: the lanes where c > m. Every lane holds a multiple of 256 (the stored scores' low bytes are 0), so max(c, m) - m
            // never borrows and its high byte is non-zero exactly there; byte j of `keep` is that byte of pixel j
            uint32_t keep = __byte_perm(__vmaxu2(cu.x, M0) - M0, __vmaxu2(cu.y, M1) - M1, 0x7531);
            const int xoff = X.xoff;
            while (keep) {
                const int j = (__ffs(keep) - 1) >> 3;
                keep &= ~(0xffu << (8 * j));
                const int cell = (hd.z >> (2 * j)) & 3;
                if (fb && !((fm >> cell) & 1u)) continue;
                const uint32_t sv = ((j < 2 ? cu.x : cu.y) >> (16 * (j & 1))) & 0xffff;
                const int x = 4 * wi + j - xoff, s = (int)(sv >> 8) + mt;
                const int pos = atomicAdd(&nK, 1);
                if (pos >= SM.kmax) *errFlag = CSLAM_E_CAPACITY;
                else klist[pos] = (uint32_t)x | ((uint32_t)y << 8) | ((uint32_t)s << 16);
                if (!fb) atomicOr(&hit, 1u << cell);
            }
        };
        {   // round 1
            const int w0 = X.w0, nh = nHi;
            for (int it = tid; it < nh; it += 256) { const int e = nzS[it]; nms_item(e >> 6, w0 + (e & 63), false, 0u); }
        }
        __syncthreads();   // B3
        // F: the tile's cells without a keypoint at ti (block-uniform: hit is final after B3 and nothing writes it before the end barrier)
        const uint32_t fm = ~hit & ((1u << min(CG, g.nColsEff - (int)blockIdx.x * CG)) - 1u);
        if (fm) {
            const int w0 = X.w0;
            {   // round 2 scoring: the deferred items with a pixel in F, appended to nzLo when non-zero
                const int nd = nDef;
                for (int it = tid; it < nd; it += 256) {
                    const int e = passS[SM.listCap - 1 - it], wi = w0 + (e & 63);
                    if ((items[2 * wi].w & fm) && score_item(e >> 6, wi)) nzS[SM.listCap - 1 - atomicAdd(&nLo, 1)] = passS[SM.listCap - 1 - it];
                }
            }
            __syncthreads();   // B4
            {   // round 2 NMS over nzHi and nzLo (at [listCap - nl, listCap)), in F only
                const int nh = nHi, nl = nLo;
                for (int it = tid; it < nh + nl; it += 256) {
                    const int e = nzS[it < nh ? it : SM.listCap - nl + (it - nh)];
                    nms_item(e >> 6, w0 + (e & 63), true, fm);
                }
            }
            __syncthreads();   // B5
        }
        // ---- C: each warp appends its stride of klist with one shared atomic; the buffer has room for nk <= kmax entries
        const int nk = min(nK, SM.kmax);
#pragma unroll 1
        for (int i = tid - lane; i < nk; i += 256) {   // warp-uniform bounds
            uint32_t v = 0; const bool sel = i + lane < nk;
            if (sel) {
                const uint32_t e = klist[i + lane];
                const uint32_t x = X.tx0 + 3 + (e & 0xff) - g.minB, y = iniY + 3 + ((e >> 8) & 0xff) - g.minB;
                v = x | (y << 12) | ((((e >> 16) & 0xff) - 1) << 24);
            }
            const unsigned ball = __ballot_sync(0xffffffffu, sel);
            int pos = 0;
            if (lane == 0) pos = atomicAdd(&nOut, __popc(ball));
            pos = __shfl_sync(0xffffffffu, pos, 0);
            if (sel) sout[pos + lane] = v;
        }
        __syncthreads();   // end barrier
        if (next == nr) break;
        if (nOut > FAST_OUT - SM.kmax) flush();
        cur = next;
    }
    if (nOut > 0) flush();   // after the last tile's end barrier, B1 or BP
}

// ------------------------------------------------------------------------------------------------- k_distribute
// DistributeOctTree (src/ORBExtractor.cpp:511-737) without lists or pointers. Facts used (DESIGN.md):
//  * children bounds depend only on the parent bounds; a key's child is decided by x<midX / y<midY;
//  * std::list::push_front everywhere => list order == descending creation sequence, so "list order" is a sort key;
//  * the order of keys inside a node only matters for the final "max response, first wins" pick, and the first key
//    of equal response is the one earliest in (cell row, cell col, y, x) order, recoverable from coordinates.
// One CTA per (level, frame). Nodes live in shared memory, keys stay in global/L2 with a per-key node index.
struct QNode { uint16_t ulx, uly, brx, bry; uint32_t cnt; uint32_t seq : 31; uint32_t flagE : 1; };

static const int DIST_THREADS = 256;
static const int DIST_WARPS = DIST_THREADS / 32;

// Dynamic shared memory of a k_distribute CTA (byte offsets) for a node capacity of M, a multiple of 32, so every region is 16-byte aligned
struct DistSmem {
    int list[2];   // node lists (QNode): a round reads one and writes the other
    int best;      // after the rounds: the best key of each node (u64), over list 0 (no node list is read after the rounds)
    int child;     // per node 4 x u32: key count of each child, then the child's new index (a kept node's new index in entry 0)
    int ord;       // per node u32: a candidate's split order (normal rounds: split flags, scanned in place)
    int kids;      // per split order u32: the candidate's non-empty children, scanned in place
    int keep;      // per node u32, finishing rounds: unsplit flags, scanned in place
    int split;     // per node u8: divided this round
    int total;
};
__host__ __device__ inline DistSmem dist_smem(int M) {
    DistSmem m;
    m.list[0] = 0;
    m.list[1] = m.list[0] + M * (int)sizeof(QNode);
    m.best = m.list[0];
    m.child = m.list[1] + M * (int)sizeof(QNode);
    m.ord = m.child + 16 * M;
    m.kids = m.ord + 4 * M;
    m.keep = m.kids + 4 * M;
    m.split = m.keep + 4 * M;
    m.total = (m.split + M + 15) & ~15;
    return m;
}
static_assert(sizeof(unsigned long long) <= sizeof(QNode), "best[i] fits in node i of list 0");

// ExtractorNode::DivideNode: a node's split point, which gives its children's bounds and the child (n1..n4 = 0..3) each key falls in
__device__ __forceinline__ int2 node_mid(const QNode& nd) {
    return make_int2(nd.ulx + ((nd.brx - nd.ulx + 1) >> 1), nd.uly + ((nd.bry - nd.uly + 1) >> 1));
}
__device__ __forceinline__ int key_child(const QNode& nd, uint32_t v) {
    const int2 m = node_mid(nd);
    const int x = v & 0xfff, y = (v >> 12) & 0xfff;
    return (x < m.x ? 0 : 1) + (y < m.y ? 0 : 2);
}

// In-place exclusive scan of data[0..n) by the whole CTA, each thread over a contiguous range; returns the total. The caller's writes
// to data must be visible (a barrier) before the call; the scan ends with a barrier.
__device__ __forceinline__ uint32_t block_exclusive_scan(uint32_t* data, int n, uint32_t* warpSums) {
    const int tid = threadIdx.x;
    const int per = (n + DIST_THREADS - 1) / DIST_THREADS;
    const int lo = min(tid * per, n), hi = min(lo + per, n);
    uint32_t s = 0;
    for (int i = lo; i < hi; i++) s += data[i];
    // block scan of s
    const int lane = tid & 31, wid = tid >> 5;
    uint32_t v = s;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { uint32_t t = __shfl_up_sync(0xffffffffu, v, o); if (lane >= o) v += t; }
    if (lane == 31) warpSums[wid] = v;
    __syncthreads();
    if (wid == 0) {
        uint32_t w = lane < DIST_WARPS ? warpSums[lane] : 0;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) { uint32_t t = __shfl_up_sync(0xffffffffu, w, o); if (lane >= o) w += t; }
        warpSums[lane] = w;
    }
    __syncthreads();
    uint32_t excl = v - s + (wid ? warpSums[wid - 1] : 0);
    const uint32_t total = warpSums[DIST_WARPS - 1];
    for (int i = lo; i < hi; i++) { uint32_t t = data[i]; data[i] = excl; excl += t; }
    __syncthreads();
    return total;
}

struct DistributeArgs {
    DevLevels L;
    const uint32_t* candCount;   // batch x nlevels
    uint32_t* kept;              // batch x nlevels x M : x | y<<12 | resp<<24 in LEVEL coordinates
    uint32_t* keptCount;         // batch x nlevels
    const uint8_t* mask; int maskPitch; int imgW, imgH, faceW, faceH;
    int M;                       // node capacity, and so the capacity of a (frame, level)'s kept list (one key per node)
    int* errFlag;
};

// A round divides its candidates: in a normal round every node with more than one key, in list order; in a finishing round (once the
// list is close to N) the expandable nodes in descending (count, seq), cut after the split that makes the list reach N. Steps of a round
// (cur / nxt: the node list read / written this round; block_exclusive_scan ends with a barrier), what each reads (r) and writes (w) in
// shared memory, and the barrier that ends it:
//  select     r cur; w split, ord, child = 0. Normal: ord = split flags -> barrier -> ord scan: ord = split order.
//             Finishing: ord = rank among the expandable nodes -> barrier
//  count      r split, cur; w child = each candidate's key count per child (shared atomics) -> barrier
//  children   r split, ord, child; w kids[ord] = the candidate's non-empty children; sh_nExp = 0 -> barrier -> kids scan: kids[o] =
//   scan      creation rank of candidate o's first child
//  cut        finishing only. r kids; w sh_J = the cut J -> barrier; r sh_J, ord; w split = 0 at ord >= J, keep = unsplit flags -> barrier
//             -> keep scan: keep = rank of a kept node among the kept nodes
//  emit       r cur, split, ord, kids, keep, child; w nxt, child = each child's new index (a kept node's in entry 0), sh_nExp -> barrier
//  move keys  r split, cur, child; w pnode (global) -> barrier
//  stop test  r sh_nExp; no barrier: the select barrier of the next round orders this read before the children step resets it
// After the rounds: best (over list 0) = max per node -> barrier; the cull compacts the nodes' best keys in list order, DIST_THREADS
// nodes at a time (a barrier after the per-warp counts, one before the next chunk rewrites them).
__global__ void __launch_bounds__(DIST_THREADS) k_distribute(DistributeArgs A) {
    extern __shared__ __align__(16) uint8_t dsm[];   // DistSmem
    const int M = A.M;
    const DistSmem SM = dist_smem(M);
    uint32_t* const child = reinterpret_cast<uint32_t*>(dsm + SM.child);
    uint32_t* const ord = reinterpret_cast<uint32_t*>(dsm + SM.ord);
    uint32_t* const kids = reinterpret_cast<uint32_t*>(dsm + SM.kids);
    uint32_t* const keep = reinterpret_cast<uint32_t*>(dsm + SM.keep);
    uint8_t* const split = dsm + SM.split;
    __shared__ uint32_t warpSums[32];
    __shared__ uint32_t warpKept[DIST_WARPS];
    __shared__ int sh_nExp, sh_J;
    const int level = blockIdx.x, frame = blockIdx.y, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const LevelGeom g = A.L.g[level];
    const int N = g.quota;

    const uint32_t nAll = A.candCount[(size_t)frame * A.L.nlevels + level];
    const int n = (int)min(nAll, (uint32_t)g.candCap);
    const uint32_t* pts = A.L.cand[level] + (size_t)frame * g.candCap;
    uint16_t* pnode = A.L.pnode[level] + (size_t)frame * g.candCap;
    uint32_t* keptOut = A.kept + ((size_t)frame * A.L.nlevels + level) * M;
    uint32_t* keptCnt = A.keptCount + (size_t)frame * A.L.nlevels + level;
    if (n == 0) { if (tid == 0) *keptCnt = 0; return; }

    QNode* cur = reinterpret_cast<QNode*>(dsm + SM.list[0]);
    QNode* nxt = reinterpret_cast<QNode*>(dsm + SM.list[1]);
    if (tid == 0) {
        QNode r; r.ulx = 0; r.uly = 0; r.brx = (uint16_t)(g.maxBX - g.minB); r.bry = (uint16_t)(g.maxBY - g.minB);
        r.cnt = (uint32_t)n; r.flagE = 0; r.seq = 0;
        cur[0] = r;
    }
    for (int p = tid; p < n; p += DIST_THREADS) pnode[p] = 0;
    __syncthreads();
    int nList = 1; uint32_t seqNext = 1; bool finishMode = false;
    int nExp = 0;   // expandable nodes (flagE) in cur: the candidates of a finishing round

    for (int round = 0; round < 64; round++) {
        const int prevSize = nList;
        // ---- select: the candidates and their split order
        int nCand;
        if (!finishMode) {
            for (int i = tid; i < nList; i += DIST_THREADS) {
                const bool s = cur[i].cnt > 1;
                split[i] = s; ord[i] = s;
                reinterpret_cast<uint4*>(child)[i] = make_uint4(0u, 0u, 0u, 0u);
            }
            __syncthreads();
            nCand = (int)block_exclusive_scan(ord, nList, warpSums);
        } else {
            nCand = nExp;
            // rank expandable nodes by descending (count, seq): the reference sorts ascending and walks from the back
            for (int i = tid; i < nList; i += DIST_THREADS) {
                int r = 0; const bool e = cur[i].flagE != 0;
                if (e) {
                    const uint32_t ci = cur[i].cnt, si = cur[i].seq;
                    for (int k = 0; k < nList; k++) {
                        if (!cur[k].flagE) continue;
                        const uint32_t ck = cur[k].cnt, sk = cur[k].seq;
                        r += (ck > ci) || (ck == ci && sk > si);
                    }
                }
                split[i] = e; ord[i] = (uint32_t)r;
                reinterpret_cast<uint4*>(child)[i] = make_uint4(0u, 0u, 0u, 0u);
            }
            __syncthreads();
        }
        if (nCand == 0) break;   // nothing can be divided (the reference would spin forever here; see DESIGN.md)
        // ---- count: children populations
        for (int p = tid; p < n; p += DIST_THREADS) {
            const int i = pnode[p];
            if (split[i]) atomicAdd(&child[4 * i + key_child(cur[i], pts[p])], 1u);
        }
        __syncthreads();
        // ---- children scan: kids[o] = the creation rank of candidate o's first child (reference creation order = split order, n1..n4)
        for (int i = tid; i < nList; i += DIST_THREADS)
            if (split[i]) {
                const uint4 c = reinterpret_cast<const uint4*>(child)[i];
                kids[ord[i]] = (c.x > 0) + (c.y > 0) + (c.z > 0) + (c.w > 0);
            }
        if (tid == 0) sh_nExp = 0;
        __syncthreads();
        const uint32_t kidsTotal = block_exclusive_scan(kids, nCand, warpSums);
        // ---- finishing cut: stop after the split that makes the list reach N. The list holds before(o) = prevSize + kids[o] - o nodes before
        // candidate o is divided; every candidate has a non-empty child, so before() does not decrease, and before(0) = prevSize < N. The cut
        // J is the first o with before(o) >= N, or nCand: exactly one o in 1..nCand has before(o - 1) < N and (o == nCand or before(o) >= N)
        int J = nCand;
        if (finishMode) {
            for (int o = tid + 1; o <= nCand; o += DIST_THREADS)
                if (prevSize + (int)kids[o - 1] - (o - 1) < N && (o == nCand || prevSize + (int)kids[o] - o >= N)) sh_J = o;
            __syncthreads();
            J = sh_J;
            for (int i = tid; i < nList; i += DIST_THREADS) {
                if (split[i] && (int)ord[i] >= J) split[i] = 0;
                keep[i] = !split[i];
            }
            __syncthreads();
            block_exclusive_scan(keep, nList, warpSums);
        }
        const int C = J < nCand ? (int)kids[J] : (int)kidsTotal;   // children created
        const int newSize = C + nList - J;
        if (newSize > M) { if (tid == 0) *A.errFlag = CSLAM_E_CAPACITY; break; }
        // ---- emit: children at C - 1 - rank (push_front), then the kept nodes in list order
        int myExp = 0;
        for (int i = tid; i < nList; i += DIST_THREADS) {
            const QNode nd = cur[i];
            if (split[i]) {
                const int2 m = node_mid(nd);
                int r = (int)kids[ord[i]];
                for (int q = 0; q < 4; q++) {
                    const uint32_t c = child[4 * i + q];
                    if (c == 0) continue;
                    QNode ch;
                    ch.ulx = (q & 1) ? m.x : nd.ulx; ch.brx = (q & 1) ? nd.brx : m.x;
                    ch.uly = (q & 2) ? m.y : nd.uly; ch.bry = (q & 2) ? nd.bry : m.y;
                    ch.cnt = c; ch.flagE = c > 1; ch.seq = seqNext + r;
                    const int pos = C - 1 - r;
                    nxt[pos] = ch;
                    child[4 * i + q] = (uint32_t)pos;
                    myExp += c > 1;
                    r++;
                }
            } else {
                // a normal round splits or keeps every node, so ord[i] nodes before i were split
                const int pos = C + (finishMode ? (int)keep[i] : i - (int)ord[i]);
                QNode kn = nd; kn.flagE = 0;
                nxt[pos] = kn;
                child[4 * i] = (uint32_t)pos;
            }
        }
        if (myExp) atomicAdd(&sh_nExp, myExp);
        __syncthreads();
        // ---- move keys
        for (int p = tid; p < n; p += DIST_THREADS) {
            const int i = pnode[p];
            pnode[p] = (uint16_t)child[4 * i + (split[i] ? key_child(cur[i], pts[p]) : 0)];
        }
        __syncthreads();
        // ---- stop test
        nExp = sh_nExp;
        { QNode* t = cur; cur = nxt; nxt = t; }
        nList = newSize; seqNext += C;
        if (!finishMode) {
            if (nList >= N || (nList == prevSize && nList >= N / 100)) break;
            if (nList + 3 * nExp > N) finishMode = true;
        } else {
            if (nList >= N || nList == prevSize) break;
        }
    }
    __syncthreads();
    // ---- best key per node: max response, ties -> earliest in (cell row, cell col, y, x) order
    unsigned long long* best = reinterpret_cast<unsigned long long*>(dsm + SM.best);
    for (int i = tid; i < nList; i += DIST_THREADS) best[i] = 0ull;
    __syncthreads();
    for (int p = tid; p < n; p += DIST_THREADS) {
        const uint32_t v = pts[p];
        const uint32_t x = v & 0xfff, y = (v >> 12) & 0xfff, r = v >> 24;
        const uint32_t cy = (y - 3) / g.hCell, cx = (x - 3) / g.wCell;
        const unsigned long long key = ((unsigned long long)cy << 32) | ((unsigned long long)cx << 24) | ((unsigned long long)y << 12) | x;
        const unsigned long long packed = ((unsigned long long)(r + 1) << 40) | (0xffffffffffull - key);
        atomicMax(&best[pnode[p]], packed);
    }
    __syncthreads();
    // ---- cull (src/ORBExtractor.cpp:883-904) in list order: ordered compaction by warp ballots, DIST_THREADS nodes at a time
    uint32_t base = 0;   // keys kept from the earlier chunks
    for (int c0 = 0; c0 < nList; c0 += DIST_THREADS) {
        const int i = c0 + tid;
        bool kp = false; uint32_t packedOut = 0;
        if (i < nList) {
            const unsigned long long b = best[i];
            const uint32_t key = (uint32_t)(0xffffffffffull - (b & 0xffffffffffull));
            const uint32_t x = key & 0xfff, y = (key >> 12) & 0xfff, r = (uint32_t)(b >> 40) - 1;
            const uint32_t lx = x + g.minB, ly = y + g.minB;
            const float ptx = __fmul_rn((float)lx, g.scale), pty = __fmul_rn((float)ly, g.scale);
            const bool face = face_of_pixel_f(ptx, pty, A.faceW, A.faceH) >= 0;
            const int mxI = (int)__fadd_rn(ptx, 0.5f), myI = (int)__fadd_rn(pty, 0.5f);
            kp = face && !(ptx < 0 || mxI >= A.imgW || pty < 0 || myI >= A.imgH);
            if (kp) kp = A.mask[(size_t)myI * A.maskPitch + mxI] != 0;
            packedOut = lx | (ly << 12) | (r << 24);
        }
        const unsigned ball = __ballot_sync(0xffffffffu, kp);
        if (lane == 0) warpKept[warp] = __popc(ball);
        __syncthreads();
        uint32_t before = 0, tot = 0;
        for (int w = 0; w < DIST_WARPS; w++) { const uint32_t t = warpKept[w]; before += w < warp ? t : 0u; tot += t; }
        if (kp) {
            const uint32_t pos = base + before + __popc(ball & ((1u << lane) - 1));
            if (pos < (uint32_t)M) keptOut[pos] = packedOut; else *A.errFlag = CSLAM_E_CAPACITY;
        }
        base += tot;
        __syncthreads();   // warpKept is rewritten by the next chunk
    }
    if (tid == 0) *keptCnt = min(base, (uint32_t)M);
}

// ------------------------------------------------------------------------------------------------- k_describe
struct DescribeArgs {
    DevLevels L;
    const uint32_t* kept; const uint32_t* keptCount; int M;   // M: kept-list stride (DistributeArgs)
    cslam_keypoint* kps; uint8_t* desc; int32_t* nOut; int kpCap;
    int* errFlag;
};

// The 7x7 blur runs on the integer tensor cores: OpenCV's 8U fixed point is exact in integers (H = sum g P <= 65280, dst = (sum g H + 32768)
// >> 16 with g = [18,34,48,56,48,34,18]), and mma.sync m16n8k32 u8 x u8 -> s32 gives the same bits.
//   pass 1  Ht[c][n] = sum_j G[c][j] P[pi(n)][j]: A = band G[c][j] = g[j - po - c] (M = output column c, 37 -> 48; K = patch column j, 64),
//           B = the row-major patch, loaded as-is with ldmatrix, its rows permuted by pi so that the accumulators come out as pass 2's operands;
//   pass 2  V[r][c] = sum_k Gv[r][k] H[k][c] on the two byte planes of H: A = band Gv[r][k] = g[k - r] (M = output row, 37 -> 48; K = H row),
//           B = Hh, then Hl accumulated onto 256 Vh + 32768, so dst is byte 2 of the sum.
// pi: in the n-tile pair (2p, 2p+1), column 2t + e holds patch row 16p + 4t + e of tile 2p and 16p + 4t + 2 + e of tile 2p+1. Lane (g, t)'s
// accumulators then hold H rows 16p + 4t .. 16p + 4t + 3 of Ht row c = 16mt + g (+8), which is exactly its pass-2 B fragment (K rows 4t..4t+3
// of column g): four byte permutes per fragment and plane, no shared-memory round trip.
// Band-limited tiles are skipped: pass 1 runs (mt, kt) = (0,0) (0,1) (1,0) (1,1) (2,1), pass 2 runs (mt, kt) = (0,0) (1,0) (1,1) (2,1) and no
// n-tile 5 (columns 40..47): 30 + 40 IMMA per key point.
static const int DP_STRIDE = 64;    // patch row stride: four 16-byte chunks; chunk q of row r is stored at chunk q ^ ((r >> 2) & 3) (dp_at)
static const int DP_ROWS = 48;      // rows the pass-1 n-tiles read; rows 43..47 (never written) only reach blurred rows 37..47, which are discarded
static const int BL_STRIDE = 48;    // blurred patch row stride (12 words: the 8 rows of a fragment's u16 stores fall in distinct banks)
static const int BL_ROWS = 40;      // blurred rows stored: 0..36 are read, 37..39 are the m-tile's padding
// Band operands: the A register of lane (g, t) for tile (mt, kt), half h of K and rows +8v is bytes g[d .. d+3] with d = 4t - g - po + 8s,
// s = 4kt + 2h - 2mt - v (po = 0 in pass 2). A word table indexed by d gives each of them as one shared load at a constant offset from a
// per-lane base, so the per-key-point band for any po costs 10 loads (pass 2: 8) and no byte shuffling.
static const int BAND_LO = -46, BAND_N = 107;   // band word table: bytes g[d .. d+3] for d in [-46, 60]
// A lane's ldmatrix rows of one 8x16-byte matrix are 16p + {0,1,4,5,8,9,12,13} (+2): with a 64-byte stride even and odd rows fall in
// different halves of the 128 bytes, and the swizzle spreads rows 4 apart over the four chunks of a half, so no two rows share banks.
__device__ __forceinline__ int dp_at(int r, int x) { return r * DP_STRIDE + (x ^ (((r >> 2) & 3) << 4)); }

__device__ __forceinline__ void ldsm_x4(uint32_t (&b)[4], uint32_t addr) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];\n" : "=r"(b[0]), "=r"(b[1]), "=r"(b[2]), "=r"(b[3]) : "r"(addr) : "memory");
}
__device__ __forceinline__ void ldsm_x2(uint32_t (&b)[2], uint32_t addr) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x2.shared.b16 {%0,%1}, [%2];\n" : "=r"(b[0]), "=r"(b[1]) : "r"(addr) : "memory");
}
// d = A (16x32 u8, row) * B (32x8 u8, col) + c
__device__ __forceinline__ void mma_u8(uint32_t (&d)[4], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, uint32_t b0, uint32_t b1, const uint32_t (&c)[4]) {
    asm("mma.sync.aligned.m16n8k32.row.col.s32.u8.u8.s32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%10,%11,%12,%13};\n"
        : "=r"(d[0]), "=r"(d[1]), "=r"(d[2]), "=r"(d[3])
        : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1), "r"(c[0]), "r"(c[1]), "r"(c[2]), "r"(c[3]));
}

__global__ void __launch_bounds__(DESC_WARPS * 32) k_describe(DescribeArgs A) {
    __shared__ __align__(16) uint8_t s_patch[DESC_WARPS][DP_ROWS * DP_STRIDE];
    __shared__ __align__(16) uint8_t s_bl[DESC_WARPS][BL_ROWS * BL_STRIDE];
    __shared__ uint32_t s_band[BAND_N];
    if (threadIdx.x < BAND_N) {   // word d - BAND_LO: bytes g[d], g[d+1], g[d+2], g[d+3] (0 outside the kernel's 7 taps)
        const unsigned long long G = 0x12ull | 0x22ull << 8 | 0x30ull << 16 | 0x38ull << 24 | 0x30ull << 32 | 0x22ull << 40 | 0x12ull << 48;
        const int d = (int)threadIdx.x + BAND_LO;
        uint32_t w = 0;
        for (int i = 0; i < 4; i++)
            if (d + i >= 0 && d + i < 7) w |= (uint32_t)((G >> (8 * (d + i))) & 0xff) << (8 * i);
        s_band[threadIdx.x] = w;
    }
    __syncthreads();
    const int frame = blockIdx.y;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    // output slot -> (level, slot in the level's kept list): lane l < MAX_LEVELS holds the inclusive prefix sum of the kept counts up to
    // level l (the scan spans 16 lanes: lanes >= MAX_LEVELS hold partial sums and take no part below)
    const int outIdx = blockIdx.x * DESC_WARPS + warp;
    const int cnt = lane < A.L.nlevels ? (int)A.keptCount[(size_t)frame * A.L.nlevels + lane] : 0;
    int incl = cnt;
#pragma unroll
    for (int o = 1; o < MAX_LEVELS; o <<= 1) { const int t = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += t; }
    const int total = __shfl_sync(0xffffffffu, incl, MAX_LEVELS - 1);
    if (outIdx == 0 && lane == 0) {
        A.nOut[frame] = min(total, A.kpCap);
        if (total > A.kpCap) *A.errFlag = CSLAM_E_CAPACITY;
    }
    if (outIdx >= min(total, A.kpCap)) return;
    const int level = __popc(__ballot_sync(0xffffffffu, lane < A.L.nlevels && incl <= outIdx));   // levels that end at or before outIdx
    const int slot = outIdx - __shfl_sync(0xffffffffu, incl - cnt, level);
    const LevelGeom g = A.L.g[level];
    const uint8_t* I = A.L.img[level] + (size_t)frame * g.pitch * g.h;
    const uint32_t v = A.kept[((size_t)frame * A.L.nlevels + level) * A.M + slot];
    const int kx = v & 0xfff, ky = (v >> 12) & 0xfff, resp = v >> 24;
    // the key-point record, written before the blur so that none of its fields stays live across it; the angle follows at the end
    cslam_keypoint* kpo = A.kps + (size_t)frame * A.kpCap + outIdx;
    if (lane == 0) {
        kpo->x = __fmul_rn((float)kx, g.scale); kpo->y = __fmul_rn((float)ky, g.scale);
        kpo->size = g.sizeF; kpo->response = (float)resp; kpo->octave = level; kpo->class_id = -1;
    }

    // ---- 43x43 neighbourhood -> patch row r, byte po + c (REFLECT_101 at the level edges, like the blur of the apron-less clone)
    uint8_t* P = s_patch[warp];
    int po;
    if (kx >= 21 && ky >= 21 && kx + 21 < g.w && ky + 21 < g.h) {
        // interior: 16-byte loads (rows are 16-byte aligned: the pitch is a multiple of 128), all issued before the first store. A row needs
        // chunks 0..2, and chunk 3 when po > 5; that chunk starts at or before column kx + 21 < w, so it ends inside the row's pitch.
        const int x0 = kx - 21, xa = x0 & ~15;
        po = x0 - xa;
        const int nch = (po + 43 + 15) >> 4;
        const uint8_t* base = I + (size_t)(ky - 21) * g.pitch + xa;
        uint4 q[6];
#pragma unroll
        for (int k = 0; k < 6; k++) {
            const int i = lane + 32 * k, r = i >> 2, ch = i & 3;
            if (i < 43 * 4 && ch < nch) q[k] = __ldg(reinterpret_cast<const uint4*>(base + (size_t)r * g.pitch) + ch);
        }
#pragma unroll
        for (int k = 0; k < 6; k++) {
            const int i = lane + 32 * k, r = i >> 2, ch = i & 3;
            if (i < 43 * 4 && ch < nch) *reinterpret_cast<uint4*>(P + dp_at(r, 16 * ch)) = q[k];
        }
    } else {
        po = 0;
        for (int i = lane; i < 43 * 43; i += 32) {
            const int r = i / 43, c = i - r * 43;
            const int yy = reflect101(ky - 21 + r, g.h), xx = reflect101(kx - 21 + c, g.w);
            P[dp_at(r, c)] = __ldg(I + (size_t)yy * g.pitch + xx);
        }
    }
    __syncwarp();
    // ---- IC_Angle on the unblurred patch: lane = column u in [-15,15], rows +-v in pairs; bit v of g_icRows[lane] = (|u| <= umax[v])
    int m10 = 0, m01 = 0;
    if (lane < 31) {
        const int u = lane - HALF_PATCH;
        const uint32_t rows = __ldg(g_icRows + lane);
        const int x = po + 21 + u;
        int colsum = (rows & 1u) ? P[dp_at(21, x)] : 0;
#pragma unroll
        for (int v = 1; v <= HALF_PATCH; v++) {
            const int lo = P[dp_at(21 - v, x)], hi = P[dp_at(21 + v, x)];
            if (rows & (1u << v)) { colsum += lo + hi; m01 += v * (hi - lo); }
        }
        m10 = u * colsum;
    }
#pragma unroll
    for (int o = 16; o; o >>= 1) { m10 += __shfl_xor_sync(0xffffffffu, m10, o); m01 += __shfl_xor_sync(0xffffffffu, m01, o); }
    const float angle = fast_atan2_deg((float)m01, (float)m10);
    // ---- 7x7 sigma-2 Gaussian on IMMA (see above), only where BRIEF can sample (+-18): 37 x 37 outputs into Bl
    uint8_t* Bl = s_bl[warp];
    {
        const int gq = lane >> 2, tq = lane & 3;
        // band words: pass 1 A register (mt, kt, h, v) is word d = 4t - g - po + 8s with s = 4kt + 2h - 2mt - v, s in [-3, 6];
        // pass 2 the same with po = 0, s in [-3, 4]
        uint32_t a1[10], a2[8];
#pragma unroll
        for (int s = -3; s <= 6; s++) a1[s + 3] = s_band[4 * tq - gq - po + 8 * s - BAND_LO];
#pragma unroll
        for (int s = -3; s <= 4; s++) a2[s + 3] = s_band[4 * tq - gq + 8 * s - BAND_LO];
        // ldmatrix row addresses: lane L gives row 4((L & 7) >> 1) + (L & 1) (+ the n-tile's 16p + 2e) of matrix L >> 3; x4 = chunks 0..3, x2 = 2..3
        const int rb = 4 * ((lane & 7) >> 1) + (lane & 1), sw = (rb >> 2) & 3;
        const uint32_t pb = (uint32_t)__cvta_generic_to_shared(P) + rb * DP_STRIDE;
        const uint32_t ad4 = pb + 16 * ((lane >> 3) ^ sw), ad2 = pb + 16 * ((2 + ((lane >> 3) & 1)) ^ sw);
        const uint32_t zero[4] = {0u, 0u, 0u, 0u};
#define A1(mt, kt) a1[4 * (kt) - 2 * (mt) + 3], a1[4 * (kt) - 2 * (mt) + 2], a1[4 * (kt) - 2 * (mt) + 5], a1[4 * (kt) - 2 * (mt) + 4]
#define A2(mt, kt) a2[4 * (kt) - 2 * (mt) + 3], a2[4 * (kt) - 2 * (mt) + 2], a2[4 * (kt) - 2 * (mt) + 5], a2[4 * (kt) - 2 * (mt) + 4]
#pragma unroll
        for (int mt = 0; mt < 3; mt++) {
            // pass 1, m-tile mt: Ht rows 16mt + g (+8) against all 48 patch rows
            uint32_t h[6][4];
#pragma unroll
            for (int nt = 0; nt < 6; nt++) {
                const uint32_t roff = (16 * (nt >> 1) + 2 * (nt & 1)) * DP_STRIDE;
                if (mt < 2) {
                    uint32_t b[4];
                    ldsm_x4(b, ad4 + roff);
                    mma_u8(h[nt], A1(mt, 0), b[0], b[1], zero);
                    mma_u8(h[nt], A1(mt, 1), b[2], b[3], h[nt]);
                } else {   // columns 32..47 meet only patch columns 32..63
                    uint32_t b[2];
                    ldsm_x2(b, ad2 + roff);
                    mma_u8(h[nt], A1(mt, 1), b[0], b[1], zero);
                }
            }
            // pass 2 on n-tiles 2mt + v (columns 16mt + 8v + g): B fragment p (K rows 16p + 4t .. +3) of each byte plane
#pragma unroll
            for (int v = 0; v < 2; v++) {
                if (mt == 2 && v == 1) continue;   // columns 40..47
                uint32_t lo[3], hi[3];
#pragma unroll
                for (int p = 0; p < 3; p++) {
                    const uint32_t y01 = __byte_perm(h[2 * p][2 * v], h[2 * p][2 * v + 1], 0x5410), y23 = __byte_perm(h[2 * p + 1][2 * v], h[2 * p + 1][2 * v + 1], 0x5410);
                    lo[p] = __byte_perm(y01, y23, 0x6420);
                    hi[p] = __byte_perm(y01, y23, 0x7531);
                }
                // high plane first; its products, times 256 plus the rounding 32768, are the low plane's accumulator inputs
                uint32_t vs[3][4];
                mma_u8(vs[0], A2(0, 0), hi[0], hi[1], zero);
                mma_u8(vs[1], A2(1, 0), hi[0], hi[1], zero);
                mma_u8(vs[1], A2(1, 1), hi[2], 0u, vs[1]);
                mma_u8(vs[2], A2(2, 1), hi[2], 0u, zero);
#pragma unroll
                for (int m2 = 0; m2 < 3; m2++)
#pragma unroll
                    for (int i = 0; i < (m2 == 2 ? 2 : 4); i++) vs[m2][i] = vs[m2][i] * 256u + 32768u;   // rows 40..47 are discarded
                mma_u8(vs[0], A2(0, 0), lo[0], lo[1], vs[0]);
                mma_u8(vs[1], A2(1, 0), lo[0], lo[1], vs[1]);
                mma_u8(vs[1], A2(1, 1), lo[2], 0u, vs[1]);
                mma_u8(vs[2], A2(2, 1), lo[2], 0u, vs[2]);
                const int col = 16 * mt + 8 * v + 2 * tq;
#pragma unroll
                for (int m2 = 0; m2 < 3; m2++)
#pragma unroll
                    for (int hv = 0; hv < (m2 == 2 ? 1 : 2); hv++)   // dst = byte 2 of 256 Vh + Vl + 32768
                        *reinterpret_cast<uint16_t*>(Bl + (16 * m2 + 8 * hv + gq) * BL_STRIDE + col) = (uint16_t)__byte_perm(vs[m2][2 * hv], vs[m2][2 * hv + 1], 0x0062);
            }
        }
#undef A1
#undef A2
    }
    __syncwarp();
    // ---- steered BRIEF: lane = output byte. A rotated coordinate x (|x| < 19) rounds to nearest even as the low bits of x + 1.5 * 2^23,
    // like __float2int_rn, without a conversion.
    const float factorPI = (float)(3.14159265358979323846 / 180.0);
    float a, b;
    det_sincosf(__fmul_rn(angle, factorPI), &b, &a);
    const float RND = 12582912.0f;   // 0x1.8p23
    // sample (r, c) at Bl[(r + 18) * BL_STRIDE + c + 18]; with R, C the bit patterns of r + RND, c + RND the offset is R * BL_STRIDE + C + k0 (mod 2^32)
    const uint32_t k0 = (uint32_t)(18 * BL_STRIDE + 18) - (uint32_t)(BL_STRIDE + 1) * (uint32_t)__float_as_int(RND);
    uint32_t val = 0;
#pragma unroll
    for (int k = 0; k < 8; k++) {
        const float4 pt = __ldg(g_pat + k * 32 + lane);   // x0, y0, x1, y1
        const uint32_t r0 = __float_as_uint(__fadd_rn(__fadd_rn(__fmul_rn(pt.x, b), __fmul_rn(pt.y, a)), RND)),
                       c0 = __float_as_uint(__fadd_rn(__fsub_rn(__fmul_rn(pt.x, a), __fmul_rn(pt.y, b)), RND));
        const uint32_t r1 = __float_as_uint(__fadd_rn(__fadd_rn(__fmul_rn(pt.z, b), __fmul_rn(pt.w, a)), RND)),
                       c1 = __float_as_uint(__fadd_rn(__fsub_rn(__fmul_rn(pt.z, a), __fmul_rn(pt.w, b)), RND));
        const int t0 = Bl[(int)(r0 * BL_STRIDE + c0 + k0)], t1 = Bl[(int)(r1 * BL_STRIDE + c1 + k0)];
        val |= (uint32_t)(t0 < t1) << k;
    }
    A.desc[((size_t)frame * A.kpCap + outIdx) * 32 + lane] = (uint8_t)val;
    if (lane == 0) kpo->angle = angle;
}

}  // namespace cslam

// =================================================================================================== host side
using namespace cslam;

enum { KIND_WARP = 0, KIND_PYRAMID, KIND_FAST, KIND_DISTRIBUTE, KIND_DESCRIBE, KIND_COUNT, KIND_END = KernelTimer::END };
static const char* kKindNames[KIND_COUNT] = {"k_warp", "k_pyramid", "k_fast", "k_distribute", "k_describe"};

// A host batch as the caller passed it: input frames (fisheye frames, or canvases of pitch inPitch) and the output buffers; pin*: the
// buffer is page-locked, so the copy engines use it directly
struct HostBatch {
    const uint8_t* in; int inPitch; bool fromWarp;
    cslam_keypoint* kps; uint8_t* desc; int32_t* n;
    bool pinIn, pinK, pinD, pinN;
};
// Where a host batch is staged and which error flag its kernels write. The device buffers hold the whole batch (frame f at f times the
// per-frame size); the page-locked ones stand in for the caller's pageable buffers. up / down: the streams of the fisheye uploads and of the
// downloads, ordered to each chunk's kernels by evUp / evRun; nullptr: the chunk's own stream (the synchronous entry points).
struct HostStage {
    uint8_t* dfe; cslam_keypoint* dk; uint8_t* dd; int32_t* dn;
    uint8_t* hIn; cslam_keypoint* hKps; uint8_t* hDesc; int32_t* hN;
    int* errFlag;
    cudaStream_t up, down; cudaEvent_t evUp, evRun;
};
// A pending ticket of cslam_frontend_submit (ticket 0: the slot is free). Its device staging, error flag and events are made the first time
// the slot is used, each page-locked staging buffer the first time the slot meets a pageable buffer of its kind. Not from the arena: the next
// entry point's reset() would hand the pieces out again while the ticket's copies still use them.
struct PendingSlot {
    int64_t ticket = 0;
    HostStage s = {};
    int* errHost = nullptr;          // page-locked copy of *s.errFlag, written after the ticket's last kernel
    cudaEvent_t evDone = nullptr;    // after the ticket's downloads and its error flag's copy
    HostBatch b = {}; int batch = 0;
};

// error flag: set by k_fast, k_distribute and k_describe when a fixed-capacity buffer overflows. arena: device staging of the synchronous
// host entry points (fisheye frames, key points, descriptors, counts).
struct cslam_frontend : cslam::Handle {
    cslam_cam_params cam;
    cslam_orb_params orb;
    int W = 0, H = 0, CW = 0, CH = 0, maxBatch = 0, kpCap = 0, M = 0;   // M: quadtree node capacity = kept-list capacity per (frame, level)
    DevLevels L;                     // host copy of the device-pointer table (passed by value to kernels)
    std::vector<float> scale, invScale, sigma2, invSigma2; std::vector<int> perLevel; int umax[16];
    std::vector<float> map1, map2;   // host float maps (3H x 3W), kept for cslam_frontend_get_maps
    const WarpTile* d_wtiles = nullptr; const uint32_t* d_went = nullptr;   // k_warp tiles and their WT_W x WT_H entry tables
    int nWarpTiles = 0, warpSlot = 0;   // warpSlot: staged source box bytes per frame (largest staged box, rounded to 16)
    uint8_t* d_mask = nullptr; int maskPitch = 0;
    uint32_t* d_candCount = nullptr; // maxBatch x nlevels
    uint32_t* d_kept = nullptr; uint32_t* d_keptCount = nullptr;
    uint8_t* h_pin_in = nullptr; cslam_keypoint* h_pin_kps = nullptr; uint8_t* h_pin_desc = nullptr; int32_t* h_pin_n = nullptr;
    // kernel lanes 0..MAX_LANES-1, forked from the handle's stream and joined back by every call; then the copy lanes of submitted
    // batches, which are never joined: UP_LANE (uploads, wait for nothing) and DOWN_LANE (downloads, wait for their chunk's kernels)
    static const int MAX_LANES = 4, UP_LANE = MAX_LANES, DOWN_LANE = MAX_LANES + 1, ALL_LANES = MAX_LANES + 2;
    cudaStream_t lane[ALL_LANES] = {}; cudaEvent_t evLane[MAX_LANES] = {}; cudaEvent_t evFork = nullptr;
    static constexpr int DEV_LANES = 2;     // lanes used by cslam_frontend_run_dev
    static constexpr int HOST_CHUNKS = 8;   // most chunks a host-buffer batch is cut into
    PendingSlot slot[CSLAM_FRONTEND_MAX_PENDING];
    int64_t lastTicket = 0;
    KernelTimer timer;           // optional per-kernel timing (cslam_frontend_set_timing); a timed batch runs as one lane and one chunk
    bool cornersDirty = false;   // level buffers hold a caller canvas pyramid (non-zero corner regions) from cslam_orb_extract
    int pyrWin[MAX_LEVELS] = {};   // k_pyramid instantiation (PYR_WIN or PYR_WIN_MAX) of each level >= 1
    ~cslam_frontend() {   // the kernel lanes are joined into the handle's stream, which destroy_handle has waited for; every lane is waited for too
        for (int i = 0; i < ALL_LANES; i++)
            if (lane[i]) { cudaStreamSynchronize(lane[i]); cudaStreamDestroy(lane[i]); }
        for (int i = 0; i < MAX_LANES; i++) if (evLane[i]) cudaEventDestroy(evLane[i]);
        for (PendingSlot& p : slot)
            for (cudaEvent_t e : {p.s.evUp, p.s.evRun, p.evDone}) if (e) cudaEventDestroy(e);
        if (evFork) cudaEventDestroy(evFork);
    }
};

static inline void mark(cslam_frontend* fe, cudaStream_t st, int kind) {
    if (kind != KIND_END) fe->launches++;
    fe->timer.record(st, kind);
}

static inline int cv_round_f(float v) { return (int)lrintf(v); }
static inline int cv_round_d(double v) { return (int)lrint(v); }

// CamModelGeneral::CubemapToFisheye (src/CamModelGeneral.cpp:265-290) + WorldToImg (include/CamModelGeneral.h:359-374):
// start-up code on the host, exactly where the reference runs it (System::CreateUndistortRectifyMap).
static void host_cubemap_to_fisheye(const cslam_cam_params& cp, double up, double vp, double& uf, double& vf) {
    float i = (float)up, j = (float)vp;
    uf = -1; vf = -1;
    const int face = face_of_pixel_f(i, j, cp.face_w, cp.face_h);
    if (face < 0) return;
    const double fx = cp.face_w / 2.0, fy = cp.face_h / 2.0;
    i = i - static_cast<int>(i / cp.face_w) * cp.face_w;
    j = j - static_cast<int>(j / cp.face_h) * cp.face_h;
    const double lz = 1.0, lx = (i - fx) * lz / fx, ly = (j - fy) * lz / fy;
    double X, Y, Z;
    switch (face) {
        case FACE_FRONT: X = lx; Y = ly; Z = lz; break;
        case FACE_LEFT: X = -lz; Y = ly; Z = lx; break;
        case FACE_RIGHT: X = lz; Y = ly; Z = -lx; break;
        case FACE_LOWER: X = lx; Y = lz; Z = -ly; break;
        default: X = lx; Y = -lz; Z = ly; break;
    }
    double norm = std::sqrt(X * X + Y * Y);
    if (norm == 0.0) norm = 1e-14;
    const double theta = std::atan(-Z / norm);
    double rho = 0.0;
    for (int k = 11; k >= 0; k--) rho = rho * theta + cp.invpoly[k];
    const double uu = X / norm * rho, vv = Y / norm * rho;
    uf = uu * cp.c + vv * cp.d + cp.u0;
    vf = uu * cp.e + vv + cp.v0;
    if (uf < 0 || uf >= cp.Iw || vf < 0 || vf >= cp.Ih) { uf = -1; vf = -1; }
}

template <class T>
static int dev_upload(cslam_frontend* fe, const T** p, const std::vector<T>& v) {
    T* q = nullptr;
    int rc = dev_alloc(fe->owned, &q, v.size(), false);
    if (rc) return rc;
    CSLAM_CUDA(cudaMemcpy(q, v.data(), v.size() * sizeof(T), cudaMemcpyHostToDevice));
    *p = q;
    return 0;
}

static void build_resize_tables(int sn, int dn, std::vector<uint16_t>& ofs, std::vector<uint32_t>& ab) {
    ofs.resize(dn); ab.resize(dn);
    const double scale = (double)sn / dn;
    for (int d = 0; d < dn; d++) {
        float f = (float)((d + 0.5) * scale - 0.5);
        int s = (int)std::floor(f);
        f -= s;
        if (s < 0) { s = 0; f = 0; }
        if (s >= sn - 1) { s = sn - 1; f = 0; }
        const int a0 = cv_round_f((1.f - f) * 2048.f), a1 = cv_round_f(f * 2048.f);
        ofs[d] = (uint16_t)s; ab[d] = (uint32_t)a0 | ((uint32_t)a1 << 16);
    }
}
struct ResizeTables { std::vector<uint16_t> xo, yo; std::vector<uint32_t> xa, ya; };   // level l-1 -> l, both axes

// k_pyramid's row-block descriptors (PYR_RY dst rows each, `win` words) from the vertical resize tables; returns the window rows the
// widest block needs, or 0 if two dst rows of a block share a top tap (impossible for a downscale)
static int build_pyr_rows(const std::vector<uint16_t>& yo, const std::vector<uint32_t>& ya, int win, std::vector<uint32_t>& rd) {
    const int dh = (int)yo.size(), nb = cdiv(dh, PYR_RY);
    rd.assign((size_t)nb * win, 0u);
    int need = 0;
    for (int b = 0; b < nb; b++) {
        const int y0 = b * PYR_RY, y1 = std::min(y0 + PYR_RY, dh), src0 = yo[y0];
        const int nwin = yo[y1 - 1] - src0 + 2;   // the last dst row's bottom tap is window row nwin - 1
        need = std::max(need, nwin);
        if (nwin > win) continue;
        uint32_t* r = &rd[(size_t)b * win];
        r[0] = (uint32_t)src0 | ((uint32_t)nwin << 16);
        for (int y = y0; y < y1; y++) {
            if (y > y0 && yo[y] <= yo[y - 1]) return 0;
            r[yo[y] - src0 + 1] = ya[y];
        }
    }
    return need;
}

// Static pixel classes of the warp path, fixed by the geometry alone. K_0: Z = the canvas corner tiles (never written by k_warp, zeroed at
// allocation, so 0); C = face pixels whose quantised map is (0,0) (outside the image circle: k_warp writes S(0,0), one constant per frame);
// live = the rest. K_l(x,y): Z if all four resize taps of (x,y) are in Z_{l-1}; C if all four are in C_{l-1} and both tap-weight pairs sum to
// 2048 (k_pyramid then returns the constant itself: (((b0 128c) >> 16) + ((b1 128c) >> 16) + 2) >> 2 = c); live otherwise.
// From them: k_pyramid pieces inside Z_l (pskip); and, per k_fast CTA tile, the phase-A work items holding a pixel whose 7x7 window is not
// all Z or all C (live / liveOff). Every other pixel's ring and centre are equal, so its arc score is 0 at any threshold and for any frame.
// A tile without live items has no corner: its skip byte is set and its CTA exits before loading the tile.
static int build_static_classes(cslam_frontend* fe, const std::vector<ResizeTables>& rt) {
    enum : uint8_t { K_LIVE = 0, K_Z = 1, K_C = 2 };
    int rc;
    std::vector<uint8_t> K((size_t)fe->CW * fe->CH), Kn;
    for (int y = 0; y < fe->CH; y++)
        for (int x = 0; x < fe->CW; x++) {
            const size_t i = (size_t)y * fe->CW + x;
            const bool corner = x / fe->W != 1 && y / fe->H != 1;
            K[i] = corner ? K_Z : (cv_round_f(fe->map1[i] * 32.f) == 0 && cv_round_f(fe->map2[i] * 32.f) == 0) ? K_C : K_LIVE;
        }
    for (int l = 0; l < fe->L.nlevels; l++) {
        const LevelGeom& g = fe->L.g[l];
        const int w = g.w, h = g.h;
        if (l > 0) {
            const LevelGeom& sg = fe->L.g[l - 1];
            const ResizeTables& r = rt[l];
            Kn.assign((size_t)w * h, K_LIVE);
            for (int y = 0; y < h; y++) {
                const int y0 = r.yo[y], y1 = std::min(y0 + 1, sg.h - 1);
                const bool unitY = (r.ya[y] & 0xffff) + (r.ya[y] >> 16) == 2048;
                for (int x = 0; x < w; x++) {
                    const int x0 = r.xo[x], x1 = std::min(x0 + 1, sg.w - 1);
                    const uint8_t k = K[(size_t)y0 * sg.w + x0];
                    if (k == K_LIVE || K[(size_t)y0 * sg.w + x1] != k || K[(size_t)y1 * sg.w + x0] != k || K[(size_t)y1 * sg.w + x1] != k) continue;
                    if (k == K_Z || (unitY && (r.xa[x] & 0xffff) + (r.xa[x] >> 16) == 2048)) Kn[(size_t)y * w + x] = k;
                }
            }
            K.swap(Kn);
            const int px = cdiv(w, PYR_WX), py = cdiv(h, PYR_RY);
            std::vector<uint8_t> ps((size_t)px * py, 1);
            for (int y = 0; y < h; y++)
                for (int x = 0; x < w; x++)
                    if (K[(size_t)y * w + x] != K_Z) ps[(size_t)(y / PYR_RY) * px + x / PYR_WX] = 0;
            if ((rc = dev_upload(fe, &fe->L.pskip[l], ps))) return rc;
        }
        // U(x,y) = k if the 7x7 window centred on (x,y) is all class k (separably: rows of 7, then columns of 7 such rows), else K_LIVE
        std::vector<uint8_t> Hr((size_t)w * h, K_LIVE), U((size_t)w * h, K_LIVE);
        for (int y = 0; y < h; y++)
            for (int x = 3; x < w - 3; x++) {
                const uint8_t* r = &K[(size_t)y * w + x];
                bool same = true;
                for (int d = -3; d <= 3 && same; d++) same = r[d] == r[0];
                if (same) Hr[(size_t)y * w + x] = r[0];
            }
        for (int y = 3; y < h - 3; y++)
            for (int x = 0; x < w; x++) {
                const uint8_t k = Hr[(size_t)y * w + x];
                bool same = k != K_LIVE;
                for (int d = -3; d <= 3 && same; d++) same = Hr[(size_t)(y + d) * w + x] == k;
                if (same) U[(size_t)y * w + x] = k;
            }
        // work items in k_fast's order and geometry (tile rows iniY.., tile columns from a0 = tx0 & ~15, item = tile word wi of detection row y)
        const int gx = cdiv(g.nColsEff, CG), gy = g.nRowsEff;
        std::vector<FastTileX> tx(gx);
        for (int cxg = 0; cxg < gx; cxg++) tx[cxg] = fast_tile_x(g, cxg);
        std::vector<uint8_t> sk((size_t)gx * gy);
        std::vector<uint32_t> off((size_t)gx * gy + 1);
        std::vector<uint16_t> items;
        for (int cy = 0; cy < gy; cy++)
            for (int cxg = 0; cxg < gx; cxg++) {
                const size_t t = (size_t)cy * gx + cxg;
                off[t] = (uint32_t)items.size();
                const int iniY = g.minB + cy * g.hCell, maxY = std::min(iniY + g.hCell + 6, g.maxBY);
                const int a0 = tx[cxg].a0, nx = tx[cxg].nx, ny = maxY - iniY - 6, xoff = tx[cxg].xoff, w0 = tx[cxg].w0, w1 = tx[cxg].w1;
                for (int y = 0; y < ny; y++)
                    for (int wi = w0; wi < w1; wi++) {
                        bool any = false;
                        for (int j = 0; j < 4; j++) {
                            const int x = 4 * wi + j - xoff;   // detection x; the kernel masks the lanes outside [0, nx)
                            if (x >= 0 && x < nx && U[(size_t)(iniY + 3 + y) * w + a0 + 4 * wi + j] == K_LIVE) any = true;
                        }
                        if (any) items.push_back((uint16_t)(y << 6 | (wi - w0)));
                    }
                sk[t] = items.size() == off[t];
            }
        off[(size_t)gx * gy] = (uint32_t)items.size();
        for (size_t t = 0; t < (size_t)gx * gy; t++) fe->L.g[l].liveCap = std::max(fe->L.g[l].liveCap, (int)(off[t + 1] - off[t]));
        while (items.size() & 7) items.push_back(0);   // k_fast stages the lists in 16-byte pieces
        if ((rc = dev_upload(fe, &fe->L.skip[l], sk)) || (rc = dev_upload(fe, &fe->L.live[l], items)) || (rc = dev_upload(fe, &fe->L.liveOff[l], off))) return rc;
    }
    return 0;
}

// k_fast's per-tile-column table of one level (FastCols): the same for every frame, cell row and image, caller canvases included
static std::vector<FastCols> build_fast_cols(const LevelGeom& g) {
    std::vector<FastCols> cols(cdiv(g.nColsEff, CG));
    std::memset(cols.data(), 0, cols.size() * sizeof(FastCols));
    for (size_t cx = 0; cx < cols.size(); cx++) {
        const FastTileX t = fast_tile_x(g, (int)cx);
        FastCols& c = cols[cx];
        if (t.nx <= 0) continue;   // k_fast exits before reading the table
        c.mgItems = fdiv_magic(t.w1 - t.w0); c.mgZero = fdiv_magic(t.q1 - t.q0);
        for (int wi = 0; wi < FAST_SW / 2; wi++)
            for (int j = 0; j < 4; j++) {
                const int x = 4 * wi + j - t.xoff;   // detection x of tile column 4*wi + j
                if (x < 0 || x >= t.nx) continue;
                const int cell = x / g.wCell, xl = x - cell * g.wCell;
                const uint32_t lane = 0xffffu << (16 * (j & 1));
                FastItem& it = c.item[wi];
                it.valid[j >> 1] |= lane;
                if (xl != 0) it.left[j >> 1] |= lane;
                if (xl != g.wCell - 1 && x != t.nx - 1) it.right[j >> 1] |= lane;
                it.cells |= (uint32_t)cell << (2 * j);
                it.cellMask |= 1u << cell;
            }
    }
    return cols;
}

extern "C" int cslam_frontend_create(cslam_frontend** out, int device, const cslam_cam_params* cam, const cslam_orb_params* orb,
                                     const uint8_t* mask, int mask_pitch, int max_batch) {
    if (!out || !cam || !orb || !mask || max_batch <= 0) { set_error("cslam_frontend_create: null/invalid argument"); return CSLAM_E_BADARG; }
    if (cam->face_w != cam->face_h || cam->face_w <= 0) { set_error("cube faces must be square (got %dx%d)", cam->face_w, cam->face_h); return CSLAM_E_BADARG; }
    if (3 * cam->face_w > 4095 || cam->Iw * 32 > 65535 || cam->Ih * 32 > 65535) { set_error("image too large for the packed coordinate formats"); return CSLAM_E_BADARG; }
    if (orb->nlevels < 1 || orb->nlevels > MAX_LEVELS || orb->nfeatures < 1 || orb->scale_factor <= 1.f || orb->scale_factor > 2.f) { set_error("bad ORB parameters (need 1 < scaleFactor <= 2)"); return CSLAM_E_BADARG; }
    cslam_frontend* fe = new cslam_frontend;
    fe->cam = *cam; fe->orb = *orb; fe->maxBatch = max_batch;
    fe->W = cam->face_w; fe->H = cam->face_h; fe->CW = 3 * fe->W; fe->CH = 3 * fe->H;
    const int nl = orb->nlevels;
    fe->kpCap = orb->nfeatures + 3 * nl;
    auto fail = [&](int code) { destroy_handle(fe); return code; };
    // the host entry points' device staging: the arena's first chunk holds a max_batch call
    const size_t B = max_batch, fb = (size_t)cam->Iw * cam->Ih;
    auto piece = [](size_t bytes) { return (bytes + 255) & ~(size_t)255; };   // DevArena::take's rounding
    int rc = fe->open(device, piece(B * fb) + piece(B * fe->kpCap * sizeof(cslam_keypoint)) + piece(B * fe->kpCap * 32) + piece(B * sizeof(int32_t)), true);
    if (rc) return fail(rc);
    // ---- ORBextractor::ORBextractor (src/ORBExtractor.cpp:381-442): scale tables, per-level quotas, umax
    fe->scale.resize(nl); fe->invScale.resize(nl); fe->sigma2.resize(nl); fe->invSigma2.resize(nl); fe->perLevel.resize(nl);
    fe->scale[0] = 1.f; fe->sigma2[0] = 1.f;
    for (int i = 1; i < nl; i++) { fe->scale[i] = fe->scale[i - 1] * orb->scale_factor; fe->sigma2[i] = fe->scale[i] * fe->scale[i]; }
    for (int i = 0; i < nl; i++) { fe->invScale[i] = 1.0f / fe->scale[i]; fe->invSigma2[i] = 1.0f / fe->sigma2[i]; }
    {
        const float factor = 1.0f / orb->scale_factor;
        float nDesired = orb->nfeatures * (1 - factor) / (1 - (float)std::pow((double)factor, (double)nl));
        int sum = 0;
        for (int l = 0; l < nl - 1; l++) { fe->perLevel[l] = cv_round_f(nDesired); sum += fe->perLevel[l]; nDesired *= factor; }
        fe->perLevel[nl - 1] = std::max(orb->nfeatures - sum, 0);
        int v, v0, vmax = (int)std::floor(HALF_PATCH * std::sqrt(2.f) / 2 + 1), vmin = (int)std::ceil(HALF_PATCH * std::sqrt(2.f) / 2);
        const double hp2 = HALF_PATCH * HALF_PATCH;
        for (v = 0; v <= vmax; ++v) fe->umax[v] = cv_round_d(std::sqrt(hp2 - v * v));
        for (v = HALF_PATCH, v0 = 0; v >= vmin; --v) { while (fe->umax[v0] == fe->umax[v0 + 1]) ++v0; fe->umax[v] = v0; ++v0; }
    }
    for (int i = 0; i < cslam_frontend::ALL_LANES; i++)
        if (cudaStreamCreateWithFlags(&fe->lane[i], cudaStreamNonBlocking) != cudaSuccess ||
            (i < cslam_frontend::MAX_LANES && cudaEventCreateWithFlags(&fe->evLane[i], cudaEventDisableTiming) != cudaSuccess)) { set_error("lane stream creation failed"); return fail(CSLAM_E_CUDA); }
    if (cudaEventCreateWithFlags(&fe->evFork, cudaEventDisableTiming) != cudaSuccess) { set_error("event creation failed"); return fail(CSLAM_E_CUDA); }
    {
        uint32_t icRows[32] = {};
        for (int u = -HALF_PATCH; u <= HALF_PATCH; u++)
            for (int v = 0; v <= HALF_PATCH; v++) if (std::abs(u) <= fe->umax[v]) icRows[HALF_PATCH + u] |= 1u << v;
        if (cudaMemcpyToSymbol(g_icRows, icRows, sizeof(icRows)) != cudaSuccess) { set_error("cudaMemcpyToSymbol failed"); return fail(CSLAM_E_CUDA); }
    }
    {
        static const signed char hostPattern[1024] = {
#include "brief_pattern.inc"
        };
        float4 pat[8 * 32];
        for (int ln = 0; ln < 32; ln++)
            for (int k = 0; k < 8; k++) {
                const signed char* q = hostPattern + ln * 32 + 4 * k;
                pat[k * 32 + ln] = make_float4(q[0], q[1], q[2], q[3]);
            }
        if (cudaMemcpyToSymbol(g_pat, pat, sizeof(pat)) != cudaSuccess) { set_error("cudaMemcpyToSymbol failed"); return fail(CSLAM_E_CUDA); }
    }
    // ---- level geometry (ComputePyramid :930-936, ComputeKeyPointsOctTree :747-761)
    std::memset(&fe->L, 0, sizeof(fe->L));
    fe->L.nlevels = nl;
    int maxQuota = 0;
    std::vector<ResizeTables> rt(nl);   // entry 0 unused
    for (int l = 0; l < nl; l++) {
        LevelGeom& g = fe->L.g[l];
        g.w = cv_round_f((float)fe->CW * fe->invScale[l]); g.h = cv_round_f((float)fe->CH * fe->invScale[l]);
        g.pitch = round_up(g.w, 128);
        g.minB = EDGE_THRESHOLD - 3; g.maxBX = g.w - EDGE_THRESHOLD + 3; g.maxBY = g.h - EDGE_THRESHOLD + 3;
        const float width = (float)(g.maxBX - g.minB), height = (float)(g.maxBY - g.minB);
        const int nCols = (int)(width / 30.f), nRows = (int)(height / 30.f);
        if (nCols < 1 || nRows < 1) { set_error("pyramid level %d (%dx%d) is too small for the 30-px FAST grid", l, g.w, g.h); return fail(CSLAM_E_BADARG); }
        g.wCell = (int)std::ceil(width / nCols); g.hCell = (int)std::ceil(height / nRows);
        if (g.wCell > CELL_MAX || g.hCell > CELL_MAX) { set_error("FAST cell %dx%d exceeds the supported %d px", g.wCell, g.hCell, CELL_MAX); return fail(CSLAM_E_BADARG); }
        g.nColsEff = 0; g.nRowsEff = 0;
        for (int j = 0; j < nCols; j++) if (!((float)(g.minB + j * g.wCell) >= g.maxBX - 6)) g.nColsEff = j + 1;
        for (int i = 0; i < nRows; i++) if (!((float)(g.minB + i * g.hCell) >= g.maxBY - 3)) g.nRowsEff = i + 1;
        g.quota = fe->perLevel[l]; maxQuota = std::max(maxQuota, g.quota);
        g.candCap = std::max(4096, g.nColsEff * g.nRowsEff * 32);
        g.scale = fe->scale[l]; g.sizeF = (float)(int)(PATCH_SIZE * fe->scale[l]);
        if ((rc = dev_alloc(fe->owned, &fe->L.img[l], (size_t)max_batch * g.pitch * g.h + 256, true))) return fail(rc);   // slack: word loads may run a few bytes past the last row; zeroed: the black corners are never written on the warp path
        if ((rc = dev_alloc(fe->owned, &fe->L.cand[l], (size_t)max_batch * g.candCap, false))) return fail(rc);
        if ((rc = dev_alloc(fe->owned, &fe->L.pnode[l], (size_t)max_batch * g.candCap, false))) return fail(rc);
        if ((rc = dev_upload(fe, &fe->L.fcols[l], build_fast_cols(g)))) return fail(rc);
        if (l > 0) {
            ResizeTables& r = rt[l];
            build_resize_tables(fe->L.g[l - 1].w, g.w, r.xo, r.xa); build_resize_tables(fe->L.g[l - 1].h, g.h, r.yo, r.ya);
            std::vector<uint32_t> rd;
            int need = build_pyr_rows(r.yo, r.ya, PYR_WIN, rd);
            fe->pyrWin[l] = PYR_WIN;
            if (need > PYR_WIN) { need = build_pyr_rows(r.yo, r.ya, PYR_WIN_MAX, rd); fe->pyrWin[l] = PYR_WIN_MAX; }
            if (need < 2 || need > PYR_WIN_MAX) { set_error("pyramid level %d: unsupported resize row window (%d rows)", l, need); return fail(CSLAM_E_BADARG); }
            const std::vector<uint4> rd4(reinterpret_cast<const uint4*>(rd.data()), reinterpret_cast<const uint4*>(rd.data() + rd.size()));
            if ((rc = dev_upload(fe, &fe->L.xofs[l], r.xo)) || (rc = dev_upload(fe, &fe->L.xab[l], r.xa)) || (rc = dev_upload(fe, &fe->L.prows[l], rd4))) return fail(rc);
        }
    }
    fe->M = round_up(std::max(maxQuota + 4, 16), 32);
    const int distSmem = dist_smem(fe->M).total;
    if (distSmem > 200 * 1024) { set_error("nfeatures too large for the shared-memory quadtree (%d B)", distSmem); return fail(CSLAM_E_BADARG); }
    if (cudaFuncSetAttribute(k_distribute, cudaFuncAttributeMaxDynamicSharedMemorySize, distSmem) != cudaSuccess) { set_error("cudaFuncSetAttribute failed"); return fail(CSLAM_E_CUDA); }
    {   // the largest k_fast layout any front end can launch: CELL_MAX cells, a live list covering every item of a tile
        LevelGeom gmax = {};
        gmax.wCell = gmax.hCell = CELL_MAX; gmax.liveCap = (FAST_SW / 2) * CELL_MAX;
        if (cudaFuncSetAttribute(k_fast, cudaFuncAttributeMaxDynamicSharedMemorySize, fast_smem(gmax).total) != cudaSuccess) { set_error("cudaFuncSetAttribute failed"); return fail(CSLAM_E_CUDA); }
    }
    // ---- System::CreateUndistortRectifyMap (src/System.cpp:301-324) on the host, then quantised like cv::remap does
    // (skipped when no fisheye geometry is given: extraction-only front end, e.g. the ORBextractor facade)
    if (cam->Iw > 0 && cam->Ih > 0) {
        const int CW = fe->CW, CH = fe->CH, W = fe->W;
        fe->map1.assign((size_t)CW * CH, 0.f); fe->map2.assign((size_t)CW * CH, 0.f);
        for (int y = 0; y < CH; y++)
            for (int x = 0; x < CW; x++) {
                double u, v;
                host_cubemap_to_fisheye(*cam, (double)x, (double)y, u, v);
                if (u < 0 || v < 0 || u >= cam->Iw || v >= cam->Ih) continue;
                fe->map1[(size_t)y * CW + x] = (float)u; fe->map2[(size_t)y * CW + x] = (float)v;
            }
        std::vector<uint32_t> q((size_t)5 * W * W);
        for (int f = 0; f < 5; f++)
            for (int y = 0; y < W; y++)
                for (int x = 0; x < W; x++) {
                    const size_t src = (size_t)(FACE_TILE_ROW[f] * W + y) * CW + FACE_TILE_COL[f] * W + x;
                    const int sx = cv_round_f(fe->map1[src] * 32.f), sy = cv_round_f(fe->map2[src] * 32.f);
                    q[((size_t)f * W + y) * W + x] = (uint32_t)sx | ((uint32_t)sy << 16);
                }
        // k_warp tiles: per tile the source box of all its taps (ix..ix+1, iy..iy+1 of every pixel whose map is not (0,0)) and the
        // per-pixel entries relative to it; a tile whose box exceeds WARP_BOX_MAX keeps the raw map and gathers from global memory
        std::vector<WarpTile> tiles;
        std::vector<uint32_t> ent;
        int slot = 0;
        for (int f = 0; f < 5; f++) {
            const int cx0 = FACE_TILE_COL[f] * W, cx1 = cx0 + W;
            for (int y0 = 0; y0 < W; y0 += WT_H)
                for (int xa = cx0 / WT_W * WT_W; xa < cx1; xa += WT_W) {
                    WarpTile t;
                    t.row0 = FACE_TILE_ROW[f] * W + y0; t.xa = xa; t.cx0 = cx0; t.cx1 = cx1; t.nr = std::min(WT_H, W - y0);
                    int minX = 1 << 30, minY = 1 << 30, maxX = -1, maxY = -1;
                    auto mapAt = [&](int r, int c) { return q[((size_t)f * W + y0 + r) * W + (xa + c - cx0)]; };
                    auto inFace = [&](int r, int c) { return r < t.nr && xa + c >= cx0 && xa + c < cx1; };
                    for (int r = 0; r < WT_H; r++)
                        for (int c = 0; c < WT_W; c++) {
                            if (!inFace(r, c)) continue;
                            const uint32_t m = mapAt(r, c);
                            if (m == 0) continue;
                            const int ix = (m & 0xffff) >> 5, iy = (m >> 16) >> 5;
                            minX = std::min(minX, ix); maxX = std::max(maxX, ix + 1); minY = std::min(minY, iy); maxY = std::max(maxY, iy + 1);
                        }
                    if (maxX < 0) { t.bx0 = t.by0 = 0; t.bw = t.bh = 0; }
                    else { t.bx0 = minX & ~3; t.by0 = minY; t.bw = round_up(maxX + 1 - t.bx0, 4); t.bh = maxY + 1 - minY; }
                    t.direct = t.bw * t.bh > WARP_BOX_MAX;
                    if (!t.direct) slot = std::max(slot, t.bw * t.bh);
                    for (int r = 0; r < WT_H; r++)
                        for (int c = 0; c < WT_W; c++) {
                            uint32_t e = 0;
                            if (inFace(r, c)) {
                                const uint32_t m = mapAt(r, c);
                                const int sx = m & 0xffff, sy = m >> 16;
                                if (t.direct) e = m;
                                else if (m == 0) e = WE_ORIGIN;
                                else e = (uint32_t)(((sy >> 5) - t.by0) * t.bw + (sx >> 5) - t.bx0) | ((uint32_t)(sx & 31) << 16) | ((uint32_t)(sy & 31) << 21);
                            }
                            ent.push_back(e);
                        }
                    tiles.push_back(t);
                }
        }
        fe->nWarpTiles = (int)tiles.size();
        fe->warpSlot = round_up(std::max(slot, 16), 16);
        const uint8_t* dt = nullptr;
        std::vector<uint8_t> tb(tiles.size() * sizeof(WarpTile));
        std::memcpy(tb.data(), tiles.data(), tb.size());
        if ((rc = dev_upload(fe, &dt, tb)) || (rc = dev_upload(fe, &fe->d_went, ent))) return fail(rc);
        fe->d_wtiles = reinterpret_cast<const WarpTile*>(dt);
        if (cudaFuncSetAttribute(k_warp, cudaFuncAttributeMaxDynamicSharedMemorySize, WARP_FPT * fe->warpSlot + 16) != cudaSuccess) { set_error("cudaFuncSetAttribute failed"); return fail(CSLAM_E_CUDA); }
        if ((rc = build_static_classes(fe, rt))) return fail(rc);
    }
    // ---- mask
    fe->maskPitch = round_up(fe->CW, 128);
    if ((rc = dev_alloc(fe->owned, &fe->d_mask, (size_t)fe->maskPitch * fe->CH, true))) return fail(rc);
    if (cudaMemcpy2D(fe->d_mask, fe->maskPitch, mask, mask_pitch, fe->CW, fe->CH, cudaMemcpyHostToDevice) != cudaSuccess) { set_error("mask upload failed"); return fail(CSLAM_E_CUDA); }
    // ---- batch buffers
    if ((rc = dev_alloc(fe->owned, &fe->d_candCount, B * nl, true)) || (rc = dev_alloc(fe->owned, &fe->d_kept, B * nl * fe->M, true)) ||
        (rc = dev_alloc(fe->owned, &fe->d_keptCount, B * nl, true)) || (rc = pinned_alloc(fe->pinned, &fe->h_pin_in, B * fb)) ||
        (rc = pinned_alloc(fe->pinned, &fe->h_pin_kps, B * fe->kpCap)) || (rc = pinned_alloc(fe->pinned, &fe->h_pin_desc, B * fe->kpCap * 32)) ||
        (rc = pinned_alloc(fe->pinned, &fe->h_pin_n, B))) return fail(rc);
    *out = fe;
    return CSLAM_OK;
}

extern "C" void cslam_frontend_destroy(cslam_frontend* fe) { destroy_handle(fe); }

extern "C" int cslam_frontend_set_timing(cslam_frontend* fe, int enable) {
    if (!fe) return CSLAM_E_BADARG;
    CSLAM_CUDA(cudaSetDevice(fe->device));
    return fe->timer.enable(enable != 0, 256);
}
extern "C" int cslam_frontend_get_timing(const cslam_frontend* fe, int kind, const char** name, double* ms, int64_t* count) {
    return fe ? fe->timer.get(kind, KIND_COUNT, kKindNames, name, ms, count) : CSLAM_E_BADARG;
}
extern "C" int cslam_frontend_kp_capacity(const cslam_frontend* fe) { return fe ? fe->kpCap : 0; }
extern "C" void* cslam_frontend_stream(const cslam_frontend* fe) { return fe ? (void*)fe->stream : nullptr; }
extern "C" int64_t cslam_frontend_launches(const cslam_frontend* fe) { return fe ? fe->launches : 0; }

static const char* kOverflowMessage = "front end: a fixed-capacity buffer overflowed on the device (candidates / nodes / keypoints)";

// the end of every synchronous call: waits for the handle's stream (every call's kernels and the synchronous calls' copies) and reports the
// handle's own flag, never a ticket's
static int sync_stream(cslam_frontend* fe) {
    const int rc = fe->sync(kOverflowMessage);
    fe->timer.collect();
    return rc;
}

// waits for all enqueued work, the pending tickets' copies included
extern "C" int cslam_frontend_sync(cslam_frontend* fe) {
    if (!fe) return CSLAM_E_BADARG;
    CSLAM_CUDA(cudaSetDevice(fe->device));
    CSLAM_CUDA(cudaStreamSynchronize(fe->lane[cslam_frontend::UP_LANE]));
    CSLAM_CUDA(cudaStreamSynchronize(fe->lane[cslam_frontend::DOWN_LANE]));
    return sync_stream(fe);
}

// Frame range [f0, f0+cnt) of the per-batch buffers, for one lane
static DevLevels shifted(const cslam_frontend* fe, int f0) {
    DevLevels L = fe->L;
    for (int l = 0; l < L.nlevels; l++) {
        const LevelGeom& g = L.g[l];
        L.img[l] += (size_t)f0 * g.pitch * g.h; L.cand[l] += (size_t)f0 * g.candCap; L.pnode[l] += (size_t)f0 * g.candCap;
    }
    return L;
}

static int launch_warp(cslam_frontend* fe, cudaStream_t st, const uint8_t* d_fisheye, int f0, int cnt) {
    if (!fe->d_wtiles) { set_error("this front end was created without fisheye geometry (Iw/Ih = 0): no warp"); return CSLAM_E_BADARG; }
    const size_t cframe = (size_t)fe->L.g[0].pitch * fe->CH;
    uint8_t* canvas = fe->L.img[0] + (size_t)f0 * cframe;
    const int Iw = fe->cam.Iw, Ih = fe->cam.Ih, pitch = fe->L.g[0].pitch;
    const int words = (Iw % 4 == 0 && ((uintptr_t)d_fisheye & 3) == 0) ? 1 : 0;   // 4-byte staging needs word-aligned source rows
    dim3 grid(fe->nWarpTiles, cdiv(cnt, WARP_FPT));
    const size_t smem = (size_t)WARP_FPT * fe->warpSlot + 16;
    mark(fe, st, KIND_WARP);
    k_warp<<<grid, 256, smem, st>>>(d_fisheye, Iw, Ih, fe->d_wtiles, fe->d_went, canvas, pitch, cframe, cnt, fe->warpSlot, words);
    CSLAM_CUDA(cudaGetLastError());
    return 0;
}

// errFlag: where k_fast, k_distribute and k_describe report an overflow (the handle's flag, or a pending ticket's)
static int launch_extract(cslam_frontend* fe, cudaStream_t st, int f0, int cnt, cslam_keypoint* d_kps, uint8_t* d_desc, int32_t* d_nout, bool useSkip,
                          int* errFlag) {
    const int nl = fe->L.nlevels;
    const DevLevels L = shifted(fe, f0);
    uint32_t* candCount = fe->d_candCount + (size_t)f0 * nl;
    CSLAM_CUDA(cudaMemsetAsync(candCount, 0, (size_t)cnt * nl * sizeof(uint32_t), st));
    for (int l = 1; l < nl; l++) {
        const LevelGeom& s = L.g[l - 1]; const LevelGeom& d = L.g[l];
        dim3 grid(cdiv(cdiv(d.w, 4), 128), cdiv(d.h, PYR_RY), cnt);
        mark(fe, st, KIND_PYRAMID);
        (fe->pyrWin[l] == PYR_WIN ? k_pyramid<PYR_WIN> : k_pyramid<PYR_WIN_MAX>)<<<grid, 128, 0, st>>>(
            L.img[l - 1], s.w, s.h, s.pitch, L.img[l], d.w, d.h, d.pitch, L.xofs[l], L.xab[l], L.prows[l], useSkip ? L.pskip[l] : nullptr);
    }
    for (int l = 0; l < nl; l++) {
        const LevelGeom& g = L.g[l];
        dim3 grid(cdiv(g.nColsEff, CG), cdiv(g.nRowsEff, FAST_R), cnt);
        mark(fe, st, KIND_FAST);
        k_fast<<<grid, 256, fast_smem(g).total, st>>>(L.img[l], g, fe->orb.ini_th_fast, fe->orb.min_th_fast, L.cand[l], candCount + l, nl, errFlag,
                                     L.fcols[l], useSkip ? L.skip[l] : nullptr, useSkip ? L.live[l] : nullptr, L.liveOff[l]);
    }
    CSLAM_CUDA(cudaGetLastError());
    DistributeArgs da;
    da.L = L; da.candCount = candCount; da.kept = fe->d_kept + (size_t)f0 * nl * fe->M; da.keptCount = fe->d_keptCount + (size_t)f0 * nl;
    da.mask = fe->d_mask; da.maskPitch = fe->maskPitch;
    da.imgW = fe->CW; da.imgH = fe->CH; da.faceW = fe->W; da.faceH = fe->H; da.M = fe->M; da.errFlag = errFlag;
    mark(fe, st, KIND_DISTRIBUTE);
    k_distribute<<<dim3(nl, cnt), DIST_THREADS, dist_smem(fe->M).total, st>>>(da);
    DescribeArgs ds;
    ds.L = L; ds.kept = da.kept; ds.keptCount = da.keptCount; ds.M = fe->M; ds.kps = d_kps; ds.desc = d_desc; ds.nOut = d_nout; ds.kpCap = fe->kpCap;
    ds.errFlag = errFlag;
    mark(fe, st, KIND_DESCRIBE);
    k_describe<<<dim3(cdiv(fe->kpCap, DESC_WARPS), cnt), DESC_WARPS * 32, 0, st>>>(ds);
    mark(fe, st, KIND_END);
    CSLAM_CUDA(cudaGetLastError());
    return 0;
}

// the arguments every batch entry point checks (`call` names it in the message); then selects the front end's device
static int check_batch(cslam_frontend* fe, const char* call, int batch, std::initializer_list<const void*> bufs) {
    if (!fe || batch <= 0 || batch > fe->maxBatch || std::count(bufs.begin(), bufs.end(), nullptr)) {
        set_error("%s: null buffer, or batch outside 1..%d", call, fe ? fe->maxBatch : 0);
        return CSLAM_E_BADARG;
    }
    CSLAM_CUDA(cudaSetDevice(fe->device));
    return 0;
}

static bool is_pinned(const void* p) {
    cudaPointerAttributes at;
    if (cudaPointerGetAttributes(&at, p) != cudaSuccess) { cudaGetLastError(); return false; }
    return at.type == cudaMemoryTypeHost;
}

static int join_lanes(cslam_frontend* fe, int nl) {
    for (int i = 0; i < nl; i++) { CSLAM_CUDA(cudaEventRecord(fe->evLane[i], fe->lane[i])); CSLAM_CUDA(cudaStreamWaitEvent(fe->stream, fe->evLane[i], 0)); }
    return 0;
}
// Lanes: chunk ck of `nchunks` contiguous frame ranges is enqueued by fn(stream, f0, cnt) on lane ck % nlanes. The lanes are forked from the
// main stream and joined back into it, also when fn fails; returns the first error. Chunks touch disjoint slices of every buffer, so the copy
// engines and the latency-bound k_distribute of one lane overlap with the ALU-bound kernels of the others.
template <class Fn>
static int enqueue(cslam_frontend* fe, int batch, int nlanes, int nchunks, Fn&& fn) {
    CSLAM_CUDA(cudaEventRecord(fe->evFork, fe->stream));
    for (int i = 0; i < nlanes; i++) CSLAM_CUDA(cudaStreamWaitEvent(fe->lane[i], fe->evFork, 0));
    int rc = 0;
    for (int ck = 0; ck < nchunks && !rc; ck++) {
        const int f0 = (int)((long long)batch * ck / nchunks), f1 = (int)((long long)batch * (ck + 1) / nchunks);
        if (f1 > f0) rc = fn(fe->lane[ck % nlanes], f0, f1 - f0);
    }
    const int jrc = join_lanes(fe, nlanes);
    return rc ? rc : jrc;
}
static int prepare_level0(cslam_frontend* fe, bool fromWarp) {
    // the warp never writes the 4 corner tiles; they must read as the reference's zeroed canvas. The warp path's k_pyramid does not
    // write the corner regions of levels >= 1 either (DevLevels::pskip), so after a caller canvas every level is cleared once.
    if (fromWarp && fe->cornersDirty) {
        for (int l = 0; l < fe->L.nlevels; l++)
            CSLAM_CUDA(cudaMemsetAsync(fe->L.img[l], 0, (size_t)fe->maxBatch * fe->L.g[l].pitch * fe->L.g[l].h, fe->stream));
        fe->cornersDirty = false;
    }
    if (!fromWarp) fe->cornersDirty = true;
    return 0;
}
static int lanes_for(const cslam_frontend* fe, int batch, int want) {
    if (fe->timer.on()) return 1;
    return std::max(1, std::min(std::min(want, cslam_frontend::MAX_LANES), batch));
}

// chunks of a host batch on `nlanes` lanes. The batch is cut into more chunks than there are lanes (chunk c runs on lane c % nlanes): the first
// upload - the only one nothing overlaps within the call - is then 1/8 of the batch instead of 1/4, and the copy engines stay busy behind the
// kernels of earlier chunks
static int host_chunks(const cslam_frontend* fe, int batch, int nlanes) {
    return fe->timer.on() ? 1 : std::max(nlanes, std::min(cslam_frontend::HOST_CHUNKS, std::max(1, batch / 8)));
}

// frames [f0, f0+cnt) of a host fisheye batch, through the page-locked hIn unless the caller's buffer is page-locked, to `dfe` on `st`
static int upload_fisheye(cslam_frontend* fe, cudaStream_t st, const uint8_t* in, bool pinIn, uint8_t* hIn, uint8_t* dfe, int f0, int cnt) {
    const size_t fb = (size_t)fe->cam.Iw * fe->cam.Ih, off = (size_t)f0 * fb;
    const uint8_t* src = in + off;
    if (!pinIn) { std::memcpy(hIn + off, src, (size_t)cnt * fb); src = hIn + off; }
    CSLAM_CUDA(cudaMemcpyAsync(dfe + off, src, (size_t)cnt * fb, cudaMemcpyHostToDevice, st));
    return 0;
}

extern "C" int cslam_warp(cslam_frontend* fe, const uint8_t* fisheye, int batch, uint8_t* canvas, int canvas_pitch) {
    int rc = check_batch(fe, "cslam_warp", batch, {fisheye, canvas});
    if (rc) return rc;
    fe->arena.reset();
    uint8_t* dfe = nullptr;
    if ((rc = prepare_level0(fe, true)) || (rc = fe->arena.take(&dfe, (size_t)batch * fe->cam.Iw * fe->cam.Ih))) return rc;
    rc = enqueue(fe, batch, 1, 1, [&](cudaStream_t st, int f0, int cnt) -> int {
        int rc = upload_fisheye(fe, st, fisheye, is_pinned(fisheye), fe->h_pin_in, dfe, f0, cnt);
        if (rc || (rc = launch_warp(fe, st, dfe + (size_t)f0 * fe->cam.Iw * fe->cam.Ih, f0, cnt))) return rc;
        // the reference writes only the five face ROIs; corner tiles of the caller's canvas are left untouched
        const int W = fe->W, pitch = fe->L.g[0].pitch;
        for (int f = f0; f < f0 + cnt; f++)
            for (int t = 0; t < 5; t++) {
                const size_t row = (size_t)FACE_TILE_ROW[t] * W, col = (size_t)FACE_TILE_COL[t] * W;
                CSLAM_CUDA(cudaMemcpy2DAsync(canvas + (size_t)f * canvas_pitch * fe->CH + row * canvas_pitch + col, canvas_pitch,
                                             fe->L.img[0] + (size_t)f * pitch * fe->CH + row * pitch + col, pitch, W, W, cudaMemcpyDeviceToHost, st));
            }
        return 0;
    });
    if (rc) { cudaStreamSynchronize(fe->stream); return rc; }
    return sync_stream(fe);
}

static HostBatch host_batch(const uint8_t* in, int inPitch, bool fromWarp, cslam_keypoint* kps, uint8_t* desc, int32_t* n_out) {
    return HostBatch{in, inPitch, fromWarp, kps, desc, n_out, is_pinned(in), is_pinned(kps), is_pinned(desc), is_pinned(n_out)};
}

// One chunk, frames [f0, f0+cnt), of a host batch: upload, k_warp (or the caller's canvases straight into level 0), launch_extract, download.
// The one sequence of cslam_frontend_run, cslam_orb_extract and cslam_frontend_submit; caller buffers are used directly when they are
// page-locked. The kernels run on `st`, the copies on s.up / s.down when those are set.
static int host_chunk(cslam_frontend* fe, const HostBatch& b, const HostStage& s, cudaStream_t st, int f0, int cnt) {
    const size_t nk = (size_t)fe->kpCap;
    cudaStream_t up = s.up ? s.up : st, down = s.down ? s.down : st;
    int rc = 0;
    if (b.fromWarp) {
        if ((rc = upload_fisheye(fe, up, b.in, b.pinIn, s.hIn, s.dfe, f0, cnt))) return rc;
        if (up != st) { CSLAM_CUDA(cudaEventRecord(s.evUp, up)); CSLAM_CUDA(cudaStreamWaitEvent(st, s.evUp, 0)); }
        if ((rc = launch_warp(fe, st, s.dfe + (size_t)f0 * fe->cam.Iw * fe->cam.Ih, f0, cnt))) return rc;
    } else {   // level 0 is shared by every call: it is written in the order of the kernels, on `st`
        const int pitch = fe->L.g[0].pitch;
        CSLAM_CUDA(cudaMemcpy2DAsync(fe->L.img[0] + (size_t)f0 * pitch * fe->CH, pitch, b.in + (size_t)f0 * b.inPitch * fe->CH, b.inPitch, fe->CW,
                                     (size_t)fe->CH * cnt, cudaMemcpyHostToDevice, st));
    }
    if ((rc = launch_extract(fe, st, f0, cnt, s.dk + (size_t)f0 * nk, s.dd + (size_t)f0 * nk * 32, s.dn + f0, b.fromWarp, s.errFlag))) return rc;
    if (down != st) { CSLAM_CUDA(cudaEventRecord(s.evRun, st)); CSLAM_CUDA(cudaStreamWaitEvent(down, s.evRun, 0)); }
    CSLAM_CUDA(cudaMemcpyAsync((b.pinK ? b.kps : s.hKps) + (size_t)f0 * nk, s.dk + (size_t)f0 * nk, (size_t)cnt * nk * sizeof(cslam_keypoint), cudaMemcpyDeviceToHost, down));
    CSLAM_CUDA(cudaMemcpyAsync((b.pinD ? b.desc : s.hDesc) + (size_t)f0 * nk * 32, s.dd + (size_t)f0 * nk * 32, (size_t)cnt * nk * 32, cudaMemcpyDeviceToHost, down));
    CSLAM_CUDA(cudaMemcpyAsync((b.pinN ? b.n : s.hN) + f0, s.dn + f0, (size_t)cnt * sizeof(int32_t), cudaMemcpyDeviceToHost, down));
    return 0;
}

// the pageable outputs of a finished host batch, out of their page-locked staging
static void copy_out(const cslam_frontend* fe, const HostBatch& b, const HostStage& s, int batch) {
    const size_t tot = (size_t)batch * fe->kpCap;
    if (!b.pinK) std::memcpy(b.kps, s.hKps, tot * sizeof(cslam_keypoint));
    if (!b.pinD) std::memcpy(b.desc, s.hDesc, tot * 32);
    if (!b.pinN) std::memcpy(b.n, s.hN, batch * sizeof(int32_t));
}

// the synchronous host entry points, staged through the arena and h_pin_*; the caller has reset the arena
static int run_host(cslam_frontend* fe, const HostBatch& b, int batch) {
    const size_t nk = (size_t)fe->kpCap;
    HostStage s = {};
    s.hIn = fe->h_pin_in; s.hKps = fe->h_pin_kps; s.hDesc = fe->h_pin_desc; s.hN = fe->h_pin_n; s.errFlag = fe->errFlag;
    int rc;
    if ((rc = prepare_level0(fe, b.fromWarp)) || (b.fromWarp && (rc = fe->arena.take(&s.dfe, (size_t)batch * fe->cam.Iw * fe->cam.Ih))) ||
        (rc = fe->arena.take(&s.dk, batch * nk)) || (rc = fe->arena.take(&s.dd, batch * nk * 32)) || (rc = fe->arena.take(&s.dn, (size_t)batch))) return rc;
    const int nlanes = lanes_for(fe, batch, cslam_frontend::MAX_LANES);
    rc = enqueue(fe, batch, nlanes, host_chunks(fe, batch, nlanes), [&](cudaStream_t st, int f0, int cnt) { return host_chunk(fe, b, s, st, f0, cnt); });
    if (rc) { cudaStreamSynchronize(fe->stream); return rc; }
    if ((rc = sync_stream(fe))) return rc;
    copy_out(fe, b, s, batch);
    return CSLAM_OK;
}

extern "C" int cslam_orb_extract(cslam_frontend* fe, const uint8_t* canvas, int canvas_pitch, int batch, cslam_keypoint* kps, uint8_t* desc, int32_t* n_out) {
    int rc = check_batch(fe, "cslam_orb_extract", batch, {canvas, kps, desc, n_out});
    if (rc) return rc;
    if (canvas_pitch < fe->CW) { set_error("cslam_orb_extract: canvas pitch %d is below the canvas width %d", canvas_pitch, fe->CW); return CSLAM_E_BADARG; }
    fe->arena.reset();
    return run_host(fe, host_batch(canvas, canvas_pitch, false, kps, desc, n_out), batch);
}

extern "C" int cslam_frontend_run(cslam_frontend* fe, const uint8_t* fisheye, int batch, cslam_keypoint* kps, uint8_t* desc, int32_t* n_out) {
    int rc = check_batch(fe, "cslam_frontend_run", batch, {fisheye, kps, desc, n_out});
    if (rc) return rc;
    fe->arena.reset();
    return run_host(fe, host_batch(fisheye, 0, true, kps, desc, n_out), batch);
}

// The staging of a pending slot for the buffers of `b`: device buffers, error flag and events on the slot's first use, each page-locked
// buffer the first time the slot meets a pageable buffer of its kind. Sized for max_batch, so a slot never grows.
static int slot_stage(cslam_frontend* fe, PendingSlot& p, const HostBatch& b) {
    HostStage& s = p.s;
    const size_t B = fe->maxBatch, nk = fe->kpCap, fb = (size_t)fe->cam.Iw * fe->cam.Ih;
    int rc = 0;
    if (!p.evDone) {   // made last: a first use that failed half-way starts again
        if ((rc = dev_alloc(fe->owned, &s.dfe, B * fb, false)) || (rc = dev_alloc(fe->owned, &s.dk, B * nk, false)) ||
            (rc = dev_alloc(fe->owned, &s.dd, B * nk * 32, false)) || (rc = dev_alloc(fe->owned, &s.dn, B, false)) ||
            (rc = dev_alloc(fe->owned, &s.errFlag, 1, false)) || (rc = pinned_alloc(fe->pinned, &p.errHost, 1))) return rc;
        s.up = fe->lane[cslam_frontend::UP_LANE]; s.down = fe->lane[cslam_frontend::DOWN_LANE];
        CSLAM_CUDA(cudaEventCreateWithFlags(&s.evUp, cudaEventDisableTiming));
        CSLAM_CUDA(cudaEventCreateWithFlags(&s.evRun, cudaEventDisableTiming));
        CSLAM_CUDA(cudaEventCreateWithFlags(&p.evDone, cudaEventDisableTiming));
    }
    if ((!b.pinIn && !s.hIn && (rc = pinned_alloc(fe->pinned, &s.hIn, B * fb))) || (!b.pinK && !s.hKps && (rc = pinned_alloc(fe->pinned, &s.hKps, B * nk))) ||
        (!b.pinD && !s.hDesc && (rc = pinned_alloc(fe->pinned, &s.hDesc, B * nk * 32))) || (!b.pinN && !s.hN && (rc = pinned_alloc(fe->pinned, &s.hN, B)))) return rc;
    return 0;
}

// Enqueues slot p's batch. Its kernels run on the kernel lanes, forked from the handle's stream and joined back: they follow every earlier
// call's kernels, which share the pyramid levels, candidate and kept lists and counters, and every later call's kernels follow them. The
// uploads (UP_LANE) wait for nothing: the slot's staging is free once its previous ticket was waited. The downloads (DOWN_LANE) wait for their
// chunk's kernels only, so the next call's kernels do not wait for them. The ticket's error flag is copied after its last kernel.
static int enqueue_ticket(cslam_frontend* fe, PendingSlot& p, int batch) {
    const HostStage& s = p.s;
    CSLAM_CUDA(cudaMemsetAsync(s.errFlag, 0, sizeof(int), fe->stream));
    const int nlanes = lanes_for(fe, batch, cslam_frontend::MAX_LANES);
    const int rc = enqueue(fe, batch, nlanes, host_chunks(fe, batch, nlanes), [&](cudaStream_t st, int f0, int cnt) { return host_chunk(fe, p.b, s, st, f0, cnt); });
    if (rc) return rc;
    CSLAM_CUDA(cudaEventRecord(s.evRun, fe->stream));
    CSLAM_CUDA(cudaStreamWaitEvent(s.down, s.evRun, 0));
    CSLAM_CUDA(cudaMemcpyAsync(p.errHost, s.errFlag, sizeof(int), cudaMemcpyDeviceToHost, s.down));
    CSLAM_CUDA(cudaEventRecord(p.evDone, s.down));
    return 0;
}

extern "C" int cslam_frontend_submit(cslam_frontend* fe, const uint8_t* fisheye, int batch, cslam_keypoint* kps, uint8_t* desc, int32_t* n_out,
                                     int64_t* ticket) {
    int rc = check_batch(fe, "cslam_frontend_submit", batch, {fisheye, kps, desc, n_out, ticket});
    if (rc) return rc;
    if (!fe->d_wtiles) { set_error("cslam_frontend_submit: this front end was created without fisheye geometry (Iw/Ih = 0): no warp"); return CSLAM_E_BADARG; }
    PendingSlot* p = nullptr;
    for (PendingSlot& q : fe->slot) if (!q.ticket) { p = &q; break; }
    if (!p) { set_error("cslam_frontend_submit: %d tickets are pending; wait for one first", CSLAM_FRONTEND_MAX_PENDING); return CSLAM_E_BADARG; }
    p->b = host_batch(fisheye, 0, true, kps, desc, n_out); p->batch = batch;
    if ((rc = slot_stage(fe, *p, p->b))) return rc;
    if ((rc = prepare_level0(fe, true)) || (rc = enqueue_ticket(fe, *p, batch))) {
        cudaStreamSynchronize(fe->stream); cudaStreamSynchronize(p->s.up); cudaStreamSynchronize(p->s.down);
        return rc;
    }
    p->ticket = *ticket = ++fe->lastTicket;
    return CSLAM_OK;
}

extern "C" int cslam_frontend_wait(cslam_frontend* fe, int64_t ticket) {
    PendingSlot* p = nullptr;
    if (fe && ticket > 0)
        for (PendingSlot& q : fe->slot) if (q.ticket == ticket) p = &q;
    if (!p) { set_error("cslam_frontend_wait: ticket %lld is not pending", (long long)ticket); return CSLAM_E_BADARG; }
    p->ticket = 0;   // waited, whatever the outcome
    CSLAM_CUDA(cudaSetDevice(fe->device));
    CSLAM_CUDA(cudaEventSynchronize(p->evDone));
    if (fe->timer.on()) {   // the timer's events are on the kernel lanes, joined into the handle's stream
        CSLAM_CUDA(cudaStreamSynchronize(fe->stream));
        fe->timer.collect();
    }
    if (*p->errHost) { set_error("%s", kOverflowMessage); return *p->errHost; }
    copy_out(fe, p->b, p->s, p->batch);
    return CSLAM_OK;
}

// returns without synchronising, so it takes nothing from the arena
extern "C" int cslam_frontend_run_dev(cslam_frontend* fe, const uint8_t* fisheye_dev, int batch, cslam_keypoint* kps_dev, uint8_t* desc_dev, int32_t* n_out_dev) {
    int rc = check_batch(fe, "cslam_frontend_run_dev", batch, {fisheye_dev, kps_dev, desc_dev, n_out_dev});
    if (rc || (rc = prepare_level0(fe, true))) return rc;
    const int nlanes = lanes_for(fe, batch, cslam_frontend::DEV_LANES);
    const size_t nk = (size_t)fe->kpCap, fsz = (size_t)fe->cam.Iw * fe->cam.Ih;
    return enqueue(fe, batch, nlanes, nlanes, [&](cudaStream_t st, int f0, int cnt) -> int {
        const int rc = launch_warp(fe, st, fisheye_dev + (size_t)f0 * fsz, f0, cnt);
        return rc ? rc : launch_extract(fe, st, f0, cnt, kps_dev + (size_t)f0 * nk, desc_dev + (size_t)f0 * nk * 32, n_out_dev + f0, true, fe->errFlag);
    });
}

extern "C" int cslam_frontend_level_size(const cslam_frontend* fe, int level, int* w, int* h) {
    if (!fe || level < 0 || level >= fe->L.nlevels) return CSLAM_E_BADARG;
    *w = fe->L.g[level].w; *h = fe->L.g[level].h;
    return CSLAM_OK;
}
extern "C" int cslam_frontend_get_level(cslam_frontend* fe, int frame, int level, uint8_t* out) {
    if (!fe || level < 0 || level >= fe->L.nlevels || frame < 0 || frame >= fe->maxBatch || !out) return CSLAM_E_BADARG;
    const LevelGeom& g = fe->L.g[level];
    CSLAM_CUDA(cudaSetDevice(fe->device));
    CSLAM_CUDA(cudaStreamSynchronize(fe->stream));
    CSLAM_CUDA(cudaMemcpy2D(out, g.w, fe->L.img[level] + (size_t)frame * g.pitch * g.h, g.pitch, g.w, g.h, cudaMemcpyDeviceToHost));
    return CSLAM_OK;
}
extern "C" int cslam_frontend_get_candidates(cslam_frontend* fe, int frame, int level, int32_t* xyr, int cap, int* n) {
    if (!fe || level < 0 || level >= fe->L.nlevels || frame < 0 || frame >= fe->maxBatch || !xyr || !n) return CSLAM_E_BADARG;
    const LevelGeom& g = fe->L.g[level];
    CSLAM_CUDA(cudaSetDevice(fe->device));
    CSLAM_CUDA(cudaStreamSynchronize(fe->stream));
    uint32_t cnt = 0;
    CSLAM_CUDA(cudaMemcpy(&cnt, fe->d_candCount + (size_t)frame * fe->L.nlevels + level, 4, cudaMemcpyDeviceToHost));
    const int m = (int)std::min<uint32_t>(cnt, (uint32_t)g.candCap);
    std::vector<uint32_t> tmp(m);
    if (m) CSLAM_CUDA(cudaMemcpy(tmp.data(), fe->L.cand[level] + (size_t)frame * g.candCap, (size_t)m * 4, cudaMemcpyDeviceToHost));
    for (int i = 0; i < m && i < cap; i++) { xyr[3 * i] = tmp[i] & 0xfff; xyr[3 * i + 1] = (tmp[i] >> 12) & 0xfff; xyr[3 * i + 2] = tmp[i] >> 24; }
    *n = m;
    return CSLAM_OK;
}
extern "C" int cslam_frontend_get_maps(const cslam_frontend* fe, float* map1, float* map2) {
    if (!fe || !map1 || !map2) return CSLAM_E_BADARG;
    std::memcpy(map1, fe->map1.data(), fe->map1.size() * 4); std::memcpy(map2, fe->map2.data(), fe->map2.size() * 4);
    return CSLAM_OK;
}
extern "C" int cslam_frontend_tables(const cslam_frontend* fe, float* scale, float* inv_scale, float* sigma2, float* inv_sigma2, int32_t* per, int32_t* umax16) {
    if (!fe) return CSLAM_E_BADARG;
    for (int i = 0; i < fe->L.nlevels; i++) { scale[i] = fe->scale[i]; inv_scale[i] = fe->invScale[i]; sigma2[i] = fe->sigma2[i]; inv_sigma2[i] = fe->invSigma2[i]; per[i] = fe->perLevel[i]; }
    for (int i = 0; i < 16; i++) umax16[i] = fe->umax[i];
    return CSLAM_OK;
}

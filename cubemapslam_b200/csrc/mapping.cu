// LocalMapping feature operations of libcubemap_b200.so (SURVEY §8(f) rank 4), sm_90a: the Hamming / projection work either side of LocalBA.
//
// Reference (CPU):
//   MapPoint::ComputeDistinctiveDescriptors             src/MapPoint.cpp:243-303   (called per MapPoint from LocalMapping::ProcessNewKeyFrame / Fuse)
//   ORBMatcher::Fuse(KeyFrame*, vector<MapPoint*>&, th) src/ORBMatcher.cpp:1126-1240 (LocalMapping::SearchInNeighbors)
//   ORBMatcher::SearchForTriangulation                  src/ORBMatcher.cpp:971-1124 + CheckDistEpipolarLine :388-407 + CamModelGeneral::GetVectorSigma
//                                                       src/CamModelGeneral.cpp:307-335 (LocalMapping::CreateNewMapPoints)
//
// k_distinctive      one CTA per MapPoint: thread i owns observation i; its median distance to the others is the k-th order statistic found by a
//                    9-step bisection on the distance value (distances are integers in [0, 256]; no N x N matrix, no sort); first least median wins.
// k_fuse_search      one warp per MapPoint: projection into the key frame, the GetFeaturesInArea window (cube_geom.cuh) walked in the
//                    reference's order, level / chi2 gates, Hamming; the winner is the FIRST least distance in that order (the loop uses <).
//                    MapPoints are independent here: the order-dependent part of Fuse (Replace / AddObservation) stays on the host objects.
// k_triangulation    one CTA per key-frame pair: KF2's FeatureVector is rebuilt by an in-CTA bitonic sort of (node, index); one thread per KF1
//                    feature scans its node's KF2 features in list order with the reference's `<=` update rule, epipole and epipolar-line tests
//                    in the reference's float arithmetic (no FMA contraction); rotation histogram + three maxima per pair.
// The ORB-matching rules (Hamming distance, rotation bin, three maxima, bitonic sort, FeatureVector lookup) are orb_match.cuh's.
#include <cstring>
#include <vector>
#include "area_table.cuh"
#include "common.cuh"
#include "cube_geom.cuh"
#include "orb_match.cuh"

namespace cslam {

static const int MAP_NCELLS = 5 * GRID_G * GRID_G;

// ------------------------------------------------------------------------------------------------- ComputeDistinctiveDescriptors
static const int DD_THREADS = 128;
static const int DD_SMEM_N = 1024;   // observation descriptors staged in shared memory up to this count, read from global beyond it
__global__ void __launch_bounds__(DD_THREADS) k_distinctive(const uint8_t* __restrict__ desc, const int32_t* __restrict__ offset, int32_t* __restrict__ best) {
    __shared__ uint4 sd[2 * DD_SMEM_N];
    __shared__ unsigned long long red[DD_THREADS / 32];
    const int p = blockIdx.x, tid = threadIdx.x;
    const int beg = offset[p], N = offset[p + 1] - beg;
    if (N <= 0) { if (tid == 0) best[p] = -1; return; }
    const uint4* D = reinterpret_cast<const uint4*>(desc) + 2 * (size_t)beg;
    const bool staged = N <= DD_SMEM_N;
    if (staged) { for (int i = tid; i < 2 * N; i += DD_THREADS) sd[i] = __ldg(D + i); }
    __syncthreads();
    const int k = (int)(0.5 * (N - 1));   // vDists[0.5*(N-1)]
    unsigned long long mine = ~0ull;
    for (int i = tid; i < N; i += DD_THREADS) {
        const uint4 a0 = staged ? sd[2 * i] : __ldg(D + 2 * i), a1 = staged ? sd[2 * i + 1] : __ldg(D + 2 * i + 1);
        // smallest v with #{j : d(i, j) <= v} >= k + 1  (d(i, i) = 0 is part of the row, like Distances[i][i] = 0)
        int lo = 0, hi = 256;
        while (lo < hi) {
            const int mid = (lo + hi) >> 1;
            int cnt = 0;
            for (int j = 0; j < N; j++) {
                const uint4 b0 = staged ? sd[2 * j] : __ldg(D + 2 * j), b1 = staged ? sd[2 * j + 1] : __ldg(D + 2 * j + 1);
                cnt += hamming256(a0, a1, b0, b1) <= mid;
            }
            if (cnt >= k + 1) hi = mid; else lo = mid + 1;
        }
        const unsigned long long key = ((unsigned long long)lo << 32) | (unsigned)i;   // least median, then least index
        mine = min(mine, key);
    }
#pragma unroll
    for (int o = 16; o; o >>= 1) mine = min(mine, __shfl_xor_sync(0xffffffffu, mine, o));
    if ((tid & 31) == 0) red[tid >> 5] = mine;
    __syncthreads();
    if (tid == 0) {
        unsigned long long m = red[0];
        for (int w = 1; w < DD_THREADS / 32; w++) m = min(m, red[w]);
        best[p] = (int)(m & 0xffffffffu);
    }
}

// ------------------------------------------------------------------------------------------------- Fuse (search)
struct FuseArgs {
    const cslam_keypoint* kKF; const uint8_t* dKF; const uint16_t* cellStart; const uint16_t* cellIdx; int nKF;
    float Tcw[12];
    int nMP; const uint8_t* valid; const float* Xw; const int32_t* level; const uint8_t* dMP;
    float th, scale[16], invSigma2[16]; int W, H;
    int32_t* bestIdx; int32_t* bestDist;
};
__global__ void __launch_bounds__(256) k_fuse_search(FuseArgs A) {
    const int m = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (m >= A.nMP) return;
    unsigned best = 256u << 20;   // dist << 20 | position in the visiting order; starts at the reference's bestDist = 256, so a complement never wins
    int bestI = -1;
    if (A.valid[m]) {
        float xc[3];
        transform_cw(A.Tcw, A.Xw + 3 * (size_t)m, xc);   // `Rcw*p3Dw + tcw`
        float u, v;
        ray_to_cubemap(xc[0], xc[1], xc[2], A.W, A.H, u, v);   // the face result is not used: KeyFrame::IsInImage decides
        if (u >= 0.0f && u < (float)(3 * A.W) && v >= 0.0f && v < (float)(3 * A.H)) {
            const int lvl = A.level[m];
            const float radius = __fmul_rn(A.th, A.scale[lvl]);
            const float inv = __fdiv_rn((float)(3 * GRID_G), (float)(3 * A.W));
            AreaQuery aq;
            if (area_query(u, v, radius, A.W, A.H, inv, aq)) {
                const uint4* dM = reinterpret_cast<const uint4*>(A.dMP) + 2 * (size_t)m;
                const uint4 a0 = __ldg(dM), a1 = __ldg(dM + 1);
                const uint4* dC = reinterpret_cast<const uint4*>(A.dKF);
                int posBase = 0;
                for (int k = 0; k < 3; k++) {
                    AreaCells rc;
                    if (!area_cells(aq, k, rc)) break;
                    for (int cb = 0; cb < rc.n; cb += 32) {   // lanes = consecutive cells (ix major, iy minor) = the reference's cell order
                        const int ci = cb + lane;
                        int s = 0, e = 0;
                        if (ci < rc.n) { const int cell = rc.cell(ci); s = A.cellStart[cell]; e = A.cellStart[cell + 1]; }
                        // position of this lane's first entry in the visiting order = entries of the earlier cells
                        int pre = e - s;
#pragma unroll
                        for (int o = 1; o < 32; o <<= 1) { const int t = __shfl_up_sync(0xffffffffu, pre, o); if (lane >= o) pre += t; }
                        const int tot = __shfl_sync(0xffffffffu, pre, 31);
                        pre -= e - s;
                        for (int a = s; a < e; a++) {
                            const int idx = A.cellIdx[a];
                            const cslam_keypoint kp = A.kKF[idx];
                            if (!(fabsf(__fsub_rn(kp.x, u)) < radius && fabsf(__fsub_rn(kp.y, v)) < radius)) continue;   // AddCells
                            if (kp.octave < lvl - 1 || kp.octave > lvl) continue;
                            const float ex = __fsub_rn(u, kp.x), ey = __fsub_rn(v, kp.y);
                            const float e2 = __fadd_rn(__fmul_rn(ex, ex), __fmul_rn(ey, ey));
                            if ((double)__fmul_rn(e2, A.invSigma2[kp.octave]) > 5.99) continue;
                            const unsigned d = (unsigned)hamming256(a0, a1, __ldg(dC + 2 * idx), __ldg(dC + 2 * idx + 1));
                            const unsigned key = (d << 20) | (unsigned)min(posBase + pre + (a - s), 0xfffff);
                            if (key < best) { best = key; bestI = idx; }
                        }
                        posBase += tot;
                    }
                }
            }
        }
    }
    // first least distance in visiting order
    unsigned b = best;
#pragma unroll
    for (int o = 16; o; o >>= 1) b = min(b, __shfl_xor_sync(0xffffffffu, b, o));
    const unsigned who = __ballot_sync(0xffffffffu, best == b && bestI >= 0);
    const int idx = who ? __shfl_sync(0xffffffffu, bestI, __ffs(who) - 1) : -1;
    if (lane == 0) { A.bestIdx[m] = idx; A.bestDist[m] = idx >= 0 ? (int)(b >> 20) : 256; }
}

// ------------------------------------------------------------------------------------------------- SearchForTriangulation
static const int TRI_THREADS = 256;
// cv::norm(Vec3f) / cv::Vec3f::dot as OpenCV evaluates them (double accumulation + double sqrt / float accumulation)
__device__ __forceinline__ double norm3_d(float a, float b, float c) {
    return __dsqrt_rn(__dadd_rn(__dadd_rn(__dmul_rn((double)a, (double)a), __dmul_rn((double)b, (double)b)), __dmul_rn((double)c, (double)c)));
}
__device__ __forceinline__ float dot3_f(float a0, float a1, float a2, float b0, float b1, float b2) {
    float s = __fadd_rn(0.0f, __fmul_rn(a0, b0)); s = __fadd_rn(s, __fmul_rn(a1, b1)); s = __fadd_rn(s, __fmul_rn(a2, b2)); return s;
}
// CamModelGeneral::GetVectorSigma(key, normalRig, 1.0f)
__device__ float vector_sigma_d(float kx, float ky, float nx, float ny, float nz, int W, int H) {
    const double fx = W / 2.0, cx = W / 2.0, cy = H / 2.0;
    float c0, c1;   // normalCam(0), normalCam(1)  (cvtRigToFaces<float>)
    switch (face_of_pixel_f(kx, ky, W, H)) {
        case FACE_FRONT: c0 = nx; c1 = ny; break;
        case FACE_LEFT: c0 = nz; c1 = ny; break;
        case FACE_RIGHT: c0 = -nz; c1 = ny; break;
        case FACE_LOWER: c0 = nx; c1 = -nz; break;
        case FACE_UPPER: c0 = nx; c1 = nz; break;
        default: c0 = 0; c1 = 0; break;
    }
    const int i = (int)floorf(__fdiv_rn(kx, (float)W)), j = (int)floorf(__fdiv_rn(ky, (float)H));
    const float u = __fsub_rn(kx, (float)(i * W)), v = __fsub_rn(ky, (float)(j * H));
    const float op0 = (float)__dsub_rn((double)u, cx), op1 = (float)__dsub_rn((double)v, cy);
    // epipolar = (c1, -c0, 0), vertical = (c0, c1, 0)
    float OO1 = (float)__ddiv_rn((double)dot3_f(op0, op1, 0.0f, c1, -c0, 0.0f), norm3_d(c1, -c0, 0.0f)); if (OO1 < 0) OO1 = -OO1;
    const float CO1 = (float)__dsqrt_rn(__dadd_rn((double)__fmul_rn(OO1, OO1), __dmul_rn(fx, fx)));
    float PO1 = (float)__ddiv_rn((double)dot3_f(op0, op1, 0.0f, c0, c1, 0.0f), norm3_d(c0, c1, 0.0f)); if (PO1 < 0) PO1 = -PO1;
    const float tan1 = __fdiv_rn(PO1, CO1);
    const float tan2 = __fdiv_rn(__fadd_rn(PO1, 1.0f), CO1);
    const float tan3 = __fdiv_rn(__fsub_rn(tan2, tan1), __fadd_rn(1.0f, __fmul_rn(tan1, tan2)));
    return __fdiv_rn(1.0f, __fsqrt_rn(__fadd_rn(__fdiv_rn(1.0f, __fmul_rn(tan3, tan3)), 1.0f)));
}
struct TriArgs {
    // KF1 (one per pair, stride n1Stride) and KF2 likewise
    const cslam_keypoint* k1; const uint8_t* d1; const float* rays1; const uint8_t* hasMP1; const int32_t* node1; const int32_t* n1; int s1;
    const cslam_keypoint* k2; const uint8_t* d2; const float* rays2; const uint8_t* hasMP2; const int32_t* node2; const int32_t* n2; int s2;
    const float* Ow1; const float* Tcw2; const float* E12;   // per pair: 3, 16, 9 floats
    float scale[16], sigma2[16]; int W, H, checkOri, n2pow;
    int32_t* match12; int32_t* nmatches;
};
__global__ void __launch_bounds__(TRI_THREADS) k_triangulation(TriArgs A) {
    extern __shared__ uint32_t key2[];   // (node << 12 | index) of KF2, sorted
    __shared__ int hist[HISTO_BINS], keep[HISTO_BINS], total;
    __shared__ float E[9], epi[2];
    const int p = blockIdx.x, tid = threadIdx.x;
    const int n1 = min(A.n1[p], A.s1), n2 = min(A.n2[p], A.s2);
    const cslam_keypoint* K1 = A.k1 + (size_t)p * A.s1; const cslam_keypoint* K2 = A.k2 + (size_t)p * A.s2;
    const uint4* D1 = reinterpret_cast<const uint4*>(A.d1 + (size_t)p * A.s1 * 32); const uint4* D2 = reinterpret_cast<const uint4*>(A.d2 + (size_t)p * A.s2 * 32);
    const float* R1 = A.rays1 + (size_t)p * A.s1 * 3; const float* R2 = A.rays2 + (size_t)p * A.s2 * 3;
    const uint8_t* M1 = A.hasMP1 + (size_t)p * A.s1; const uint8_t* M2 = A.hasMP2 + (size_t)p * A.s2;
    const int32_t* N1 = A.node1 + (size_t)p * A.s1; const int32_t* N2 = A.node2 + (size_t)p * A.s2;
    int32_t* out = A.match12 + (size_t)p * A.s1;
    for (int i = tid; i < A.n2pow; i += TRI_THREADS) key2[i] = i < n2 ? ((uint32_t)N2[i] << 12) | (uint32_t)i : 0xffffffffu;
    if (tid < HISTO_BINS) hist[tid] = 0;
    if (tid < 9) E[tid] = A.E12[(size_t)p * 9 + tid];
    if (tid == 0) {
        total = 0;
        float c[3];
        transform_cw(A.Tcw2 + (size_t)p * 16, A.Ow1 + (size_t)p * 3, c);   // C2 = R2w*Cw + t2w
        float ex, ey;
        ray_to_cubemap(c[0], c[1], c[2], A.W, A.H, ex, ey);
        epi[0] = ex; epi[1] = ey;
    }
    __syncthreads();
    block_bitonic_sort(key2, A.n2pow);
    const float ex = epi[0], ey = epi[1];
    for (int i1 = tid; i1 < n1; i1 += TRI_THREADS) {
        int bestIdx2 = -1;
        if (!M1[i1] && N1[i1] >= 0) {   // node -1: in no FeatureVector node of KF1, never a query
            const int lo = node_lower_bound(key2, n2, (uint32_t)N1[i1]);
            const uint4 a0 = __ldg(D1 + 2 * i1), a1 = __ldg(D1 + 2 * i1 + 1);
            const float r0 = R1[3 * i1], r1 = R1[3 * i1 + 1], r2 = R1[3 * i1 + 2];
            // epipolar plane normal in the frame of KF2: [a b c] = ray1^T E12 (columns of E12)
            const float a = __fadd_rn(__fadd_rn(__fmul_rn(r0, E[0]), __fmul_rn(r1, E[3])), __fmul_rn(r2, E[6]));
            const float b = __fadd_rn(__fadd_rn(__fmul_rn(r0, E[1]), __fmul_rn(r1, E[4])), __fmul_rn(r2, E[7]));
            const float c = __fadd_rn(__fadd_rn(__fmul_rn(r0, E[2]), __fmul_rn(r1, E[5])), __fmul_rn(r2, E[8]));
            const float den = __fadd_rn(__fadd_rn(__fmul_rn(a, a), __fmul_rn(b, b)), __fmul_rn(c, c));
            int bestDist = 50;   // TH_LOW
            for (int q = lo; q < n2 && (key2[q] >> 12) == (uint32_t)N1[i1]; q++) {
                const int i2 = key2[q] & 0xfff;
                if (M2[i2]) continue;
                const int dist = hamming256(a0, a1, __ldg(D2 + 2 * i2), __ldg(D2 + 2 * i2 + 1));
                if (dist > 50 || dist > bestDist) continue;
                const cslam_keypoint kp2 = K2[i2];
                const float dx = __fsub_rn(ex, kp2.x), dy = __fsub_rn(ey, kp2.y);
                if (__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)) < __fmul_rn(100.0f, A.scale[kp2.octave])) continue;
                // CheckDistEpipolarLine
                if (den == 0) continue;
                const float num = __fadd_rn(__fadd_rn(__fmul_rn(a, R2[3 * i2]), __fmul_rn(b, R2[3 * i2 + 1])), __fmul_rn(c, R2[3 * i2 + 2]));
                const float sigma = vector_sigma_d(kp2.x, kp2.y, a, b, c, A.W, A.H);
                const float sigmaSquare = __fmul_rn(sigma, sigma);
                const float dsqr = __fdiv_rn(__fmul_rn(num, num), __fmul_rn(__fmul_rn(den, sigmaSquare), A.sigma2[kp2.octave]));
                if ((double)dsqr < 3.84) { bestIdx2 = i2; bestDist = dist; }
            }
        }
        out[i1] = bestIdx2;
        if (bestIdx2 >= 0) {
            atomicAdd(&total, 1);
            if (A.checkOri) atomicAdd(&hist[rot_bin(K1[i1].angle, K2[bestIdx2].angle)], 1);
        }
    }
    __syncthreads();
    if (A.checkOri) {
        if (tid == 0) three_maxima(hist, keep);
        __syncthreads();
        for (int i1 = tid; i1 < n1; i1 += TRI_THREADS) {
            const int m = out[i1];
            if (m < 0) continue;
            if (!keep[rot_bin(K1[i1].angle, K2[m].angle)]) { out[i1] = -1; atomicSub(&total, 1); }
        }
        __syncthreads();
    }
    if (tid == 0) A.nmatches[p] = total;
}

}  // namespace cslam

using namespace cslam;

struct cslam_mapper : cslam::Handle {};

extern "C" int cslam_mapper_create(cslam_mapper** out, int device) {
    if (!out) return CSLAM_E_BADARG;
    cslam_mapper* m = new cslam_mapper;
    int rc;
    if ((rc = m->open(device, (size_t)1 << 20, false)) || (rc = prepare_frame_index())) { destroy_handle(m); return rc; }
    cudaFuncSetAttribute(k_triangulation, cudaFuncAttributeMaxDynamicSharedMemorySize, 4096 * 4);
    *out = m;
    return CSLAM_OK;
}
extern "C" void cslam_mapper_destroy(cslam_mapper* m) { destroy_handle(m); }
extern "C" int64_t cslam_mapper_launches(const cslam_mapper* m) { return m ? m->launches : 0; }

extern "C" int cslam_distinctive_descriptors(cslam_mapper* m, const uint8_t* desc, const int32_t* offset, int n_points, int32_t* best) {
    if (!m || !offset || !best || n_points < 0 || (n_points && offset[n_points] > 0 && !desc)) { set_error("cslam_distinctive_descriptors: bad argument"); return CSLAM_E_BADARG; }
    if (n_points == 0) return CSLAM_OK;
    for (int p = 0; p < n_points; p++) if (offset[p + 1] < offset[p] || offset[p] < 0) { set_error("cslam_distinctive_descriptors: offsets must be non-decreasing"); return CSLAM_E_BADARG; }
    CSLAM_CUDA(cudaSetDevice(m->device));
    m->arena.reset();
    const size_t total = (size_t)offset[n_points];
    uint8_t* dD; const int32_t* dO; int32_t* dB; int rc;
    if ((rc = m->arena.take(&dD, total * 32 + 32)) || (rc = m->arena.upload(&dO, offset, (size_t)n_points + 1)) || (rc = m->arena.take(&dB, n_points))) return rc;
    if (total) CSLAM_CUDA(cudaMemcpyAsync(dD, desc, total * 32, cudaMemcpyHostToDevice, m->stream));
    k_distinctive<<<n_points, DD_THREADS, 0, m->stream>>>(dD, dO, dB); m->launches++;
    CSLAM_CUDA(cudaGetLastError());
    CSLAM_CUDA(cudaMemcpyAsync(best, dB, (size_t)n_points * 4, cudaMemcpyDeviceToHost, m->stream));
    return m->sync();
}

extern "C" int cslam_fuse_search(cslam_mapper* m, const cslam_keypoint* k_kf, const uint8_t* d_kf, int n_kf, const float* Tcw, int n_mp, const uint8_t* mp_valid, const float* mp_xw,
                                 const int32_t* mp_level, const uint8_t* mp_desc, float th, const float* scale_factors, const float* inv_level_sigma2, int nlevels, int face_w,
                                 int face_h, int32_t* best_idx, int32_t* best_dist) {
    if (!m || n_kf < 0 || n_kf > 4096 || n_mp < 0 || !Tcw || !scale_factors || !inv_level_sigma2 || nlevels <= 0 || nlevels > 16 || face_w <= 0 || face_w != face_h ||
        (n_kf && (!k_kf || !d_kf)) || (n_mp && (!mp_valid || !mp_xw || !mp_level || !mp_desc || !best_idx || !best_dist))) { set_error("cslam_fuse_search: bad argument (n_kf <= 4096, nlevels <= 16)"); return CSLAM_E_BADARG; }
    if (n_mp == 0) return CSLAM_OK;
    for (int i = 0; i < n_mp; i++) if (mp_valid[i] && (mp_level[i] < 0 || mp_level[i] >= nlevels)) { set_error("cslam_fuse_search: predicted level out of range"); return CSLAM_E_BADARG; }
    CSLAM_CUDA(cudaSetDevice(m->device));
    m->arena.reset();
    DevArena& a = m->arena;
    const int cap = std::max(n_kf, 1);
    const cslam_keypoint* dK; const uint8_t *dD, *dV, *dM; const int32_t *dN, *dL; const float* dX; uint16_t *dCS, *dCI; int32_t *dBI, *dBD; int rc;
    if ((rc = a.upload(&dK, k_kf, n_kf)) || (rc = a.upload(&dD, d_kf, (size_t)n_kf * 32)) || (rc = a.upload(&dN, &n_kf, 1)) || (rc = a.take(&dCS, MAP_NCELLS + 1)) ||
        (rc = a.take(&dCI, cap)) || (rc = a.upload(&dV, mp_valid, n_mp)) || (rc = a.upload(&dX, mp_xw, (size_t)n_mp * 3)) || (rc = a.upload(&dL, mp_level, n_mp)) ||
        (rc = a.upload(&dM, mp_desc, (size_t)n_mp * 32)) || (rc = a.take(&dBI, n_mp)) || (rc = a.take(&dBD, n_mp)) ||
        (rc = frame_index(m->stream, m->launches, dK, dN, 1, cap, face_w, face_h, nullptr, dCS, dCI))) return rc;
    FuseArgs A;
    A.kKF = dK; A.dKF = dD; A.cellStart = dCS; A.cellIdx = dCI; A.nKF = n_kf;
    for (int i = 0; i < 12; i++) A.Tcw[i] = Tcw[i];
    A.nMP = n_mp; A.valid = dV; A.Xw = dX; A.level = dL; A.dMP = dM; A.th = th; A.W = face_w; A.H = face_h;
    for (int i = 0; i < 16; i++) { A.scale[i] = scale_factors[std::min(i, nlevels - 1)]; A.invSigma2[i] = inv_level_sigma2[std::min(i, nlevels - 1)]; }
    A.bestIdx = dBI; A.bestDist = dBD;
    k_fuse_search<<<(n_mp + 7) / 8, 256, 0, m->stream>>>(A); m->launches++;
    CSLAM_CUDA(cudaGetLastError());
    CSLAM_CUDA(cudaMemcpyAsync(best_idx, dBI, (size_t)n_mp * 4, cudaMemcpyDeviceToHost, m->stream));
    CSLAM_CUDA(cudaMemcpyAsync(best_dist, dBD, (size_t)n_mp * 4, cudaMemcpyDeviceToHost, m->stream));
    return m->sync();
}

extern "C" int cslam_search_for_triangulation(cslam_mapper* m, int npairs, const cslam_keypoint* k1, const uint8_t* d1, const float* rays1, const uint8_t* has_mp1,
                                              const int32_t* node1, const int32_t* n1, int stride1, const cslam_keypoint* k2, const uint8_t* d2, const float* rays2,
                                              const uint8_t* has_mp2, const int32_t* node2, const int32_t* n2, int stride2, const float* Ow1, const float* Tcw2, const float* E12,
                                              const float* scale_factors, const float* level_sigma2, int nlevels, int face_w, int face_h, int check_orientation,
                                              int32_t* match12, int32_t* nmatches) {
    if (!m || npairs < 0 || stride1 <= 0 || stride2 <= 0 || stride1 > 4096 || stride2 > 4096 || !scale_factors || !level_sigma2 || nlevels <= 0 || nlevels > 16 || face_w <= 0 ||
        face_w != face_h || (npairs && (!k1 || !d1 || !rays1 || !has_mp1 || !node1 || !n1 || !k2 || !d2 || !rays2 || !has_mp2 || !node2 || !n2 || !Ow1 || !Tcw2 || !E12 || !match12 || !nmatches))) {
        set_error("cslam_search_for_triangulation: bad argument (at most 4096 features per key frame)"); return CSLAM_E_BADARG;
    }
    if (npairs == 0) return CSLAM_OK;
    const size_t t1 = (size_t)npairs * stride1, t2 = (size_t)npairs * stride2;
    for (int p = 0; p < npairs; p++)   // only the rows the kernel reads: [p*stride, p*stride + min(n[p], stride))
        if (!node_ids_ok(node1 + (size_t)p * stride1, (size_t)std::max(0, std::min(n1[p], stride1))) ||
            !node_ids_ok(node2 + (size_t)p * stride2, (size_t)std::max(0, std::min(n2[p], stride2)))) {
            set_error("cslam_search_for_triangulation: node ids must be in [-1, 2^20 - 1) (pair %d)", p); return CSLAM_E_BADARG;
        }
    CSLAM_CUDA(cudaSetDevice(m->device));
    m->arena.reset();
    DevArena& a = m->arena;
    const cslam_keypoint *dK1, *dK2; const uint8_t *dD1, *dD2, *dM1, *dM2; const float *dR1, *dR2, *dO, *dT, *dE; const int32_t *dN1, *dN2, *dC1, *dC2; int32_t *dOut, *dNm; int rc;
    if ((rc = a.upload(&dK1, k1, t1)) || (rc = a.upload(&dD1, d1, t1 * 32)) || (rc = a.upload(&dR1, rays1, t1 * 3)) || (rc = a.upload(&dM1, has_mp1, t1)) || (rc = a.upload(&dN1, node1, t1)) ||
        (rc = a.upload(&dK2, k2, t2)) || (rc = a.upload(&dD2, d2, t2 * 32)) || (rc = a.upload(&dR2, rays2, t2 * 3)) || (rc = a.upload(&dM2, has_mp2, t2)) || (rc = a.upload(&dN2, node2, t2)) ||
        (rc = a.upload(&dC1, n1, npairs)) || (rc = a.upload(&dC2, n2, npairs)) || (rc = a.upload(&dO, Ow1, (size_t)npairs * 3)) || (rc = a.upload(&dT, Tcw2, (size_t)npairs * 16)) ||
        (rc = a.upload(&dE, E12, (size_t)npairs * 9)) || (rc = a.take(&dOut, t1)) || (rc = a.take(&dNm, npairs))) return rc;
    const cudaStream_t st = m->stream;
    TriArgs A;
    A.k1 = dK1; A.d1 = dD1; A.rays1 = dR1; A.hasMP1 = dM1; A.node1 = dN1; A.n1 = dC1; A.s1 = stride1;
    A.k2 = dK2; A.d2 = dD2; A.rays2 = dR2; A.hasMP2 = dM2; A.node2 = dN2; A.n2 = dC2; A.s2 = stride2;
    A.Ow1 = dO; A.Tcw2 = dT; A.E12 = dE; A.W = face_w; A.H = face_h; A.checkOri = check_orientation ? 1 : 0;
    for (int i = 0; i < 16; i++) { A.scale[i] = scale_factors[std::min(i, nlevels - 1)]; A.sigma2[i] = level_sigma2[std::min(i, nlevels - 1)]; }
    const int p2 = pow2_at_least(stride2);
    A.n2pow = p2; A.match12 = dOut; A.nmatches = dNm;
    k_triangulation<<<npairs, TRI_THREADS, (size_t)p2 * 4, st>>>(A); m->launches++;
    CSLAM_CUDA(cudaGetLastError());
    CSLAM_CUDA(cudaMemcpyAsync(match12, dOut, t1 * 4, cudaMemcpyDeviceToHost, st));
    CSLAM_CUDA(cudaMemcpyAsync(nmatches, dNm, (size_t)npairs * 4, cudaMemcpyDeviceToHost, st));
    return m->sync();
}

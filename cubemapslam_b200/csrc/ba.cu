// Optimizer::LocalBundleAdjustment of libcubemap_b200.so on sm_90a (PoseOptimization lives in pose_opt.cu).
//
// Reference (CPU, g2o): src/Optimizer.cpp:192-451; edge src/g2o_cubemap_vertices_edges.cpp:164-233; LM loop
// ThirdParty/g2o/g2o/core/optimization_algorithm_levenberg.cpp:61-189; Schur solve core/block_solver.hpp:354-486.
// The hypergraph is replaced by flat fp64 arrays; all arithmetic stays fp64 (the gate is 1e-5 relative on poses/points),
// including the reference's float32 round trip inside the projection (ba_math.cuh).
//
// Every accumulation is OUTPUT-STATIONARY (no floating-point atomics anywhere), hence bit-reproducible run to run:
//   k_ba_errors      per edge; chi2 by fixed-shape block sums + a last-block pass over the block partials
//   k_ba_lin_points  thread per landmark: Hll, bl in registers over the landmark's edges (sorted edge order), Hpl per edge
//   k_ba_lin_poses   CTA per free pose over its edge list: the 21+6 unique entries of (Hpp, bp)
//   k_ba_dinv        per landmark (Hll + lambda I)^-1 and Dinv*bl
//   k_ba_schur       CTA per pose pair (p1 <= p2) over the pair's precomputed co-observation list (edge a1 of p1, edge a2 of p2,
//                    same landmark, landmark order): S[p1,p2] = [p1==p2] Hpp - sum (B1 Dinv) B2^T, g[p1] = bp - sum B1 (Dinv bl)
//   k_ba_solve       one thread-block CLUSTER: blocked right-looking LDL^T of the n x n reduced camera system (n = 6 x free poses)
//                    with the right-hand side carried as an extra row; panel factorisation and trailing update spread over
//                    the cluster's SMs, panels exchanged through L2, cluster barriers between phases; no size cap
//   k_ba_backsub / k_ba_update / k_ba_scale / k_ba_restore   landmark back-substitution, oplus (with backup), gain-ratio scale
// Multi-GPU: landmarks (with their edges) are sharded l % nranks; every rank forms its partial reduced system [S | g | bpr] and the
// partials are summed either by one ncclAllReduce or by the one-shot NVLink kernel k_ba_xchg_reduce (peer pointers), in fixed rank order
// so that every rank solves bit-identical systems. The trial's scalars (chi2, scale) travel through k_ba_small_xchg. Payloads are
// double-buffered by epoch parity: a rank may run one exchange ahead of a peer that is still reading the previous one.
// LM control flow (accept/reject, lambda schedule, ORB-SLAM2's stop rule, pbStopFlag) stays on the host like in the reference.
#include <cooperative_groups.h>
#include <dlfcn.h>
#include <algorithm>
#include <cfloat>
#include <cstring>
#include <limits>
#include <vector>
#include "optimizer.cuh"

namespace cg = cooperative_groups;

namespace cslam {

// Ownership: landmark l belongs to rank l % nranks, and a rank's edge arrays hold only the edges of its own landmarks. Everything below is
// built from those edges, so another rank's landmark has an empty lmStart range and is inactive (ptAct == 0): kernels over edges, tuples
// or active landmarks need no owner test. Only k_ba_mask_points makes one, when the points of all ranks are summed.
struct BADev {
    int nKF, nMP, nE, nQ, nP, n;     // nQ non-fixed key frames (static per call), nP active free poses, n = 6 nP
    double f;                        // fx=fy=cx=cy
    Pose* pose; Pose* poseBak;
    double* X; double* Xbak;
    const int* eMP; const int* eKF;  // edges sorted by landmark (stable)
    const double* obs;               // 3 per edge: mx, my, w
    const int8_t* face;
    double* err; uint8_t* level;
    const int* poseIdx; const uint8_t* ptAct;   // per KF: compact active-free index or -1; per MP: 1 if it has an active edge
    const int* kfOfQ;                // per candidate pose q: KF index
    const int* lmStart;              // nMP+1, CSR over sorted edges
    const int* peStart; const int* peList;      // CSR of sorted edge ids by KF (ascending = landmark order)
    const long long* pairStart;      // nQ*nQ+1: co-observation list of (q1,q2), q1<=q2, row-major
    const int4* tuples;              // (a1, a2, landmark, -): the landmark rides along so that k_ba_schur has no tuple -> edge -> landmark load chain
    double *Hpp, *bp, *Hll, *bl, *Hpl, *Dinv, *db, *xp, *xl;
    double *S, *bpr;                 // the reduced camera system [S n*n | g n | bpr n] in BAHost::red; k_ba_solve reads g as row n of S
    double* scal;                    // [0] chi2, [1] scale, [2] max diag (as bits), [3] solve flag, [4] lambda of the current trial,
                                     // [5] 1 + largest key of a NaN diagonal, [6] 1 + largest key (as bits; 0 = none; see k_ba_diag_keys)
    double* part; unsigned* ticket;  // block partials + arrival counter of the deterministic grid reductions
    double* posePart; unsigned* poseTicket;   // k_ba_lin_poses: slice sums [nQ][POSE_SPLIT][27] + arrival counter per pose
    int robust; double delta, dsqr;
    int rank, nranks;                // k_ba_mask_points' owner test; k_ba_scale adds the replicated pose term on rank 0 only
};

static const int DINV_LD = 10;   // doubles per landmark in Dinv: 9 + 1 pad, so that every block is 16-byte aligned for the 128-bit loads of k_ba_schur

// Deterministic grid-wide sum: fixed-shape block sums, block partials in part[], the last block to arrive adds them in a fixed shape.
// Returns true in thread 0 of the last block, with the total in *total.
__device__ __forceinline__ bool grid_sum(double v, double* part, unsigned* ticket, double* sh, double* total) {
    __shared__ bool last;
    const double s = block_sum(v, sh);
    if (threadIdx.x == 0) {
        part[blockIdx.x] = s;
        __threadfence();
        last = atomicAdd(ticket, 1u) == gridDim.x - 1;
    }
    __syncthreads();
    if (!last) return false;
    __threadfence();
    double t = 0;
    for (unsigned i = threadIdx.x; i < gridDim.x; i += blockDim.x) t += __ldcg(part + i);
    t = block_sum(t, sh);
    if (threadIdx.x == 0) { *total = t; *ticket = 0; }
    return threadIdx.x == 0;
}

// computeActiveErrors + activeRobustChi2 (partial sum over the landmarks this rank owns) -> *out
__global__ void __launch_bounds__(256) k_ba_errors(BADev D, double* out) {
    __shared__ double sh[32];
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    double c = 0;
    if (e < D.nE && D.level[e] == 0) {
        double Xc[3], er[2];
        pose_map(D.pose[D.eKF[e]], D.X + 3 * D.eMP[e], Xc);
        edge_error(D.face[e], D.f, D.obs[3 * e], D.obs[3 * e + 1], Xc, er);
        D.err[2 * e] = er[0]; D.err[2 * e + 1] = er[1];
        const double chi = D.obs[3 * e + 2] * (er[0] * er[0] + er[1] * er[1]);
        if (D.robust) { double r0, r1; huber(D.delta, D.dsqr, chi, r0, r1); c = r0; } else c = chi;
    }
    double tot;
    if (grid_sum(c, D.part, D.ticket, sh, &tot)) *out = tot;
}

// Jacobians of one active edge (src/g2o_cubemap_vertices_edges.cpp:164-223) and its robust weight / weighted residual
struct EdgeLin { double Jx[2][3], Jp[2][6], w, r0, r1; };
__device__ __forceinline__ void linearize_edge(const BADev& D, int e, bool needPose, EdgeLin& L) {
    const int k = D.eKF[e], l = D.eMP[e];
    const Pose T = D.pose[k];
    double Xc[3], G[2][3], R[3][3];
    pose_map(T, D.X + 3 * l, Xc);
    edge_G(D.face[e], D.f, Xc, G);
    quat_to_matrix(T.q, R);
#pragma unroll
    for (int i = 0; i < 2; i++)
#pragma unroll
        for (int j = 0; j < 3; j++) L.Jx[i][j] = G[i][0] * R[0][j] + G[i][1] * R[1][j] + G[i][2] * R[2][j];
    if (needPose) edge_Jpose(G, Xc, L.Jp);
    const double e0 = D.err[2 * e], e1 = D.err[2 * e + 1], w0 = D.obs[3 * e + 2];
    double rho1 = 1.0;
    if (D.robust) { double r0; huber(D.delta, D.dsqr, w0 * (e0 * e0 + e1 * e1), r0, rho1); }
    L.w = rho1 * w0; L.r0 = -L.w * e0; L.r1 = -L.w * e1;
}

// buildSystem, landmark side (base_binary_edge.hpp:55-120): Hll, bl of one landmark accumulated in registers in edge order, Hpl per edge
static const int LM_LANES = 4;   // lanes that share one landmark in k_ba_lin_points / k_ba_backsub (edge a of the landmark goes to lane a % 4)
__global__ void __launch_bounds__(128) k_ba_lin_points(BADev D) {
    const int l = (blockIdx.x * blockDim.x + threadIdx.x) / LM_LANES, sub = threadIdx.x % LM_LANES;
    const bool in = l < D.nMP;
    double H[6] = {0, 0, 0, 0, 0, 0}, b[3] = {0, 0, 0};
    const int eBeg = in ? D.lmStart[l] : 0, eEnd = in ? D.lmStart[l + 1] : 0;
    for (int e = eBeg + sub; e < eEnd; e += LM_LANES) {
        double* B = D.Hpl + 18 * (size_t)e;
        const int pi = D.poseIdx[D.eKF[e]];
        if (D.level[e] != 0) {   // inactive edges contribute zero blocks (the co-observation lists are built once per call)
#pragma unroll
            for (int i = 0; i < 18; i++) B[i] = 0.0;
            continue;
        }
        EdgeLin L;
        linearize_edge(D, e, pi >= 0, L);
        int q = 0;
#pragma unroll
        for (int i = 0; i < 3; i++) {
            b[i] += L.Jx[0][i] * L.r0 + L.Jx[1][i] * L.r1;
#pragma unroll
            for (int j = i; j < 3; j++) H[q++] += L.w * (L.Jx[0][i] * L.Jx[0][j] + L.Jx[1][i] * L.Jx[1][j]);
        }
        if (pi >= 0) {
#pragma unroll
            for (int i = 0; i < 6; i++)
#pragma unroll
                for (int j = 0; j < 3; j++) B[3 * i + j] = L.w * (L.Jp[0][i] * L.Jx[0][j] + L.Jp[1][i] * L.Jx[1][j]);
        } else {
#pragma unroll
            for (int i = 0; i < 18; i++) B[i] = 0.0;
        }
    }
    // fixed-shape sum over the 4 lanes of the landmark (all 32 lanes of the warp take part)
#pragma unroll
    for (int i = 0; i < 6; i++) { H[i] += __shfl_xor_sync(0xffffffffu, H[i], 1); H[i] += __shfl_xor_sync(0xffffffffu, H[i], 2); }
#pragma unroll
    for (int i = 0; i < 3; i++) { b[i] += __shfl_xor_sync(0xffffffffu, b[i], 1); b[i] += __shfl_xor_sync(0xffffffffu, b[i], 2); }
    if (!in || sub) return;
    double* Hl = D.Hll + 9 * (size_t)l;
    Hl[0] = H[0]; Hl[1] = H[1]; Hl[2] = H[2]; Hl[3] = H[1]; Hl[4] = H[3]; Hl[5] = H[4]; Hl[6] = H[2]; Hl[7] = H[4]; Hl[8] = H[5];
    D.bl[3 * l] = b[0]; D.bl[3 * l + 1] = b[1]; D.bl[3 * l + 2] = b[2];
}

// buildSystem, pose side: POSE_SPLIT CTAs per candidate pose, each over a slice of the pose's edge list; 21 unique entries of Hpp + 6 of bp.
// Slice sums go to posePart[q][slice][27]; the last CTA of the pose to arrive adds the slices in slice order (fixed shape -> reproducible).
static const int POSE_SPLIT = 8;
__global__ void __launch_bounds__(256) k_ba_lin_poses(BADev D) {
    __shared__ double red[8][28];
    __shared__ bool last;
    const int qi = blockIdx.x, sl = blockIdx.y;
    const int k = D.kfOfQ[qi], p = D.poseIdx[k];
    if (p < 0) return;
    double acc[27];
#pragma unroll
    for (int i = 0; i < 27; i++) acc[i] = 0.0;
    for (int q = D.peStart[k] + sl * 256 + threadIdx.x; q < D.peStart[k + 1]; q += POSE_SPLIT * 256) {
        const int e = D.peList[q];
        if (D.level[e] != 0) continue;
        EdgeLin L;
        linearize_edge(D, e, true, L);
        int t = 0;
#pragma unroll
        for (int a = 0; a < 6; a++)
#pragma unroll
            for (int b = a; b < 6; b++) acc[t++] += L.w * (L.Jp[0][a] * L.Jp[0][b] + L.Jp[1][a] * L.Jp[1][b]);
#pragma unroll
        for (int a = 0; a < 6; a++) acc[21 + a] += L.Jp[0][a] * L.r0 + L.Jp[1][a] * L.r1;
    }
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
#pragma unroll
    for (int i = 0; i < 27; i++) {
        double v = acc[i];
#pragma unroll
        for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
        if (lane == 0) red[w][i] = v;
    }
    __syncthreads();
    double* mine = D.posePart + ((size_t)qi * POSE_SPLIT + sl) * 27;
    if (threadIdx.x < 27) {
        double s = 0;
        for (int ww = 0; ww < 8; ww++) s += red[ww][threadIdx.x];
        __stcg(mine + threadIdx.x, s);
    }
    __threadfence();
    __syncthreads();
    if (threadIdx.x == 0) last = atomicAdd(D.poseTicket + qi, 1u) == POSE_SPLIT - 1;
    __syncthreads();
    if (!last) return;
    __threadfence();
    if (threadIdx.x < 27) {
        double s = 0;
        for (int j = 0; j < POSE_SPLIT; j++) s += __ldcg(D.posePart + ((size_t)qi * POSE_SPLIT + j) * 27 + threadIdx.x);
        red[0][threadIdx.x] = s;
    }
    if (threadIdx.x == 0) D.poseTicket[qi] = 0;
    __syncthreads();
    if (threadIdx.x < 36) {
        const int a = threadIdx.x / 6, b = threadIdx.x % 6, lo = min(a, b), hi = max(a, b);
        D.Hpp[36 * p + threadIdx.x] = red[0][lo * 6 - lo * (lo - 1) / 2 + (hi - lo)];
    }
    if (threadIdx.x < 6) D.bp[6 * p + threadIdx.x] = red[0][21 + threadIdx.x];
}

// computeLambdaInit (optimization_algorithm_levenberg.cpp:166-178) runs m = std::max(fabs(H_jj), m) in index-mapping order: free poses, then
// active points, each vertex's diagonal in order. std::max returns its first argument when a comparison involves NaN, so a NaN diagonal sets
// m = NaN and the next diagonal replaces it: m is the maximum over the diagonals after the LAST NaN one, or NaN when that NaN is the last
// diagonal. Key of diagonal j: 6 p + j for free pose p, 6 nP + 3 l + j for active landmark l (the global index keeps the order) = the thread
// index i below. Two order-free steps, atomicMax of bit patterns of non-negative doubles: the largest NaN key and the largest key
// (k_ba_diag_keys), then the largest |H_jj| above the NaN key (k_ba_maxdiag).
__device__ __forceinline__ bool diag_of_key(const BADev& D, int i, double* d) {
    if (i < D.nP * 6) { *d = D.Hpp[36 * (i / 6) + 7 * (i % 6)]; return true; }
    const int j = i - D.nP * 6;
    if (j < D.nMP * 3 && D.ptAct[j / 3]) { *d = D.Hll[9 * (j / 3) + 4 * (j % 3)]; return true; }
    return false;
}
__device__ __forceinline__ void warp_max_to(double m, double* dst) {   // m >= 0
#pragma unroll
    for (int o = 16; o; o >>= 1) m = fmax(m, __shfl_xor_sync(0xffffffffu, m, o));
    if ((threadIdx.x & 31) == 0 && m > 0) atomicMax(reinterpret_cast<unsigned long long*>(dst), (unsigned long long)__double_as_longlong(m));
}
__global__ void __launch_bounds__(256) k_ba_diag_keys(BADev D) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    double d = 0;
    const bool act = diag_of_key(D, i, &d);
    warp_max_to(act && isnan(d) ? i + 1.0 : 0.0, &D.scal[5]);
    warp_max_to(act ? i + 1.0 : 0.0, &D.scal[6]);
}
__global__ void __launch_bounds__(256) k_ba_maxdiag(BADev D) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    double d = 0;
    const bool act = diag_of_key(D, i, &d) && i + 1.0 > D.scal[5];
    warp_max_to(act ? fabs(d) : 0.0, &D.scal[2]);
}

// Dinv = (Hll + lambda I)^-1 (3x3 cofactors, like Eigen), db = Dinv * bl
__global__ void __launch_bounds__(256) k_ba_dinv(BADev D) {
    const double lambda = D.scal[4];
    const int l = blockIdx.x * blockDim.x + threadIdx.x;
    if (l >= D.nMP) return;
    double* Dv = D.Dinv + DINV_LD * (size_t)l;
    if (!D.ptAct[l]) {
#pragma unroll
        for (int i = 0; i < 9; i++) Dv[i] = 0.0;
        D.db[3 * l] = 0; D.db[3 * l + 1] = 0; D.db[3 * l + 2] = 0;
        return;
    }
    double M[9];
#pragma unroll
    for (int i = 0; i < 9; i++) M[i] = D.Hll[9 * (size_t)l + i];
    M[0] += lambda; M[4] += lambda; M[8] += lambda;
    const double c00 = M[4] * M[8] - M[5] * M[7], c01 = M[5] * M[6] - M[3] * M[8], c02 = M[3] * M[7] - M[4] * M[6];
    const double id = 1.0 / (M[0] * c00 + M[1] * c01 + M[2] * c02);
    double Di[9];
    Di[0] = c00 * id; Di[1] = (M[2] * M[7] - M[1] * M[8]) * id; Di[2] = (M[1] * M[5] - M[2] * M[4]) * id;
    Di[3] = c01 * id; Di[4] = (M[0] * M[8] - M[2] * M[6]) * id; Di[5] = (M[2] * M[3] - M[0] * M[5]) * id;
    Di[6] = c02 * id; Di[7] = (M[1] * M[6] - M[0] * M[7]) * id; Di[8] = (M[0] * M[4] - M[1] * M[3]) * id;
#pragma unroll
    for (int i = 0; i < 9; i++) Dv[i] = Di[i];
#pragma unroll
    for (int i = 0; i < 3; i++) D.db[3 * l + i] = Di[3 * i] * D.bl[3 * l] + Di[3 * i + 1] * D.bl[3 * l + 1] + Di[3 * i + 2] * D.bl[3 * l + 2];
}

// ---- co-observation lists: for every pair of candidate poses q1 <= q2 the (a1, a2) edge pairs that share a landmark, in landmark order.
// Built once per cslam_local_ba call over ALL edges (edges that become inactive later carry zero Hpl blocks).
__device__ __forceinline__ int partner_edge(const BADev& D, int a1, int k2) {
    const int l = D.eMP[a1];
    for (int a2 = D.lmStart[l]; a2 < D.lmStart[l + 1]; a2++) if (D.eKF[a2] == k2) return a2;
    return -1;
}
__global__ void __launch_bounds__(128) k_ba_pairs_count(BADev D, long long* cnt) {
    __shared__ int wsum[4];
    const int q1 = blockIdx.y, q2 = blockIdx.x;
    if (q1 > q2) { if (threadIdx.x == 0) cnt[(size_t)q1 * D.nQ + q2] = 0; return; }
    const int k1 = D.kfOfQ[q1], k2 = D.kfOfQ[q2], beg = D.peStart[k1], end = D.peStart[k1 + 1];
    if (q1 == q2) { if (threadIdx.x == 0) cnt[(size_t)q1 * D.nQ + q2] = end - beg; return; }
    int c = 0;
    for (int q = beg + threadIdx.x; q < end; q += blockDim.x) c += partner_edge(D, D.peList[q], k2) >= 0;
#pragma unroll
    for (int o = 16; o; o >>= 1) c += __shfl_xor_sync(0xffffffffu, c, o);
    if ((threadIdx.x & 31) == 0) wsum[threadIdx.x >> 5] = c;
    __syncthreads();
    if (threadIdx.x == 0) cnt[(size_t)q1 * D.nQ + q2] = wsum[0] + wsum[1] + wsum[2] + wsum[3];
}
// exclusive scan of `m` counts (in place) + total, one CTA
__global__ void __launch_bounds__(1024) k_ba_pairs_scan(long long* v, int m) {
    __shared__ long long wtot[32];
    __shared__ long long carry;
    if (threadIdx.x == 0) carry = 0;
    __syncthreads();
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    for (int base = 0; base < m; base += 1024) {
        const int i = base + threadIdx.x;
        const long long x = i < m ? v[i] : 0;
        long long s = x;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) { const long long t = __shfl_up_sync(0xffffffffu, s, o); if (lane >= o) s += t; }
        if (lane == 31) wtot[w] = s;
        __syncthreads();
        if (w == 0) {
            long long t = wtot[lane];
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) { const long long u = __shfl_up_sync(0xffffffffu, t, o); if (lane >= o) t += u; }
            wtot[lane] = t;
        }
        __syncthreads();
        const long long excl = carry + (w ? wtot[w - 1] : 0) + s - x;
        if (i < m) v[i] = excl;
        __syncthreads();
        if (threadIdx.x == 1023) carry = excl + x;
        __syncthreads();
    }
    if (threadIdx.x == 0) v[m] = carry;
}
__global__ void __launch_bounds__(128) k_ba_pairs_fill(BADev D, const long long* start, int4* tuples) {
    __shared__ int wcnt[4];
    __shared__ long long base;
    const int q1 = blockIdx.y, q2 = blockIdx.x;
    if (q1 > q2) return;
    const int k1 = D.kfOfQ[q1], k2 = D.kfOfQ[q2], beg = D.peStart[k1], end = D.peStart[k1 + 1];
    int4* out = tuples + start[(size_t)q1 * D.nQ + q2];
    if (q1 == q2) { for (int q = beg + threadIdx.x; q < end; q += blockDim.x) { const int a = D.peList[q]; out[q - beg] = make_int4(a, a, D.eMP[a], 0); } return; }
    if (threadIdx.x == 0) base = 0;
    __syncthreads();
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    for (int q0 = beg; q0 < end; q0 += blockDim.x) {   // ordered compaction: output order = order of the pose's edge list = landmark order
        const int q = q0 + threadIdx.x;
        int a1 = -1, a2 = -1;
        if (q < end) { a1 = D.peList[q]; a2 = partner_edge(D, a1, k2); }
        const unsigned ball = __ballot_sync(0xffffffffu, a2 >= 0);
        if (lane == 0) wcnt[w] = __popc(ball);
        __syncthreads();
        int pre = 0;
        for (int ww = 0; ww < w; ww++) pre += wcnt[ww];
        if (a2 >= 0) out[base + pre + __popc(ball & ((1u << lane) - 1))] = make_int4(a1, a2, D.eMP[a1], 0);
        __syncthreads();
        if (threadIdx.x == 0) base += wcnt[0] + wcnt[1] + wcnt[2] + wcnt[3];
        __syncthreads();
    }
}

// Schur complement (block_solver.hpp:381-439), output-stationary: one CTA per pose pair accumulates its 6x6 block in registers over the
// pair's co-observation list, then a fixed-shape reduction. The diagonal pair also forms g = bp - sum B (Dinv bl) and bpr = bp.
// Two threads share a tuple (rows 0-2 / rows 3-5 of the 6x6 block): 18 + 3 accumulators per thread keep the kernel at a register count
// that lets the list loads of many tuples be in flight per SM (the kernel is L2-latency bound, the Hpl / Dinv blocks are L2 resident).
// The rank's partial system [S n*n | g n | bpr n] goes to `out`: the reduced system itself on one GPU, the rank's exchange payload otherwise.
static const int SCHUR_T = 256;
__global__ void __launch_bounds__(SCHUR_T) k_ba_schur(BADev D, double* out, int addLambda) {
    const double lambdaDiag = addLambda ? D.scal[4] : 0.0;
    __shared__ double red[SCHUR_T / 32][44];
    const int q1 = blockIdx.y, q2 = blockIdx.x;
    if (q1 > q2) return;
    const int p1 = D.poseIdx[D.kfOfQ[q1]], p2 = D.poseIdx[D.kfOfQ[q2]];
    if (p1 < 0 || p2 < 0) return;
    const bool diag = q1 == q2;
    const int h = threadIdx.x & 1;
    double acc[21];
#pragma unroll
    for (int i = 0; i < 21; i++) acc[i] = 0.0;
    const long long beg = D.pairStart[(size_t)q1 * D.nQ + q2], end = D.pairStart[(size_t)q1 * D.nQ + q2 + 1];
    long long t = beg + (threadIdx.x >> 1);
    int4 nxt = t < end ? D.tuples[t] : make_int4(0, 0, 0, 0);
    for (; t < end; t += SCHUR_T / 2) {
        const int4 tp = nxt;
        if (t + SCHUR_T / 2 < end) nxt = D.tuples[t + SCHUR_T / 2];   // the next tuple's index load flies under this tuple's block loads
        const int l = tp.z;
        // 19 128-bit loads per thread: every lane reads a different block, so the L1 wavefront count per byte is what bounds this kernel
        const double2* B1v = reinterpret_cast<const double2*>(D.Hpl + 18 * (size_t)tp.x) + 4 * h;   // doubles 8h .. 8h+9: rows 3h..3h+2 are w[h .. h+8]
        const double2* B2v = reinterpret_cast<const double2*>(D.Hpl + 18 * (size_t)tp.y);
        const double2* Div = reinterpret_cast<const double2*>(D.Dinv + DINV_LD * (size_t)l);
        double w[10], di[10], b2[18], b1[9];
#pragma unroll
        for (int i = 0; i < 5; i++) { const double2 v = B1v[i]; w[2 * i] = v.x; w[2 * i + 1] = v.y; const double2 u = Div[i]; di[2 * i] = u.x; di[2 * i + 1] = u.y; }
#pragma unroll
        for (int i = 0; i < 9; i++) { const double2 v = B2v[i]; b2[2 * i] = v.x; b2[2 * i + 1] = v.y; }
#pragma unroll
        for (int i = 0; i < 9; i++) b1[i] = h ? w[i + 1] : w[i];
#pragma unroll
        for (int i = 0; i < 3; i++) {
            const double t0 = b1[3 * i] * di[0] + b1[3 * i + 1] * di[3] + b1[3 * i + 2] * di[6];
            const double t1 = b1[3 * i] * di[1] + b1[3 * i + 1] * di[4] + b1[3 * i + 2] * di[7];
            const double t2 = b1[3 * i] * di[2] + b1[3 * i + 1] * di[5] + b1[3 * i + 2] * di[8];
#pragma unroll
            for (int j = 0; j < 6; j++) acc[6 * i + j] += t0 * b2[3 * j] + t1 * b2[3 * j + 1] + t2 * b2[3 * j + 2];
        }
        if (diag) {
            const double d0 = D.db[3 * l], d1 = D.db[3 * l + 1], d2 = D.db[3 * l + 2];
#pragma unroll
            for (int i = 0; i < 3; i++) acc[18 + i] += b1[3 * i] * d0 + b1[3 * i + 1] * d1 + b1[3 * i + 2] * d2;
        }
    }
    // lanes of equal parity hold the same rows: xor offsets 16 .. 2 leave the row sums in lanes 0 (rows 0-2) and 1 (rows 3-5)
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
#pragma unroll
    for (int i = 0; i < 21; i++) {
        if (i >= 18 && !diag) break;
        double v = acc[i];
#pragma unroll
        for (int o = 16; o > 1; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
        if (lane < 2) red[w][i < 18 ? 18 * lane + i : 36 + 3 * lane + (i - 18)] = v;
    }
    __syncthreads();
    const int n = D.n;
    if (threadIdx.x < 36) {
        const int i = threadIdx.x / 6, j = threadIdx.x % 6;
        double s = 0;
#pragma unroll
        for (int ww = 0; ww < SCHUR_T / 32; ww++) s += red[ww][threadIdx.x];
        double v = -s;
        if (diag) { v += D.Hpp[36 * p1 + threadIdx.x]; if (i == j) v += lambdaDiag; }
        out[(size_t)(6 * p1 + i) * n + 6 * p2 + j] = v;
        if (!diag) out[(size_t)(6 * p2 + j) * n + 6 * p1 + i] = v;
    } else if (diag && threadIdx.x < 42) {
        const int i = threadIdx.x - 36;
        double s = 0;
#pragma unroll
        for (int ww = 0; ww < SCHUR_T / 32; ww++) s += red[ww][threadIdx.x];
        const double b = D.bp[6 * p1 + i];
        double* g = out + (size_t)n * n;
        g[6 * p1 + i] = b - s;
        g[n + 6 * p1 + i] = b;   // bpr
    }
}

// ---------------------------------------------------------------------------------------------- reduced camera system solve
// Blocked right-looking LDL^T (no pivoting; LinearSolverEigen's SimplicialLDLT has none either) of the n x n system in ONE thread-block
// cluster. The right-hand side g sits right behind S, i.e. it is row n of an (n+1) x n matrix: carrying it through the factorisation
// as one more row performs the forward substitution (row n of L = D^-1 L^-1 g).
//
// Everything here is LATENCY bound (n ~ 300: 9 MFLOP; the per-instruction latencies can be measured with tools/ubench_fp64.cu), so every phase is written to keep its dependent chain short
// and to have all of a thread's L2 loads in flight together. Per panel of NB = 32 columns:
//   (1) every CTA factors the NB x NB diagonal block redundantly: thread (r, g) keeps elements (r, 4g..4g+3) in registers, the pivot column is
//       published through a double-buffered shared column -> one barrier per column; 1 / pivot = rcp.approx + 2 Newton steps (~55 clk).
//       Then M = (unit lower factor)^-1: each warp solves L m = e_k for 4 columns, lane = row, pivot entries by shuffle (no barrier);
//   (2) the rows below become a product instead of forward substitutions: X = A_rows M^T, L = X / d; FOUR lanes per row, lane j forms
//       the columns j, j+4, ... from the row held in registers (no dependent chain, no shuffles), a contiguous chunk of rows per CTA;
//       L goes back into S (row-major, for the back substitution) and L, L d go to the transposed panel buffers Lt / LDt;
//   (3) cluster barrier; every CTA copies both panels to shared memory (16-byte L2 loads, 4 in flight per thread); trailing update with
//       4 x 2 register tiles enumerated over the lower triangle only and dealt over all threads of the cluster; cluster barrier.
// Back substitution by cluster rank 0, panel by panel from the bottom: x_b = M_b^T y_b (one warp, 32 independent products per lane; M_b
// was parked in L2 scratch by (2)) instead of a 32-step triangular solve, then the rows above take y -= L_b^T x_b. scal[3] = 1 on a zero / non-finite pivot (LinearSolverEigen's failure): the LM trial is rejected.
static const int LD_NB = 32;
static const int SOLVE_T = 256;
static const int SOLVE_CLUSTER = 8;   // CTAs per solver cluster: the largest portable cluster size

// 1 / d to within an ulp: MUFU.RCP64H seed (~20 bits) and two Newton steps, instead of the ~127 clk IEEE divide on the critical path
__device__ __forceinline__ double fast_rcp(double d) {
    double r;
    asm("rcp.approx.ftz.f64 %0, %1;" : "=d"(r) : "d"(d));
    r = fma(r, fma(-d, r, 1.0), r);
    r = fma(r, fma(-d, r, 1.0), r);
    return r;
}

__global__ void __launch_bounds__(SOLVE_T) k_ba_solve(BADev D, double* __restrict__ Lt, double* __restrict__ LDt, double* __restrict__ Mg, int ldp, int stage) {
    extern __shared__ double dsm[];                 // [stage ? 2 * NB * ldp : 0] panels, then y[n] for the back substitution
    __shared__ double Pd[LD_NB][LD_NB + 1];         // L of the diagonal block (strictly lower part)
    __shared__ double Msm[LD_NB][LD_NB + 1];        // M = L^-1 of the diagonal block (zeros above the diagonal)
    __shared__ double colbuf[2][LD_NB];             // the pivot column of the current / next step
    __shared__ double dinvv[LD_NB];
    __shared__ int fail;
    cg::cluster_group cluster = cg::this_cluster();
    const int C = cluster.num_blocks(), crank = cluster.block_rank();
    const int n = D.n, tid = threadIdx.x;
    double* A = D.S;
    double* sL = dsm; double* sLD = dsm + (size_t)LD_NB * ldp;
    if (tid == 0) fail = 0;
    __syncthreads();
    for (int jb = 0; jb < n; jb += LD_NB) {
        const int nb = min(LD_NB, n - jb), rows = n + 1 - jb;
        // (1) diagonal block: thread (r, g) owns (r, 4g .. 4g+3)
        const int r = tid >> 3, g4 = (tid & 7) * 4;
        double a[4];
#pragma unroll
        for (int k = 0; k < 4; k++) { const int c = g4 + k; a[k] = (r < nb && c <= r) ? __ldcg(A + (size_t)(jb + r) * n + jb + c) : 0.0; }
        if (g4 == 0) colbuf[0][r] = a[0];
        __syncthreads();
#pragma unroll
        for (int c = 0; c < LD_NB; c++) {
            if (c < nb) {   // block-uniform
                const double* col = colbuf[c & 1];
                const double dc = col[c], ld = col[r];
                double l4[4];
#pragma unroll
                for (int k = 0; k < 4; k++) l4[k] = col[g4 + k];
                const double inv = fast_rcp(dc);
                if (tid == 0) dinvv[c] = inv;
                if (r > c) {
#pragma unroll
                    for (int k = 0; k < 4; k++) { const int c2 = g4 + k; if (c2 > c && c2 <= r) a[k] -= ld * (l4[k] * inv); }
                }
                if ((c >> 2) == (tid & 7)) Pd[r][c] = r > c ? ld * inv : 0.0;
                if (c + 1 < nb && ((c + 1) >> 2) == (tid & 7)) colbuf[(c + 1) & 1][r] = a[(c + 1) & 3];
                __syncthreads();
            }
        }
        // M = L^-1: warp w solves L m = e_k for the columns k = w, w+8, w+16, w+24 (lane = row; right-looking, the pivot entry travels by shuffle,
        // no block barrier inside). Columns >= nb of a short last panel stay unit vectors and are never used.
        {
            const int w = tid >> 5, ln = tid & 31;
            double mk[4], lrow[LD_NB];
#pragma unroll
            for (int c = 0; c < LD_NB; c++) lrow[c] = (c < nb && ln < nb && ln > c) ? Pd[ln][c] : 0.0;
#pragma unroll
            for (int q = 0; q < 4; q++) mk[q] = ln == w + 8 * q ? 1.0 : 0.0;
#pragma unroll
            for (int c = 0; c < LD_NB; c++) {
#pragma unroll
                for (int q = 0; q < 4; q++) {
                    if (c >= 8 * q) {   // column k = w + 8q is zero above row k >= 8q: earlier steps do nothing
                        const double mc = __shfl_sync(0xffffffffu, mk[q], c);
                        mk[q] -= lrow[c] * mc;   // lrow[c] == 0 for lanes <= c
                    }
                }
            }
#pragma unroll
            for (int q = 0; q < 4; q++) Msm[ln][w + 8 * q] = mk[q];
        }
        __syncthreads();
        if (tid < nb) { const double iv = dinvv[tid]; if (!isfinite(iv) || iv == 0.0) fail = 1; }   // zero / non-finite pivot <=> its reciprocal is not a finite non-zero number
        __syncthreads();
        if (fail) break;   // block-uniform and identical in every CTA of the cluster (same data)
        // (2) rows below the diagonal block (including the rhs row): a contiguous chunk of rows per CTA, 4 lanes per row, 8 columns per lane.
        // Per element the subtractions run over c2 = 0, 1, ... in the order of the plain forward substitution.
        const int trR = rows - nb;
        const int chunk = (trR + C - 1) / C, r0c = crank * chunk, r1c = min(r0c + chunk, trR);
        {
            // X = A_rows M^T (x_c = sum_{c2 <= c} a_c2 M[c][c2]), L = X / d. 4 lanes per row; lane j forms the columns j, j+4, ... (balanced: the
            // sum for column j + 4 m runs to c2 = 4 m + 3, the entries of M above the diagonal are zeros) from the whole row held in registers.
            const int j = tid & 3, slot = tid >> 2;
            for (int base = r0c; base < r1c; base += SOLVE_T / 4) {
                const int rr = base + slot;
                const bool valid = rr < r1c;
                double* Arow = A + (size_t)(jb + nb + (valid ? rr : r0c)) * n + jb;
                double av[LD_NB];
#pragma unroll
                for (int c = 0; c < LD_NB; c++) av[c] = (valid && c < nb) ? __ldcg(Arow + c) : 0.0;
                const double* Mj = &Msm[j][0];
#pragma unroll
                for (int mq = 0; mq < LD_NB / 4; mq++) {
                    if (4 * mq < nb) {   // block-uniform
                        double x0 = 0, x1 = 0;
#pragma unroll
                        for (int c2 = 0; c2 < 4 * mq + 4; c2 += 2) { x0 += av[c2] * Mj[4 * mq * (LD_NB + 1) + c2]; x1 += av[c2 + 1] * Mj[4 * mq * (LD_NB + 1) + c2 + 1]; }
                        const double x = x0 + x1;
                        const int c = j + 4 * mq;
                        if (valid && c < nb) {
                            const double lv = x * dinvv[c];
                            __stcg(Arow + c, lv);
                            __stcg(Lt + (size_t)c * ldp + rr, lv); __stcg(LDt + (size_t)c * ldp + rr, x);
                        }
                    }
                }
            }
        }
        // M of this panel to the scratch the back substitution reads (cluster rank 0)
        if (crank == 0)
            for (int i = tid; i < LD_NB * LD_NB; i += SOLVE_T) { const int rr = i / LD_NB, c = i - rr * LD_NB; __stcg(Mg + (size_t)(jb / LD_NB) * LD_NB * LD_NB + i, (rr < nb && c < nb) ? Msm[rr][c] : 0.0); }
        cluster.sync();
        // (3) trailing update A[i][k] -= sum_c (L d)[i][c] L[k][c], rows i include the rhs row, columns k < trC, k <= i
        const int trC = n - jb - nb;
        if (trC > 0) {
            if (stage) {
                // thread (half, q): panel columns c = 2 u + half, double2 words q and q + 128 of a panel row; 8 columns (16 .. 32 loads) in flight
                const int w2 = (trR + 1) >> 1, st2 = ldp >> 1, half = tid >> 7, q0 = tid & 127;
                const double2* gL = reinterpret_cast<const double2*>(Lt); const double2* gD = reinterpret_cast<const double2*>(LDt);
                double2* hL = reinterpret_cast<double2*>(sL); double2* hD = reinterpret_cast<double2*>(sLD);
                const bool q0ok = q0 < w2, q1ok = q0 + 128 < w2;
                for (int c0 = half; c0 < nb; c0 += 16) {
                    double2 vl[8][2], vd[8][2];
#pragma unroll
                    for (int u = 0; u < 8; u++) {
                        const int c = c0 + 2 * u;
                        if (c < nb) {
                            if (q0ok) { vl[u][0] = __ldcg(gL + c * st2 + q0); vd[u][0] = __ldcg(gD + c * st2 + q0); }
                            if (q1ok) { vl[u][1] = __ldcg(gL + c * st2 + q0 + 128); vd[u][1] = __ldcg(gD + c * st2 + q0 + 128); }
                        }
                    }
#pragma unroll
                    for (int u = 0; u < 8; u++) {
                        const int c = c0 + 2 * u;
                        if (c < nb) {
                            if (q0ok) { hL[c * st2 + q0] = vl[u][0]; hD[c * st2 + q0] = vd[u][0]; }
                            if (q1ok) { hL[c * st2 + q0 + 128] = vl[u][1]; hD[c * st2 + q0 + 128] = vd[u][1]; }
                        }
                    }
                }
                for (int q = q0 + 256; q < w2; q += 128)   // panels longer than 512 rows (not the staged regime in practice)
                    for (int c = half; c < nb; c += 2) { hL[c * st2 + q] = __ldcg(gL + c * st2 + q); hD[c * st2 + q] = __ldcg(gD + c * st2 + q); }
                __syncthreads();
            }
            const int tR = (trR + 3) >> 2, tC = (trC + 1) >> 1;
            // tile row br (4 rows) holds the tile columns bc with 2 bc <= 4 br + 3, i.e. bc <= 2 br + 1: 2 br + 2 tiles, br (br + 1) before it
            const int nTiles = tR * (tR + 1);
            for (int i = crank * SOLVE_T + tid; i < nTiles; i += C * SOLVE_T) {
                int br = (int)((sqrtf(4.0f * (float)i + 1.0f) - 1.0f) * 0.5f);
                while (br * (br + 1) > i) br--;
                while ((br + 1) * (br + 2) <= i) br++;
                const int bc = i - br * (br + 1);
                if (bc >= tC) continue;
                const int r0 = 4 * br, k0 = 2 * bc;
                // destination values first: their L2 latency runs under the product loop
                double dv[4][2]; bool ok[4][2];
#pragma unroll
                for (int q = 0; q < 4; q++) {
                    const int rr = r0 + q;
                    const double* dst = A + (size_t)(jb + nb + min(rr, trR - 1)) * n + jb + nb;
                    ok[q][0] = rr < trR && k0 <= rr && k0 < trC; ok[q][1] = rr < trR && k0 + 1 <= rr && k0 + 1 < trC;
                    dv[q][0] = ok[q][0] ? __ldcg(dst + k0) : 0.0; dv[q][1] = ok[q][1] ? __ldcg(dst + k0 + 1) : 0.0;
                }
                double acc[4][2] = {{0, 0}, {0, 0}, {0, 0}, {0, 0}};
                if (stage) {
                    const double2* qL = reinterpret_cast<const double2*>(sL + k0);
                    const double2* qD = reinterpret_cast<const double2*>(sLD + r0);
                    const int st = ldp >> 1;
#pragma unroll 8
                    for (int c = 0; c < nb; c++) {
                        const double2 bv = qL[c * st], a01 = qD[c * st], a23 = qD[c * st + 1];
                        acc[0][0] += a01.x * bv.x; acc[0][1] += a01.x * bv.y; acc[1][0] += a01.y * bv.x; acc[1][1] += a01.y * bv.y;
                        acc[2][0] += a23.x * bv.x; acc[2][1] += a23.x * bv.y; acc[3][0] += a23.y * bv.x; acc[3][1] += a23.y * bv.y;
                    }
                } else {
#pragma unroll 8
                    for (int c = 0; c < nb; c++) {
                        const double2 bv = __ldcg(reinterpret_cast<const double2*>(Lt + (size_t)c * ldp + k0));
                        const double2 a01 = __ldcg(reinterpret_cast<const double2*>(LDt + (size_t)c * ldp + r0));
                        const double2 a23 = __ldcg(reinterpret_cast<const double2*>(LDt + (size_t)c * ldp + r0 + 2));
                        acc[0][0] += a01.x * bv.x; acc[0][1] += a01.x * bv.y; acc[1][0] += a01.y * bv.x; acc[1][1] += a01.y * bv.y;
                        acc[2][0] += a23.x * bv.x; acc[2][1] += a23.x * bv.y; acc[3][0] += a23.y * bv.x; acc[3][1] += a23.y * bv.y;
                    }
                }
#pragma unroll
                for (int q = 0; q < 4; q++) {
                    double* dst = A + (size_t)(jb + nb + min(r0 + q, trR - 1)) * n + jb + nb;
                    if (ok[q][0]) __stcg(dst + k0, dv[q][0] - acc[q][0]);
                    if (ok[q][1]) __stcg(dst + k0 + 1, dv[q][1] - acc[q][1]);
                }
            }
        }
        cluster.sync();
    }
    if (fail) { if (crank == 0 && tid == 0) D.scal[3] = 1.0; return; }
    if (crank != 0) return;
    // backward: L^T x = z, z = row n of L (= D^-1 L^-1 g), panel by panel from the bottom: x_b = M_b^T y_b, then y_above -= L[b][above]^T x_b
    double* y = dsm + (stage ? 2 * (size_t)LD_NB * ldp : 0);
    for (int i = tid; i < n; i += SOLVE_T) y[i] = __ldcg(A + (size_t)n * n + i);
    __syncthreads();
    for (int pb = (n - 1) / LD_NB; pb >= 0; pb--) {
        const int j0 = pb * LD_NB, nb = min(LD_NB, n - j0);
        // rows above the block: L[j0 + j][i] for this thread's rows i; M_b[j][lane] for warp 0 (all independent of y: in flight together)
        double v0[LD_NB], v1[LD_NB];
        const int i0 = tid, i1 = tid + SOLVE_T;
#pragma unroll
        for (int j = 0; j < LD_NB; j++) {
            v0[j] = (j < nb && i0 < j0) ? __ldcg(A + (size_t)(j0 + j) * n + i0) : 0.0;
            v1[j] = (j < nb && i1 < j0) ? __ldcg(A + (size_t)(j0 + j) * n + i1) : 0.0;
        }
        if (tid < 32) {
            double mc[LD_NB], yv[LD_NB];
#pragma unroll
            for (int j = 0; j < LD_NB; j++) { mc[j] = __ldcg(Mg + (size_t)pb * LD_NB * LD_NB + j * LD_NB + tid); yv[j] = j < nb ? y[j0 + j] : 0.0; }
            double s0 = 0, s1 = 0, s2 = 0, s3 = 0;
#pragma unroll
            for (int j = 0; j < LD_NB; j += 4) { s0 += mc[j] * yv[j]; s1 += mc[j + 1] * yv[j + 1]; s2 += mc[j + 2] * yv[j + 2]; s3 += mc[j + 3] * yv[j + 3]; }
            __syncwarp();
            if (tid < nb) y[j0 + tid] = (s0 + s1) + (s2 + s3);
        }
        __syncthreads();
        {
            double s0 = 0, s1 = 0;
#pragma unroll
            for (int j = 0; j < LD_NB; j++) if (j < nb) { const double xj = y[j0 + j]; s0 += v0[j] * xj; s1 += v1[j] * xj; }
            if (i0 < j0) y[i0] -= s0;
            if (i1 < j0) y[i1] -= s1;
        }
        for (int i = tid + 2 * SOLVE_T; i < j0; i += SOLVE_T) {
            double sacc = 0;
            for (int j = 0; j < nb; j++) sacc += __ldcg(A + (size_t)(j0 + j) * n + i) * y[j0 + j];
            y[i] -= sacc;
        }
        __syncthreads();
    }
    for (int i = tid; i < n; i += SOLVE_T) D.xp[i] = y[i];
}

// xl = Dinv (bl - Hpl^T xp)   (block_solver.hpp:461-481). A failed reduced solve (scal[3] != 0) left xp unwritten: the trial is a zero step
// (xl = 0 here, xp taken as 0 by k_ba_update and k_ba_scale), as the LM loop models LinearSolver failure.
__global__ void __launch_bounds__(128) k_ba_backsub(BADev D) {
    const int l = (blockIdx.x * blockDim.x + threadIdx.x) / LM_LANES, sub = threadIdx.x % LM_LANES;
    const bool in = l < D.nMP, act = in && D.ptAct[l];
    double cl[3] = {0, 0, 0};
    const int eBeg = act ? D.lmStart[l] : 0, eEnd = act ? D.lmStart[l + 1] : 0;
    for (int a = eBeg + sub; a < eEnd; a += LM_LANES) {
        if (D.level[a] != 0) continue;
        const int p = D.poseIdx[D.eKF[a]];
        if (p < 0) continue;
        const double* B = D.Hpl + 18 * (size_t)a;
        const double* xq = D.xp + 6 * p;
#pragma unroll
        for (int j = 0; j < 3; j++) { double s = 0;
#pragma unroll
            for (int i = 0; i < 6; i++) s += B[3 * i + j] * xq[i]; cl[j] += s; }
    }
#pragma unroll
    for (int j = 0; j < 3; j++) { cl[j] += __shfl_xor_sync(0xffffffffu, cl[j], 1); cl[j] += __shfl_xor_sync(0xffffffffu, cl[j], 2); }
    if (!in || sub) return;
    if (!act || D.scal[3] != 0.0) { D.xl[3 * l] = 0; D.xl[3 * l + 1] = 0; D.xl[3 * l + 2] = 0; return; }
#pragma unroll
    for (int j = 0; j < 3; j++) cl[j] = D.bl[3 * l + j] - cl[j];
    const double* Di = D.Dinv + DINV_LD * (size_t)l;
#pragma unroll
    for (int i = 0; i < 3; i++) D.xl[3 * l + i] = Di[3 * i] * cl[0] + Di[3 * i + 1] * cl[1] + Di[3 * i + 2] * cl[2];
}

__device__ __noinline__ Pose pose_oplus_ba(const Pose& est, const double* u) { return pose_oplus(est, u); }

// push() + oplus (base_vertex.h:96-99, types_six_dof_expmap.h:73-76, types_sba.h:52-56)
__global__ void __launch_bounds__(256) k_ba_update(BADev D) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < D.nKF) { const Pose T = D.pose[i]; D.poseBak[i] = T; const int p = D.poseIdx[i]; if (p >= 0 && D.scal[3] == 0.0) D.pose[i] = pose_oplus_ba(T, D.xp + 6 * p); }
    if (i < D.nMP) {
        const double x = D.X[3 * i], y = D.X[3 * i + 1], z = D.X[3 * i + 2];
        D.Xbak[3 * i] = x; D.Xbak[3 * i + 1] = y; D.Xbak[3 * i + 2] = z;
        if (D.ptAct[i]) { D.X[3 * i] = x + D.xl[3 * i]; D.X[3 * i + 1] = y + D.xl[3 * i + 1]; D.X[3 * i + 2] = z + D.xl[3 * i + 2]; }
    }
}
// pop()
__global__ void __launch_bounds__(256) k_ba_restore(BADev D) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < D.nKF) D.pose[i] = D.poseBak[i];
    if (i < D.nMP) { D.X[3 * i] = D.Xbak[3 * i]; D.X[3 * i + 1] = D.Xbak[3 * i + 1]; D.X[3 * i + 2] = D.Xbak[3 * i + 2]; }
}

// computeScale: sum_j x_j (lambda x_j + b_j); the pose part is added by rank 0 only (replicated), landmarks by their owner. After a failed
// solve x = 0 goes through the same formula (a NaN lambda or b still gives NaN, as in the LM loop)
__global__ void __launch_bounds__(256) k_ba_scale(BADev D, double* out) {
    __shared__ double sh[32];
    const double lambda = D.scal[4];
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    double v = 0;
    if (i < D.n && D.rank == 0) { const double x = D.scal[3] == 0.0 ? D.xp[i] : 0.0; v = x * (lambda * x + D.bpr[i]); }
    const int j = i - D.n;
    if (j >= 0 && j < 3 * D.nMP) { const int l = j / 3; if (D.ptAct[l]) v = D.xl[j] * (lambda * D.xl[j] + D.bl[j]); }
    double tot;
    if (grid_sum(v, D.part, D.ticket, sh, &tot)) *out = tot;
}

// outlier test of src/Optimizer.cpp:384 / :411: chi2 of the LAST COMPUTED error (g2o keeps e->_error from the last
// computeActiveErrors, which may belong to a rejected trial) or non-positive depth in the rig frame
__global__ void __launch_bounds__(256) k_ba_classify(BADev D, uint8_t* flag) {
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= D.nE) return;
    double Xc[3];
    pose_map(D.pose[D.eKF[e]], D.X + 3 * D.eMP[e], Xc);
    const double chi = D.obs[3 * e + 2] * (D.err[2 * e] * D.err[2 * e] + D.err[2 * e + 1] * D.err[2 * e + 1]);
    flag[e] = (chi > 5.991 || !(Xc[2] > 0.0)) ? 1 : 0;
}

// ---------------------------------------------------------------------------------------------- one-shot NVLink all-reduce
// Multi-GPU LocalBA: every rank owns an exchange region that all peers map (CUDA IPC): two payloads [S n*n | g n | bpr n] (epoch
// parity), then 256 bytes of flags and the small-exchange slots. After k_ba_schur has written the rank's partial system into its payload
// of this epoch, k_ba_xchg_signal publishes `epoch` in every peer's flag slot for this rank (system-scope release); k_ba_xchg_reduce waits
// until all peers have published `epoch`, then every rank sums the payloads of all ranks in rank order (identical result everywhere) into
// its private reduced system BAHost::red and adds lambda to the diagonal. One 0.7 MB exchange per LM trial instead of five NCCL calls; a
// bounded spin turns a lost peer into an error, not a hang.
struct XchgPeers { const double* payload[8]; volatile unsigned* flags[8]; int n, rank; };
__global__ void k_ba_xchg_signal(XchgPeers P, unsigned epoch) {
    if (threadIdx.x < P.n) {
        __threadfence_system();
        P.flags[threadIdx.x][P.rank] = epoch;   // slot `rank` of peer threadIdx.x's flag array
        __threadfence_system();
    }
}
__global__ void __launch_bounds__(256) k_ba_xchg_reduce(XchgPeers P, unsigned epoch, double* dst, size_t count, int n, const double* lambdaPtr, int* err) {
    __shared__ int ok;
    const double lambda = *lambdaPtr;
    if (threadIdx.x == 0) {
        ok = 1;
        volatile unsigned* mine = P.flags[P.rank];
        for (int r = 0; r < P.n; r++) {
            long long spins = 0;
            while ((int)(mine[r] - epoch) < 0) { if (++spins > (1ll << 26)) { ok = 0; break; } __nanosleep(64); }   // a fast peer may already be one epoch ahead
            if (!ok) break;
        }
        __threadfence_system();
    }
    __syncthreads();
    if (!ok) { if (threadIdx.x == 0) *err = 1; return; }
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < count; i += (size_t)gridDim.x * blockDim.x) {
        double s = 0;
        for (int r = 0; r < P.n; r++) s += __ldcv(P.payload[r] + i);
        if (i < (size_t)n * n && (i / n) == (i % n)) s += lambda;
        dst[i] = s;
    }
}

// The scalars of a trial (chi2, scale; lambda_init's max diagonal) travel the same way: <= 4 doubles per rank in a double-buffered slot of
// the exchange region, one warp, one launch, fixed rank order (instead of a ~30 us ncclAllReduce per trial and per iteration).
struct SmallPeers { volatile unsigned* flags[8]; const double* slot[8]; double* mine; int n, rank; };
__global__ void k_ba_small_xchg(SmallPeers P, unsigned epoch, const double* src, double* dst, int count, int isMax, int* err) {
    const int t = threadIdx.x;
    double* slot = P.mine + (epoch & 1) * 4;
    if (t < count) slot[t] = src[t];
    __threadfence_system();
    __syncwarp();
    if (t < P.n) P.flags[t][P.rank] = epoch;
    __threadfence_system();
    bool ok = true;
    if (t < P.n) {
        volatile unsigned* mine = P.flags[P.rank];
        long long spins = 0;
        while ((int)(mine[t] - epoch) < 0) { if (++spins > (1ll << 26)) { ok = false; break; } __nanosleep(32); }
    }
    ok = __all_sync(0xffffffffu, ok);
    __threadfence_system();
    if (!ok) { if (t == 0) *err = 1; return; }
    if (t < count) {
        double v = __ldcv(P.slot[0] + (epoch & 1) * 4 + t);
        for (int r = 1; r < P.n; r++) { const double u = __ldcv(P.slot[r] + (epoch & 1) * 4 + t); v = isMax ? fmax(v, u) : v + u; }
        dst[t] = v;
    }
}
// multi-GPU: a rank classifies the edges of its own landmarks; the flags go to the caller's edge positions of a zeroed array that is max-reduced
__global__ void __launch_bounds__(256) k_ba_scatter_flags(int nLocal, const int* __restrict__ perm, const uint8_t* __restrict__ flag, uint8_t* __restrict__ out) {
    const int s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s < nLocal) out[perm[s]] = flag[s];
}
// NCCL path: lambda goes onto the diagonal of the summed system (the one-shot path adds it in k_ba_xchg_reduce)
__global__ void __launch_bounds__(256) k_ba_add_lambda(double* S, int n, double lambda) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) S[(size_t)i * n + i] += lambda;
}
// a rank's copy of another rank's point is stale: every point is taken from its owner (sum over ranks of owner ? X : 0)
__global__ void __launch_bounds__(256) k_ba_mask_points(BADev D) {
    const int l = blockIdx.x * blockDim.x + threadIdx.x;
    if (l < D.nMP && l % D.nranks != D.rank) { D.X[3 * l] = 0; D.X[3 * l + 1] = 0; D.X[3 * l + 2] = 0; }
}

}  // namespace cslam

// =================================================================================================== host side
using namespace cslam;

// ---- NCCL through dlopen (libnccl.so.2 is already mapped when torch.distributed is in use); no link-time dependency
typedef struct { char internal[128]; } nccl_uid_t;
struct NcclApi {
    void* h = nullptr;
    int (*GetUniqueId)(nccl_uid_t*) = nullptr;
    int (*CommInitRank)(nccl_comm_t*, int, nccl_uid_t, int) = nullptr;
    int (*AllReduce)(const void*, void*, size_t, int, int, nccl_comm_t, cudaStream_t) = nullptr;
    int (*AllGather)(const void*, void*, size_t, int, nccl_comm_t, cudaStream_t) = nullptr;
    int (*CommDestroy)(nccl_comm_t) = nullptr;
    const char* (*GetErrorString)(int) = nullptr;
};
static NcclApi* nccl_api() {
    static NcclApi api; static bool tried = false;
    if (tried) return api.h ? &api : nullptr;
    tried = true;
    const char* names[] = {"libnccl.so.2", "libnccl.so"};
    for (const char* n : names) { api.h = dlopen(n, RTLD_NOW | RTLD_GLOBAL); if (api.h) break; }
    if (!api.h) return nullptr;
    api.GetUniqueId = (int (*)(nccl_uid_t*))dlsym(api.h, "ncclGetUniqueId");
    api.CommInitRank = (int (*)(nccl_comm_t*, int, nccl_uid_t, int))dlsym(api.h, "ncclCommInitRank");
    api.AllReduce = (int (*)(const void*, void*, size_t, int, int, nccl_comm_t, cudaStream_t))dlsym(api.h, "ncclAllReduce");
    api.AllGather = (int (*)(const void*, void*, size_t, int, nccl_comm_t, cudaStream_t))dlsym(api.h, "ncclAllGather");
    api.CommDestroy = (int (*)(nccl_comm_t))dlsym(api.h, "ncclCommDestroy");
    api.GetErrorString = (const char* (*)(int))dlsym(api.h, "ncclGetErrorString");
    if (!api.GetUniqueId || !api.CommInitRank || !api.AllReduce || !api.CommDestroy) { dlclose(api.h); api.h = nullptr; return nullptr; }
    return &api;
}
enum { NCCL_U8 = 1, NCCL_I32 = 2, NCCL_F64 = 8, NCCL_SUM = 0, NCCL_MAX = 2 };
enum { BK_ERRORS = 0, BK_LIN_POINTS, BK_LIN_POSES, BK_DINV, BK_SCHUR, BK_XCHG, BK_SOLVE, BK_BACKSUB, BK_UPDATE, BK_SCALE, BK_COUNT, BK_END = KernelTimer::END };
static const char* kBaKindNames[BK_COUNT] = {"k_ba_errors", "k_ba_lin_points", "k_ba_lin_poses", "k_ba_dinv", "k_ba_schur", "exchange", "k_ba_solve", "k_ba_backsub", "k_ba_update", "k_ba_scale"};

extern "C" int cslam_optimizer_create(cslam_optimizer** out, int device) {
    if (!out) return CSLAM_E_BADARG;
    cslam_optimizer* o = new cslam_optimizer;
    int rc;
    if ((rc = o->open(device, (size_t)64 << 20, false)) || (rc = pinned_alloc(o->pinned, &o->h_scal, 16))) { destroy_handle(o); return rc; }
    cudaFuncSetAttribute(k_ba_solve, cudaFuncAttributeMaxDynamicSharedMemorySize, 204 * 1024);
    *out = o;
    return CSLAM_OK;
}
static void close_peers(cslam_optimizer* o) {
    for (auto& p : o->peers) { if (p.base && !p.mine) cudaIpcCloseMemHandle(p.base); else if (p.base) cudaFree(p.base); }
}
cslam_optimizer::~cslam_optimizer() {
    close_peers(this);
    if (comm && nccl_api()) nccl_api()->CommDestroy(comm);
}
extern "C" void cslam_optimizer_destroy(cslam_optimizer* o) { destroy_handle(o); }
extern "C" int64_t cslam_optimizer_launches(const cslam_optimizer* o) { return o ? o->launches : 0; }
extern "C" int cslam_optimizer_set_timing(cslam_optimizer* o, int enable) {
    if (!o) return CSLAM_E_BADARG;
    CSLAM_CUDA(cudaSetDevice(o->device));
    return o->timer.enable(enable != 0, 64);
}
extern "C" int cslam_optimizer_get_timing(const cslam_optimizer* o, int kind, const char** name, double* ms, int64_t* count) {
    return o ? o->timer.get(kind, BK_COUNT, kBaKindNames, name, ms, count) : CSLAM_E_BADARG;
}

extern "C" int cslam_nccl_unique_id(uint8_t id128[128]) {
    NcclApi* a = nccl_api();
    if (!a) { set_error("libnccl.so.2 not found"); return CSLAM_E_NCCL; }
    nccl_uid_t id; int rc = a->GetUniqueId(&id);
    if (rc) { set_error("ncclGetUniqueId failed (%d)", rc); return CSLAM_E_NCCL; }
    std::memcpy(id128, id.internal, 128);
    return CSLAM_OK;
}

// Exchange buffers of the one-shot all-reduce: allocate, publish the CUDA IPC handle through ncclAllGather, map every peer.
static const size_t XCHG_FLAG_BYTES = 256;
static int setup_xchg(cslam_optimizer* o, size_t payloadBytes) {
    NcclApi* a = nccl_api();
    if (o->nranks > 8 || !a->AllGather) return 1;   // fall back to NCCL
    close_peers(o);
    o->peers.assign(o->nranks, cslam_optimizer::Peer());
    void* mine = nullptr;
    const size_t bytes = 2 * ((payloadBytes + 255) & ~(size_t)255) + XCHG_FLAG_BYTES;   // two payload buffers (epoch parity) + the flag slots
    CSLAM_CUDA(cudaMalloc(&mine, bytes));
    CSLAM_CUDA(cudaMemset(mine, 0, bytes));
    cudaIpcMemHandle_t h;
    CSLAM_CUDA(cudaIpcGetMemHandle(&h, mine));
    cudaIpcMemHandle_t* dAll = nullptr;
    CSLAM_CUDA(cudaMalloc((void**)&dAll, sizeof(h) * o->nranks));
    CSLAM_CUDA(cudaMemcpy(dAll + o->rank, &h, sizeof(h), cudaMemcpyHostToDevice));
    int rc = a->AllGather(dAll + o->rank, dAll, sizeof(h), NCCL_U8, o->comm, o->stream);
    if (rc) { set_error("ncclAllGather (IPC handles) failed (%d)", rc); return CSLAM_E_NCCL; }
    std::vector<cudaIpcMemHandle_t> all(o->nranks);
    CSLAM_CUDA(cudaMemcpyAsync(all.data(), dAll, sizeof(h) * o->nranks, cudaMemcpyDeviceToHost, o->stream));
    CSLAM_CUDA(cudaStreamSynchronize(o->stream));
    cudaFree(dAll);
    bool ok = true;
    for (int r = 0; r < o->nranks; r++) {
        if (r == o->rank) { o->peers[r].base = mine; o->peers[r].mine = true; continue; }
        void* p = nullptr;
        if (cudaIpcOpenMemHandle(&p, all[r], cudaIpcMemLazyEnablePeerAccess) != cudaSuccess) { cudaGetLastError(); ok = false; break; }
        o->peers[r].base = p;
    }
    // all ranks must agree on the path
    double* flag = nullptr;
    CSLAM_CUDA(cudaMalloc((void**)&flag, 8));
    const double v = ok ? 0.0 : 1.0;
    CSLAM_CUDA(cudaMemcpy(flag, &v, 8, cudaMemcpyHostToDevice));
    rc = a->AllReduce(flag, flag, 1, NCCL_F64, NCCL_SUM, o->comm, o->stream);
    double bad = 1;
    CSLAM_CUDA(cudaMemcpyAsync(&bad, flag, 8, cudaMemcpyDeviceToHost, o->stream));
    CSLAM_CUDA(cudaStreamSynchronize(o->stream));
    cudaFree(flag);
    if (rc || bad != 0.0) return 1;
    o->xchgBytes = payloadBytes; o->oneShot = true; o->epoch = 0; o->epoch2 = 0;
    return 0;
}

extern "C" int cslam_optimizer_init_nccl(cslam_optimizer* o, const uint8_t id128[128], int rank, int nranks) {
    if (!o || !id128 || nranks < 1 || rank < 0 || rank >= nranks) return CSLAM_E_BADARG;
    NcclApi* a = nccl_api();
    if (!a) { set_error("libnccl.so.2 not found"); return CSLAM_E_NCCL; }
    CSLAM_CUDA(cudaSetDevice(o->device));
    nccl_uid_t id; std::memcpy(id.internal, id128, 128);
    int rc = a->CommInitRank(&o->comm, nranks, id, rank);
    if (rc) { set_error("ncclCommInitRank failed: %s", a->GetErrorString ? a->GetErrorString(rc) : "?"); return CSLAM_E_NCCL; }
    o->rank = rank; o->nranks = nranks;
    return CSLAM_OK;
}

// Per-edge input conversion on the device (was a host loop): cube face of the key point (CamModelGeneral::FaceInCubemap(cv::Point2f),
// float arithmetic as the reference), position inside the face as double (GetPosInFace<double>), information weight; s = position in the
// landmark-sorted order, perm[s] = the caller's edge index (perm == nullptr: the caller's order is already grouped by landmark).
__global__ void __launch_bounds__(256) k_ba_prep_edges(int nE, const int* __restrict__ perm, const float2* __restrict__ kp, const float* __restrict__ isig, int faceW, int faceH,
                                                       double* __restrict__ obs, int8_t* __restrict__ face, int* __restrict__ bad) {
    const int s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= nE) return;
    const int e = perm ? perm[s] : s;
    const float2 k = kp[e];
    const int f = face_of_pixel_f(k.x, k.y, faceW, faceH);
    if (f < 0) atomicMin(bad, e);
    face[s] = (int8_t)f;
    obs[3 * s] = pos_in_face(k.x, faceW);
    obs[3 * s + 1] = pos_in_face(k.y, faceH);
    obs[3 * s + 2] = (double)isig[e];
}
__global__ void __launch_bounds__(256) k_ba_prep_points(int n3, const float* __restrict__ in, double* __restrict__ out) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n3) out[i] = (double)in[i];
}

static int grid(int n, int t = 256) { return std::max(1, cdiv(n, t)); }   // blocks of t threads for n items, at least one

namespace {
struct BAHost {
    cslam_optimizer* o; BADev D; cslam_ba_problem* p; cslam_ba_result* res;
    int nEg = 0;                      // the caller's edges (D.nE: the edges this rank works on)
    const int* perm = nullptr;        // sorted edge position -> caller's edge index; nullptr = identity (input already grouped by landmark)
    const int* h_eMP = nullptr; const int* h_eKF = nullptr; int nActive = 0;   // landmark-sorted edge endpoints on the host
    std::vector<Pose> poses; std::vector<uint8_t> level; std::vector<int> poseIdx; std::vector<uint8_t> ptAct;
    const int* d_perm = nullptr; int* d_bad = nullptr; long long* pairCnt = nullptr;
    int* d_poseIdx = nullptr; uint8_t* d_ptAct = nullptr; uint8_t* d_flag = nullptr; int* d_pact = nullptr;
    double* Lt = nullptr; double* LDt = nullptr; double* Minv = nullptr; int ldp = 0;   // panel buffers, inverses of the diagonal blocks' unit factors
    double* red = nullptr;            // the reduced camera system [S | g | bpr], private to the rank
    double* HppFull = nullptr;        // multi-GPU: all-reduced copy of the pose blocks for computeLambdaInit
    size_t xstride = 0;               // one-shot path: doubles between the two payload buffers of an exchange region
    int* d_xerr = nullptr;
    double lambda = -1, ni = 2; int nBad = 0; int iterations = 0, trials = 0, stopAfterTrials = 0;
    bool errorsCurrent = false; double lastChi = 0;   // D.err / chi2 belong to the current state (set by an accepted trial)
    const volatile uint8_t* stop = nullptr;
    bool useOneShot = false;
    cudaGraphExec_t trialGraph = nullptr; int64_t launchesPerTrial = 0;
    ~BAHost() { drop_graph(); }
    // pbStopFlag; stopAfterTrials (a test hook, 0 = off): as if the flag became non-zero right after that trial of the call
    bool terminate() const { return (stop && *stop != 0) || (stopAfterTrials > 0 && trials >= stopAfterTrials); }
    size_t payload() const { return (size_t)D.n * D.n + 2 * (size_t)D.n; }
    void tick(int kind) { o->timer.record(o->stream, kind); }
    void drop_graph() { if (trialGraph) { cudaGraphExecDestroy(trialGraph); trialGraph = nullptr; } }

    // ---- set-up of one call, in call order
    // Edges sorted by landmark (stable), CSR by landmark and by key frame. On several GPUs a rank keeps only the edges of its own landmarks
    // (see BADev), so every per-edge kernel, the co-observation lists and the Schur work shrink by 1 / nranks. Host work is two passes over
    // the endpoint arrays, in scratch vectors that live in the optimizer object (no page faults per call).
    int sort_edges() {
        cslam_optimizer::HostScratch& hs = o->hs;
        const bool multi = o->nranks > 1;
        auto mine = [&](int l) { return !multi || l % o->nranks == o->rank; };
        hs.lmStart.assign(D.nMP + 1, 0);
        bool grouped = !multi;
        int nE = 0;
        for (int e = 0; e < nEg; e++) {
            const int l = p->edge_mp[e], k = p->edge_kf[e];
            if (l < 0 || l >= D.nMP || k < 0 || k >= D.nKF) { set_error("edge %d references a vertex out of range", e); return CSLAM_E_BADARG; }
            if (!mine(l)) continue;
            hs.lmStart[l + 1]++; nE++;
            if (e && l < p->edge_mp[e - 1]) grouped = false;
        }
        D.nE = nE;
        for (int l = 0; l < D.nMP; l++) hs.lmStart[l + 1] += hs.lmStart[l];
        if (grouped) { perm = nullptr; h_eMP = p->edge_mp; h_eKF = p->edge_kf; }
        else {
            hs.perm.resize(nE); hs.eMP.resize(nE); hs.eKF.resize(nE); hs.fill.assign(hs.lmStart.begin(), hs.lmStart.end() - 1);
            for (int e = 0; e < nEg; e++) { const int l = p->edge_mp[e]; if (mine(l)) hs.perm[hs.fill[l]++] = e; }
            for (int s = 0; s < nE; s++) { const int e = hs.perm[s]; hs.eMP[s] = p->edge_mp[e]; hs.eKF[s] = p->edge_kf[e]; }
            perm = hs.perm.data(); h_eMP = hs.eMP.data(); h_eKF = hs.eKF.data();
        }
        hs.peStart.assign(D.nKF + 1, 0); hs.peList.resize(nE);
        for (int s = 0; s < nE; s++) hs.peStart[h_eKF[s] + 1]++;
        for (int k = 0; k < D.nKF; k++) hs.peStart[k + 1] += hs.peStart[k];
        hs.fill.assign(hs.peStart.begin(), hs.peStart.end() - 1);
        for (int s = 0; s < nE; s++) hs.peList[hs.fill[h_eKF[s]]++] = s;
        return 0;
    }
    // Poses, CSRs and sorted endpoints to the device. k_ba_prep_edges forms each edge's face, position in the face and weight, and leaves
    // the smallest caller index of an off-face key point in d_bad (checked by build_pairs); k_ba_prep_points converts the points to fp64.
    // Every host source of an upload outlives the call (BAHost members, the optimizer's scratch, the caller's arrays), so the copies stay
    // valid whether or not the runtime has staged them when cudaMemcpyAsync returns.
    int stage_inputs() {
        const int nKF = D.nKF, nMP = D.nMP, nE = D.nE;
        cslam_optimizer::HostScratch& hs = o->hs;
        poses.resize(nKF);
        for (int k = 0; k < nKF; k++) poses[k] = pose_from_Tcw32(p->Tcw + 16 * k);
        level.assign(nE, 0); poseIdx.assign(nKF, -1); ptAct.assign(nMP, 0);
        hs.kfOfQ.clear();
        for (int k = 0; k < nKF; k++) if (!p->kf_fixed[k]) hs.kfOfQ.push_back(k);
        D.nQ = (int)hs.kfOfQ.size();
        const Pose* cpose = nullptr; const float2* d_kp = nullptr; const float* d_isig = nullptr; const float* d_pts32 = nullptr;
        double* d_obs = nullptr; int8_t* d_face = nullptr;
        DevArena& A = o->arena;
        int rc;
        if ((rc = A.upload(&cpose, poses.data(), poses.size())) || (rc = A.upload(&D.lmStart, hs.lmStart.data(), hs.lmStart.size())) ||
            (rc = A.upload(&D.peStart, hs.peStart.data(), hs.peStart.size())) || (rc = A.upload(&D.peList, hs.peList.data(), hs.peList.size())) ||
            (rc = A.upload(&D.kfOfQ, hs.kfOfQ.data(), hs.kfOfQ.size())) || (rc = A.upload(&D.eMP, h_eMP, nE)) || (rc = A.upload(&D.eKF, h_eKF, nE)) ||
            (rc = A.upload(&d_kp, reinterpret_cast<const float2*>(p->kp_xy), nEg)) || (rc = A.upload(&d_isig, p->inv_sigma2, nEg)) ||
            (rc = A.upload(&d_pts32, p->points, (size_t)nMP * 3)) || (rc = A.take(&D.X, (size_t)nMP * 3)) || (rc = A.take(&d_obs, (size_t)nE * 3)) ||
            (rc = A.take(&d_face, nE)) || (rc = A.take(&d_bad, 1)) || (perm && (rc = A.upload(&d_perm, perm, nE)))) return rc;
        CSLAM_CUDA(cudaMemsetAsync(d_bad, 0x7f, sizeof(int), o->stream));
        if (nE > 0) { k_ba_prep_edges<<<grid(nE), 256, 0, o->stream>>>(nE, d_perm, d_kp, d_isig, p->face_w, p->face_h, d_obs, d_face, d_bad); o->launches++; }
        if (nMP > 0) { k_ba_prep_points<<<grid(nMP * 3), 256, 0, o->stream>>>(nMP * 3, d_pts32, D.X); o->launches++; }
        D.obs = d_obs; D.face = d_face; D.pose = const_cast<Pose*>(cpose);
        // device state of the LM loop, sized for every candidate pose; on several GPUs, the exchange path of the reduced system
        const int nQ = D.nQ, nmax = 6 * nQ;
        const size_t payloadMax = (size_t)nmax * nmax + 2 * (size_t)nmax;
        const int maxBlocks = std::max(grid(nE), grid(nmax + 3 * nMP));
        ldp = ((nmax + 1 + 8) + 3) & ~3;
        if ((rc = A.take(&D.poseBak, nKF)) || (rc = A.take(&D.Xbak, (size_t)nMP * 3)) || (rc = A.take(&D.err, (size_t)nE * 2, true)) || (rc = A.take(&D.level, nE, true)) ||
            (rc = A.take(&d_poseIdx, nKF)) || (rc = A.take(&d_pact, nKF + 1)) || (rc = A.take(&d_ptAct, nMP)) || (rc = A.take(&d_flag, nE)) ||
            (rc = A.take(&D.Hpp, (size_t)std::max(nQ, 1) * 36)) || (rc = A.take(&D.bp, (size_t)std::max(nQ, 1) * 6)) || (rc = A.take(&D.Hll, (size_t)nMP * 9)) ||
            (rc = A.take(&D.bl, (size_t)nMP * 3)) || (rc = A.take(&D.Hpl, (size_t)nE * 18)) || (rc = A.take(&D.Dinv, (size_t)nMP * DINV_LD)) ||
            (rc = A.take(&D.db, (size_t)nMP * 3)) || (rc = A.take(&red, payloadMax)) || (rc = A.take(&D.xp, std::max(nmax, 1), true)) ||
            (rc = A.take(&D.xl, (size_t)nMP * 3, true)) || (rc = A.take(&D.scal, 8, true)) || (rc = A.take(&D.part, maxBlocks)) || (rc = A.take(&D.ticket, 4, true)) ||
            (rc = A.take(&D.posePart, (size_t)std::max(nQ, 1) * POSE_SPLIT * 27)) || (rc = A.take(&D.poseTicket, std::max(nQ, 1), true)) ||
            (rc = A.take(&Lt, (size_t)LD_NB * ldp)) || (rc = A.take(&LDt, (size_t)LD_NB * ldp)) || (rc = A.take(&Minv, (size_t)(nmax / LD_NB + 1) * LD_NB * LD_NB)) ||
            (rc = A.take(&pairCnt, (size_t)nQ * nQ + 1)) || (rc = A.take(&d_xerr, 1, true))) return rc;
        D.poseIdx = d_poseIdx; D.ptAct = d_ptAct;
        if (o->nranks > 1) {
            // The one-shot path falls back to ncclAllReduce by itself where CUDA IPC is unavailable; CSLAM_BA_NCCL_ONLY forces that
            // fallback, the only way to exercise it on a machine where IPC works.
            const bool ncclOnly = getenv("CSLAM_BA_NCCL_ONLY") != nullptr;
            if (!ncclOnly && (!o->oneShot || o->xchgBytes < payloadMax * 8)) {
                const int xr = setup_xchg(o, payloadMax * 8);
                if (xr < 0) return xr;
            }
            useOneShot = o->oneShot && o->xchgBytes >= payloadMax * 8 && !ncclOnly;
            xstride = ((o->xchgBytes + 255) & ~(size_t)255) / 8;
            if ((rc = A.take(&HppFull, (size_t)std::max(nQ, 1) * 36))) return rc;
        }
        return 0;
    }
    // Co-observation lists (once per call, over all of the rank's edges), and the off-face check of k_ba_prep_edges at the same synchronise.
    int build_pairs() {
        const int nQ = D.nQ;
        long long total = 0; int badEdge = 0;
        if (nQ > 0) {
            k_ba_pairs_count<<<dim3(nQ, nQ), 128, 0, o->stream>>>(D, pairCnt); o->launches++;
            k_ba_pairs_scan<<<1, 1024, 0, o->stream>>>(pairCnt, nQ * nQ); o->launches++;
            CSLAM_CUDA(cudaMemcpyAsync(&total, pairCnt + (size_t)nQ * nQ, sizeof(long long), cudaMemcpyDeviceToHost, o->stream));
        }
        CSLAM_CUDA(cudaMemcpyAsync(&badEdge, d_bad, sizeof(int), cudaMemcpyDeviceToHost, o->stream));
        CSLAM_CUDA(cudaStreamSynchronize(o->stream));
        if (badEdge < nEg) { set_error("edge %d: keypoint (%g,%g) is on no cube face (the reference calls exit() here)", badEdge, p->kp_xy[2 * badEdge], p->kp_xy[2 * badEdge + 1]); return CSLAM_E_BADARG; }
        if (nQ == 0) return 0;
        int4* tuples = nullptr;
        int rc;
        if ((rc = o->arena.take(&tuples, (size_t)std::max<long long>(total, 1)))) return rc;
        k_ba_pairs_fill<<<dim3(nQ, nQ), 128, 0, o->stream>>>(D, pairCnt, tuples); o->launches++;
        CSLAM_CUDA(cudaGetLastError());
        D.pairStart = pairCnt; D.tuples = tuples;
        return 0;
    }

    // ---- the LM loop
    int allreduce(const char* what, void* buf, size_t count, int op, int type = NCCL_F64) {   // in place; `what` names the data in the error
        if (o->nranks <= 1) return 0;
        int rc = nccl_api()->AllReduce(buf, buf, count, type, op, o->comm, o->stream);
        if (rc) { set_error("ncclAllReduce (%s) failed (%d)", what, rc); return CSLAM_E_NCCL; }
        return 0;
    }
    // <= 4 doubles, in place: the one-shot path when the peer views exist, NCCL otherwise
    int allreduce_small(double* buf, int count, bool isMax) {
        if (o->nranks <= 1) return 0;
        if (!useOneShot) return allreduce("trial scalars", buf, count, isMax ? NCCL_MAX : NCCL_SUM);
        SmallPeers P; P.n = o->nranks; P.rank = o->rank;
        const size_t off = 2 * xstride * 8;
        for (int r = 0; r < o->nranks; r++) { P.flags[r] = (volatile unsigned*)((char*)o->peers[r].base + off + 64); P.slot[r] = (const double*)((char*)o->peers[r].base + off + 128); }
        P.mine = (double*)((char*)o->peers[o->rank].base + off + 128);
        k_ba_small_xchg<<<1, 32, 0, o->stream>>>(P, ++o->epoch2, buf, buf, count, isMax ? 1 : 0, d_xerr); o->launches++;
        return 0;
    }
    int fetch(const double* src, int count) {
        CSLAM_CUDA(cudaMemcpyAsync(o->h_scal, src, count * sizeof(double), cudaMemcpyDeviceToHost, o->stream));
        CSLAM_CUDA(cudaStreamSynchronize(o->stream));
        return 0;
    }

    // initializeOptimization(level 0): active edges, active vertices, compact pose indices (sparse_optimizer.cpp:206-267,166-190)
    int initialize() {
        std::vector<int> pAct(D.nKF + 1, 0);   // [nKF] = this rank has an active edge
        std::fill(ptAct.begin(), ptAct.end(), 0);
        nActive = 0;
        for (int e = 0; e < D.nE; e++) if (level[e] == 0) { pAct[h_eKF[e]] = 1; ptAct[h_eMP[e]] = 1; nActive++; }
        pAct[D.nKF] = nActive > 0;
        if (o->nranks > 1) {   // a rank sees the edges of its own landmarks only: pose activity and "anything to optimize" are global facts
            CSLAM_CUDA(cudaMemcpyAsync(d_pact, pAct.data(), (D.nKF + 1) * sizeof(int), cudaMemcpyHostToDevice, o->stream));
            if (int rc = allreduce("pose activity", d_pact, D.nKF + 1, NCCL_MAX, NCCL_I32)) return rc;
            CSLAM_CUDA(cudaMemcpyAsync(pAct.data(), d_pact, (D.nKF + 1) * sizeof(int), cudaMemcpyDeviceToHost, o->stream));
            CSLAM_CUDA(cudaStreamSynchronize(o->stream));
            nActive = pAct[D.nKF];   // only tested against zero
        }
        int nP = 0;
        for (int k = 0; k < D.nKF; k++) poseIdx[k] = (pAct[k] && !p->kf_fixed[k]) ? nP++ : -1;
        D.nP = nP; D.n = 6 * nP;
        D.S = red; D.bpr = red + (size_t)D.n * D.n + D.n;
        CSLAM_CUDA(cudaMemcpyAsync(d_poseIdx, poseIdx.data(), D.nKF * sizeof(int), cudaMemcpyHostToDevice, o->stream));
        CSLAM_CUDA(cudaMemcpyAsync(d_ptAct, ptAct.data(), D.nMP, cudaMemcpyHostToDevice, o->stream));
        CSLAM_CUDA(cudaMemcpyAsync(D.level, level.data(), D.nE, cudaMemcpyHostToDevice, o->stream));
        errorsCurrent = false;   // level / robust kernel changed
        drop_graph();   // the captured trial bakes in nP / n / the level array's meaning
        return 0;
    }
    int errors_chi2(double* chi) {   // computeActiveErrors + activeRobustChi2
        k_ba_errors<<<grid(D.nE), 256, 0, o->stream>>>(D, D.scal); o->launches++;
        int rc;
        if ((rc = allreduce_small(D.scal, 1, false))) return rc;
        if ((rc = fetch(D.scal, 1))) return rc;
        *chi = o->h_scal[0];
        return 0;
    }
    int build_system() {
        k_ba_lin_points<<<grid(D.nMP * LM_LANES, 128), 128, 0, o->stream>>>(D); o->launches++;
        tick(BK_LIN_POSES);
        if (D.nQ > 0) { k_ba_lin_poses<<<dim3(D.nQ, POSE_SPLIT), 256, 0, o->stream>>>(D); o->launches++; }
        CSLAM_CUDA(cudaGetLastError());
        return 0;
    }
    int lambda_init(double* lam) {
        int rc;
        CSLAM_CUDA(cudaMemsetAsync(D.scal + 2, 0, sizeof(double), o->stream));
        CSLAM_CUDA(cudaMemsetAsync(D.scal + 5, 0, 2 * sizeof(double), o->stream));
        BADev M = D;
        if (o->nranks > 1 && D.nP > 0) {   // computeLambdaInit needs the full pose blocks: sum a COPY of the partial blocks once per optimize()
            CSLAM_CUDA(cudaMemcpyAsync(HppFull, D.Hpp, (size_t)D.nP * 36 * 8, cudaMemcpyDeviceToDevice, o->stream));
            if ((rc = allreduce("pose blocks", HppFull, (size_t)D.nP * 36, NCCL_SUM))) return rc;
            M.Hpp = HppFull;
        }
        k_ba_diag_keys<<<grid(D.nP * 6 + D.nMP * 3), 256, 0, o->stream>>>(M); o->launches++;
        if ((rc = allreduce_small(D.scal + 5, 2, true))) return rc;
        k_ba_maxdiag<<<grid(D.nP * 6 + D.nMP * 3), 256, 0, o->stream>>>(M); o->launches++;
        if ((rc = allreduce_small(D.scal + 2, 1, true))) return rc;
        if ((rc = fetch(D.scal, 7))) return rc;
        const double nanKey = o->h_scal[5], lastKey = o->h_scal[6];
        *lam = nanKey > 0 && nanKey == lastKey ? std::numeric_limits<double>::quiet_NaN() : 1e-5 * o->h_scal[2];
        return 0;
    }
    // One LM trial on the stream: lambda -> device, BlockSolver::solve (Dinv, Schur, [exchange], reduced solve, back substitution), push + oplus,
    // computeActiveErrors + activeRobustChi2, computeScale, the four scalars -> pinned host memory. Single-GPU trials are replayed as ONE CUDA graph.
    int enqueue_trial() {
        int rc;
        CSLAM_CUDA(cudaMemcpyAsync(D.scal + 4, o->h_scal + 8, sizeof(double), cudaMemcpyHostToDevice, o->stream));   // h_scal[8] = lambda
        tick(BK_DINV);
        k_ba_dinv<<<grid(D.nMP), 256, 0, o->stream>>>(D); o->launches++;
        CSLAM_CUDA(cudaMemsetAsync(D.scal + 3, 0, sizeof(double), o->stream));   // solve flag (no reduced system, n = 0, cannot fail)
        if (D.n > 0) {
            const bool multi = o->nranks > 1, oneShot = multi && useOneShot;
            const unsigned ep = oneShot ? ++o->epoch : 0;
            double* part = oneShot ? (double*)o->peers[o->rank].base + (ep & 1) * xstride : red;   // where this rank's partial system goes
            tick(BK_SCHUR);
            k_ba_schur<<<dim3(D.nQ, D.nQ), SCHUR_T, 0, o->stream>>>(D, part, multi ? 0 : 1); o->launches++;
            if (multi) {
                tick(BK_XCHG);
                if (oneShot) {
                    XchgPeers P; P.n = o->nranks; P.rank = o->rank;
                    const size_t off = 2 * xstride * 8;
                    for (int r = 0; r < o->nranks; r++) { P.payload[r] = (const double*)o->peers[r].base + (ep & 1) * xstride; P.flags[r] = (volatile unsigned*)((char*)o->peers[r].base + off); }
                    k_ba_xchg_signal<<<1, 32, 0, o->stream>>>(P, ep); o->launches++;
                    k_ba_xchg_reduce<<<std::min(132, grid((int)std::min<size_t>(payload(), 1u << 30))), 256, 0, o->stream>>>(P, ep, red, payload(), D.n, D.scal + 4, d_xerr); o->launches++;
                } else {
                    if ((rc = allreduce("reduced system", red, payload(), NCCL_SUM))) return rc;
                    k_ba_add_lambda<<<grid(D.n), 256, 0, o->stream>>>(red, D.n, lambda); o->launches++;
                }
            }
            tick(BK_SOLVE);
            const size_t panel = 2 * (size_t)LD_NB * ldp * 8, ybytes = (size_t)D.n * 8;
            const int stage = panel + ybytes <= 200 * 1024 ? 1 : 0;
            cudaLaunchConfig_t cfg = {};
            cfg.gridDim = dim3(SOLVE_CLUSTER); cfg.blockDim = dim3(SOLVE_T); cfg.dynamicSmemBytes = (stage ? panel : 0) + ybytes; cfg.stream = o->stream;
            cudaLaunchAttribute at[1];
            at[0].id = cudaLaunchAttributeClusterDimension; at[0].val.clusterDim.x = SOLVE_CLUSTER; at[0].val.clusterDim.y = 1; at[0].val.clusterDim.z = 1;
            cfg.attrs = at; cfg.numAttrs = 1;
            CSLAM_CUDA(cudaLaunchKernelEx(&cfg, k_ba_solve, D, Lt, LDt, Minv, ldp, stage)); o->launches++;
        }
        tick(BK_BACKSUB);
        k_ba_backsub<<<grid(D.nMP * LM_LANES, 128), 128, 0, o->stream>>>(D); o->launches++;
        tick(BK_UPDATE);
        k_ba_update<<<grid(std::max(D.nKF, D.nMP)), 256, 0, o->stream>>>(D); o->launches++;
        tick(BK_ERRORS);
        k_ba_errors<<<grid(D.nE), 256, 0, o->stream>>>(D, D.scal); o->launches++;
        tick(BK_SCALE);
        k_ba_scale<<<grid(D.n + 3 * D.nMP), 256, 0, o->stream>>>(D, D.scal + 1); o->launches++;
        tick(BK_END);
        if ((rc = allreduce_small(D.scal, 2, false))) return rc;
        CSLAM_CUDA(cudaMemcpyAsync(o->h_scal, D.scal, 4 * sizeof(double), cudaMemcpyDeviceToHost, o->stream));
        CSLAM_CUDA(cudaGetLastError());
        return 0;
    }
    int run_trial() {
        int rc;
        o->h_scal[8] = lambda;
        const bool useGraph = o->nranks == 1 && !o->timer.on();
        if (useGraph) {
            if (!trialGraph) {
                cudaGraph_t g = nullptr;
                const int64_t l0 = o->launches;
                CSLAM_CUDA(cudaStreamBeginCapture(o->stream, cudaStreamCaptureModeThreadLocal));
                rc = enqueue_trial();
                cudaError_t ce = cudaStreamEndCapture(o->stream, &g);
                if (rc) { if (g) cudaGraphDestroy(g); return rc; }
                CSLAM_CUDA(ce);
                CSLAM_CUDA(cudaGraphInstantiate(&trialGraph, g, 0));
                cudaGraphDestroy(g);
                launchesPerTrial = o->launches - l0; o->launches = l0;
            }
            CSLAM_CUDA(cudaGraphLaunch(trialGraph, o->stream));
            o->launches += launchesPerTrial;
        } else if ((rc = enqueue_trial())) return rc;
        CSLAM_CUDA(cudaStreamSynchronize(o->stream));
        o->timer.collect();
        return 0;
    }
    // OptimizationAlgorithmLevenberg::solve ; result 0 OK, 1 Terminate
    int lm_iteration(int iteration, int* result) {
        int rc; double currentChi = 0;
        tick(BK_ERRORS);
        // computeActiveErrors + activeRobustChi2: after an accepted trial the errors and chi2 of this very state are already on the device
        // (the trial evaluated them; same kernel, same inputs -> same bits), so only the first iteration and the ones after a rejection compute
        if (errorsCurrent) currentChi = lastChi;
        else if ((rc = errors_chi2(&currentChi))) return rc;
        const double iniChi = currentChi; double tempChi = currentChi;
        tick(BK_LIN_POINTS);
        if ((rc = build_system())) return rc;
        tick(BK_END);
        if (iteration == 0) { if ((rc = lambda_init(&lambda))) return rc; ni = 2; nBad = 0; }
        double rho = 0; int qmax = 0; int accepted = 0;
        do {
            if ((rc = run_trial())) return rc;
            tempChi = o->h_scal[0];
            bool ok2 = o->h_scal[3] == 0.0;
            trials++;
            if (!ok2) tempChi = DBL_MAX;
            rho = currentChi - tempChi;
            const double scale = o->h_scal[1] + 1e-3;
            rho /= scale;
            // levenberg.cpp:126-149 as it stands: a failed solve is a zero step with tempChi = DBL_MAX, and rho is whatever that gives (NaN
            // for an infinite currentChi or a NaN scale, which ends the trial loop on a rejected trial)
            if (rho > 0 && std::isfinite(tempChi)) {
                double alpha = 1. - std::pow((2 * rho - 1), 3);
                alpha = std::min(alpha, 2. / 3.);
                lambda *= std::max(1. / 3., alpha); ni = 2; currentChi = tempChi; accepted = 1;
                errorsCurrent = true; lastChi = o->h_scal[0];   // the trial's chi2 of this state (tempChi is DBL_MAX after a failed solve)
            } else {
                errorsCurrent = false;   // pop(): the state is the old one again, the error array holds the trial's
                lambda *= ni; ni *= 2;
                k_ba_restore<<<grid(std::max(D.nKF, D.nMP)), 256, 0, o->stream>>>(D); o->launches++;
            }
            qmax++;
        } while (rho < 0 && qmax < 10 && !terminate());
        if (res && res->lm_log && iterations < res->log_cap) {
            double* L = res->lm_log + 4 * iterations; L[0] = currentChi; L[1] = lambda; L[2] = qmax; L[3] = accepted;
        }
        iterations++;
        *result = 0;
        if (qmax == 10 || rho == 0) { *result = 1; return 0; }
        if ((iniChi - currentChi) * 1e3 < iniChi) nBad++; else nBad = 0;
        if (nBad >= 3) *result = 1;
        return 0;
    }
    int optimize(int its) {
        if (nActive == 0) return 0;   // g2o: "0 vertices to optimize"
        int result = 0;
        for (int i = 0; i < its && !terminate() && result == 0; i++) { int rc = lm_iteration(i, &result); if (rc) return rc; }
        if (o->nranks > 1 && useOneShot) {
            int xe = 0;
            CSLAM_CUDA(cudaMemcpyAsync(&xe, d_xerr, sizeof(int), cudaMemcpyDeviceToHost, o->stream));
            CSLAM_CUDA(cudaStreamSynchronize(o->stream));
            if (xe) { set_error("one-shot all-reduce: a peer never signalled (timeout)"); return CSLAM_E_NCCL; }
        }
        return 0;
    }
    int classify(std::vector<uint8_t>& flags) {   // flags of this rank's edges (all edges on one GPU)
        k_ba_classify<<<grid(D.nE), 256, 0, o->stream>>>(D, d_flag); o->launches++;
        flags.resize(D.nE);
        CSLAM_CUDA(cudaMemcpyAsync(flags.data(), d_flag, D.nE, cudaMemcpyDeviceToHost, o->stream));
        CSLAM_CUDA(cudaStreamSynchronize(o->stream));
        return 0;
    }
    // src/Optimizer.cpp:397-450: outlier flags in the caller's edge order, float32 poses and points (fp64 copies on request). On several GPUs
    // every rank returns the flags of all edges (max over the owners' flags) and every point from its owner.
    int write_back(const std::vector<uint8_t>& flags) {
        int rc;
        const int nKF = D.nKF, nMP = D.nMP;
        const bool multi = o->nranks > 1;
        std::vector<uint8_t> gflags;
        if (multi) {
            uint8_t* d_gflag = nullptr;
            if ((rc = o->arena.take(&d_gflag, std::max(nEg, 1), true))) return rc;
            if (D.nE > 0) { k_ba_scatter_flags<<<grid(D.nE), 256, 0, o->stream>>>(D.nE, d_perm, d_flag, d_gflag); o->launches++; }
            if ((rc = allreduce("flags", d_gflag, nEg, NCCL_MAX, NCCL_U8))) return rc;
            gflags.resize(nEg);
            CSLAM_CUDA(cudaMemcpyAsync(gflags.data(), d_gflag, nEg, cudaMemcpyDeviceToHost, o->stream));
            k_ba_mask_points<<<grid(nMP), 256, 0, o->stream>>>(D); o->launches++;
            if ((rc = allreduce("points", D.X, (size_t)nMP * 3, NCCL_SUM))) return rc;
        }
        CSLAM_CUDA(cudaMemcpyAsync(poses.data(), D.pose, nKF * sizeof(Pose), cudaMemcpyDeviceToHost, o->stream));
        std::vector<double>& X = o->hs.X;
        X.resize((size_t)nMP * 3);
        CSLAM_CUDA(cudaMemcpyAsync(X.data(), D.X, X.size() * 8, cudaMemcpyDeviceToHost, o->stream));
        if ((rc = o->sync())) return rc;
        for (int k = 0; k < nKF; k++) {
            pose_to_Tcw32(poses[k], p->Tcw + 16 * k);
            if (res && res->pose_fp64) pose_to_fp64(poses[k], res->pose_fp64 + 7 * k);
        }
        for (size_t i = 0; i < X.size(); i++) { p->points[i] = (float)X[i]; if (res && res->points_fp64) res->points_fp64[i] = X[i]; }
        if (res) {
            if (res->outlier) { if (multi) std::memcpy(res->outlier, gflags.data(), nEg); else for (int s = 0; s < D.nE; s++) res->outlier[perm ? perm[s] : s] = flags[s]; }
            res->iterations = iterations; res->trials = trials;
        }
        return CSLAM_OK;
    }
};
}  // namespace

extern "C" int cslam_local_ba(cslam_optimizer* o, cslam_ba_problem* p, const volatile uint8_t* stop_flag, int its1, int its2, cslam_ba_result* r) {
    if (!o || !p || p->n_kf <= 0 || p->n_mp < 0 || p->n_edges < 0 || !p->Tcw || !p->kf_fixed || (p->n_mp && !p->points)) { set_error("cslam_local_ba: bad problem"); return CSLAM_E_BADARG; }
    if (p->face_w != p->face_h || p->face_w <= 0) { set_error("cube faces must be square"); return CSLAM_E_BADARG; }
    CSLAM_CUDA(cudaSetDevice(o->device));
    o->arena.reset();
    if (r) { r->iterations = 0; r->trials = 0; if (r->outlier) std::memset(r->outlier, 0, p->n_edges); }
    if (stop_flag && *stop_flag) return CSLAM_OK;   // src/Optimizer.cpp:359-361
    BAHost H; H.o = o; H.p = p; H.res = r; H.stop = stop_flag; H.nEg = p->n_edges; H.stopAfterTrials = r ? r->stop_after_trials : 0;
    BADev& D = H.D; std::memset(&D, 0, sizeof(D));
    D.nKF = p->n_kf; D.nMP = p->n_mp; D.f = p->face_w / 2.0; D.rank = o->rank; D.nranks = o->nranks;
    D.robust = 1; D.delta = huber_delta(); D.dsqr = D.delta * D.delta;
    int rc;
    if ((rc = H.sort_edges()) || (rc = H.stage_inputs()) || (rc = H.build_pairs())) return rc;
    // src/Optimizer.cpp:363-395: optimize(5); unless stopped, drop the outliers and the robust kernel and optimize(10); classify again
    std::vector<uint8_t> flags;
    if ((rc = H.initialize()) || (rc = H.optimize(its1))) return rc;
    if (!H.terminate()) {
        if ((rc = H.classify(flags))) return rc;
        for (int s = 0; s < D.nE; s++) if (flags[s]) H.level[s] = 1;
        D.robust = 0;
        if ((rc = H.initialize()) || (rc = H.optimize(its2))) return rc;
    }
    if ((rc = H.classify(flags))) return rc;
    return H.write_back(flags);
}

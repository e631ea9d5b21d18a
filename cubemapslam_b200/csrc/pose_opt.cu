// Optimizer::PoseOptimization of libcubemap_b200.so (reference src/Optimizer.cpp:48-190; edge src/g2o_cubemap_vertices_edges.cpp:61-124), sm_90a.
// One CTA per frame, the whole 4 x optimize(10) schedule of the reference inside the kernel (dense 6x6 LM, LinearSolverDense).
#include <cfloat>
#include <cstring>
#include <vector>
#include "optimizer.cuh"

namespace cslam {

// ------------------------------------------------------------------------------------------------- PoseOptimization
// One CTA per frame; the whole schedule of src/Optimizer.cpp:138-181 (4 rounds x optimize(10), dense 6x6 LM) runs inside
// the kernel. Block reductions of chi2 and of the 27 unique entries of (H,b); thread 0 does the 6x6 LDL^T and the LM logic.
struct PoseOptArgs {
    const int* offset; float* Tcw; const float* Xw; const float* kpxy; const float* invSigma2;
    int faceW, faceH; uint8_t* outlier; int32_t* inliers; double* pose64; double* err; uint8_t* level;
    const int32_t* count; int stride;   // offset == nullptr: frame f owns correspondences [f*stride, f*stride + count[f])
    double* log; int32_t* nlog;         // optional LM log (test hook, nullptr in production): PO_LOG_ROWS rows of (chi2, lambda, trials, accepted) per frame
};
constexpr int PO_LOG_ROWS = 40;         // 4 rounds x optimize(10)

// The kernel is a long sequential schedule of block-wide phases. Every phase is an out-of-line device function (all threads call it
// convergently; barriers inside): ptxas handles each phase on its own instead of one enormous inlined body (which took ~20 minutes).
struct PoFrame {            // block-uniform per-frame context
    const float* Xw; const float* kpxy; const float* invSigma2; double* err; uint8_t* level; uint8_t* outlier;
    int beg, n, faceW, faceH; double fc, delta, dsqr;
};
struct PoShared { double sh[32]; double Hs[27]; double red[8][27]; Pose pose, pose0, backup; double x[6], lambda, ni, bc; int ctrl; };

__device__ __forceinline__ int po_obs_face(const PoFrame& F, int e, double& mx, double& my, double& w) {
    const float kx = F.kpxy[2 * e], ky = F.kpxy[2 * e + 1];
    const int face = face_of_pixel_f(kx, ky, F.faceW, F.faceH);
    mx = pos_in_face(kx, F.faceW); my = pos_in_face(ky, F.faceH);
    w = (double)F.invSigma2[e];
    return face;
}
__device__ __noinline__ double po_block_sum(double v, PoShared* S) {   // sum broadcast to every thread
    const double s = block_sum(v, S->sh);
    if (threadIdx.x == 0) S->bc = s;
    __syncthreads();
    const double r = S->bc;
    __syncthreads();
    return r;
}
// computeActiveErrors + activeRobustChi2
__device__ __noinline__ double po_compute_errors(const PoFrame& F, PoShared* S, bool robust) {
    double c = 0;
    const Pose pose = S->pose;
    for (int i = threadIdx.x; i < F.n; i += blockDim.x) {
        const int e = F.beg + i;
        if (F.level[e] != 0) continue;
        double mx, my, w; const int face = po_obs_face(F, e, mx, my, w);
        const double Xw[3] = {(double)F.Xw[3 * e], (double)F.Xw[3 * e + 1], (double)F.Xw[3 * e + 2]};
        double Xc[3], er[2];
        pose_map(pose, Xw, Xc); edge_error(face, F.fc, mx, my, Xc, er);
        F.err[2 * e] = er[0]; F.err[2 * e + 1] = er[1];
        const double chi = w * (er[0] * er[0] + er[1] * er[1]);
        if (robust) { double r0, r1; huber(F.delta, F.dsqr, chi, r0, r1); c += r0; } else c += chi;
    }
    return po_block_sum(c, S);
}
// buildSystem: the 21 + 6 unique entries of (H, b) -> S->Hs
__device__ __noinline__ void po_build_system(const PoFrame& F, PoShared* S, bool robust) {
    double acc[27];
#pragma unroll
    for (int k = 0; k < 27; k++) acc[k] = 0;
    const Pose pose = S->pose;
    for (int i = threadIdx.x; i < F.n; i += blockDim.x) {
        const int e = F.beg + i;
        if (F.level[e] != 0) continue;
        double mx, my, w0; const int face = po_obs_face(F, e, mx, my, w0);
        const double Xw[3] = {(double)F.Xw[3 * e], (double)F.Xw[3 * e + 1], (double)F.Xw[3 * e + 2]};
        double Xc[3], G[2][3], Jp[2][6];
        pose_map(pose, Xw, Xc); edge_G(face, F.fc, Xc, G); edge_Jpose(G, Xc, Jp);
        const double e0 = F.err[2 * e], e1 = F.err[2 * e + 1];
        double rho1 = 1.0;
        if (robust) { double r0; huber(F.delta, F.dsqr, w0 * (e0 * e0 + e1 * e1), r0, rho1); }
        int k = 0;
#pragma unroll
        for (int a = 0; a < 6; a++)
#pragma unroll
            for (int b = a; b < 6; b++) acc[k++] += (rho1 * w0) * (Jp[0][a] * Jp[0][b] + Jp[1][a] * Jp[1][b]);
#pragma unroll
        for (int a = 0; a < 6; a++) acc[21 + a] -= rho1 * (Jp[0][a] * w0 * e0 + Jp[1][a] * w0 * e1);
    }
#pragma unroll
    for (int k = 0; k < 27; k++) {
        double v = acc[k];
#pragma unroll
        for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
        if ((threadIdx.x & 31) == 0) S->red[threadIdx.x >> 5][k] = v;
    }
    __syncthreads();
    if (threadIdx.x < 27) { double s = 0; for (int w = 0; w < (int)(blockDim.x >> 5); w++) s += S->red[w][threadIdx.x]; S->Hs[threadIdx.x] = s; }
    __syncthreads();
}
// one LM trial's linear solve + oplus by thread 0: 6x6 LDL^T like LinearSolverDense (fails unless positive: LDLT::isPositive)
__device__ __noinline__ void po_trial_thread0(PoShared* S) {
    S->backup = S->pose;
    double M[6][6], d[6], b[6]; int k = 0; bool ok = true;
    for (int a = 0; a < 6; a++) for (int c = a; c < 6; c++) { M[a][c] = S->Hs[k]; M[c][a] = S->Hs[k]; k++; }
    for (int a = 0; a < 6; a++) { M[a][a] += S->lambda; b[a] = S->Hs[21 + a]; }
    for (int j = 0; j < 6 && ok; j++) {
        double dj = M[j][j];
        for (int c = 0; c < j; c++) dj -= M[j][c] * M[j][c] * d[c];
        if (!(dj > 0.0) || !isfinite(dj)) { ok = false; break; }
        d[j] = dj;
        for (int i2 = j + 1; i2 < 6; i2++) { double s = M[i2][j]; for (int c = 0; c < j; c++) s -= M[i2][c] * M[j][c] * d[c]; M[i2][j] = s / dj; }
    }
    double* x = S->x;
    if (ok) {
        for (int i2 = 0; i2 < 6; i2++) { double s = b[i2]; for (int c = 0; c < i2; c++) s -= M[i2][c] * x[c]; x[i2] = s; }
        for (int i2 = 0; i2 < 6; i2++) x[i2] /= d[i2];
        for (int i2 = 5; i2 >= 0; i2--) { double s = x[i2]; for (int c = i2 + 1; c < 6; c++) s -= M[c][i2] * x[c]; x[i2] = s; }
        S->pose = pose_oplus(S->pose, x);
    } else { for (int i2 = 0; i2 < 6; i2++) x[i2] = 0; }
    S->ctrl = ok ? 1 : 0;
}
// classification (src/Optimizer.cpp:149-177): outliers get a fresh error, inliers keep the last computed one; returns #bad
__device__ __noinline__ int po_classify(const PoFrame& F, PoShared* S) {
    int bad = 0;
    const Pose pose = S->pose;
    for (int i = threadIdx.x; i < F.n; i += blockDim.x) {
        const int e = F.beg + i;
        double mx, my, w; const int face = po_obs_face(F, e, mx, my, w);
        if (F.outlier[e]) {
            const double Xw[3] = {(double)F.Xw[3 * e], (double)F.Xw[3 * e + 1], (double)F.Xw[3 * e + 2]};
            double Xc[3], er[2];
            pose_map(pose, Xw, Xc); edge_error(face, F.fc, mx, my, Xc, er);
            F.err[2 * e] = er[0]; F.err[2 * e + 1] = er[1];
        }
        const float chi = (float)(w * (F.err[2 * e] * F.err[2 * e] + F.err[2 * e + 1] * F.err[2 * e + 1]));
        if (chi > 5.991f) { F.outlier[e] = 1; F.level[e] = 1; bad++; } else { F.outlier[e] = 0; F.level[e] = 0; }
    }
    return (int)po_block_sum((double)bad, S);
}

__global__ void __launch_bounds__(256) k_pose_opt(PoseOptArgs A) {
    __shared__ PoShared S;
    const int f = blockIdx.x, tid = threadIdx.x, T = blockDim.x;
    PoFrame F;
    F.Xw = A.Xw; F.kpxy = A.kpxy; F.invSigma2 = A.invSigma2; F.err = A.err; F.level = A.level; F.outlier = A.outlier;
    if (A.offset) { F.beg = A.offset[f]; F.n = A.offset[f + 1] - F.beg; } else { F.beg = f * A.stride; F.n = min(A.count[f], A.stride); } F.faceW = A.faceW; F.faceH = A.faceH; F.fc = A.faceW / 2.0;
    F.delta = huber_delta(); F.dsqr = F.delta * F.delta;
    const int beg = F.beg, n = F.n;
    if (tid == 0) { S.pose0 = pose_from_Tcw32(A.Tcw + 16 * f); S.pose = S.pose0; }
    for (int i = tid; i < n; i += T) { A.outlier[beg + i] = 0; A.level[beg + i] = 0; A.err[2 * (beg + i)] = 0; A.err[2 * (beg + i) + 1] = 0; }
    __syncthreads();
    if (n < 3) { if (tid == 0) { A.inliers[f] = 0; if (A.pose64) pose_to_fp64(S.pose0, A.pose64 + 7 * f); if (A.nlog) A.nlog[f] = 0; } return; }
    int nBadEdges = 0, nRows = 0;
    bool robust = true;
    for (int it = 0; it < 4; it++) {
        if (tid == 0) S.pose = S.pose0;
        __syncthreads();
        int nAct = 0;
        for (int i = tid; i < n; i += T) nAct += A.level[beg + i] == 0;
        nAct = (int)po_block_sum((double)nAct, &S);
        if (nAct > 0) {
            int nBad = 0;
            for (int iter = 0; iter < 10; iter++) {
                double currentChi = po_compute_errors(F, &S, robust);
                const double iniChi = currentChi;
                po_build_system(F, &S, robust);
                if (tid == 0 && iter == 0) {
                    double m = 0; int k = 0;
                    // std::max(fabs(H_jj), m) of computeLambdaInit (optimization_algorithm_levenberg.cpp:176): a NaN diagonal makes m NaN
                    // until a later diagonal replaces it, which fmax would skip
                    for (int a = 0; a < 6; a++) { const double d = fabs(S.Hs[k]); m = d < m ? m : d; k += 6 - a; }
                    S.lambda = 1e-5 * m; S.ni = 2;
                }
                if (iter == 0) nBad = 0;
                __syncthreads();
                double rho = 0; int qmax = 0; bool accepted = false;
                do {
                    if (tid == 0) po_trial_thread0(&S);
                    __syncthreads();
                    const bool ok2 = S.ctrl != 0;
                    double tempChi = po_compute_errors(F, &S, robust);
                    if (!ok2) tempChi = DBL_MAX;
                    double scale = 0;
                    for (int a = 0; a < 6; a++) scale += S.x[a] * (S.lambda * S.x[a] + S.Hs[21 + a]);
                    scale += 1e-3;
                    rho = (currentChi - tempChi) / scale;
                    const bool good = rho > 0 && isfinite(tempChi);
                    __syncthreads();
                    if (tid == 0) {
                        if (good) { const double tr = 2 * rho - 1; double alpha = 1. - tr * tr * tr; alpha = fmin(alpha, 2. / 3.); S.lambda *= fmax(1. / 3., alpha); S.ni = 2; }
                        else { S.lambda *= S.ni; S.ni *= 2; S.pose = S.backup; }
                    }
                    if (good) currentChi = tempChi;
                    accepted |= good;
                    __syncthreads();
                    qmax++;
                } while (rho < 0 && qmax < 10);
                if (A.log && tid == 0) {   // the oracle's IterLog row of this LM iteration
                    double* r = A.log + ((size_t)f * PO_LOG_ROWS + nRows) * 4;
                    r[0] = currentChi; r[1] = S.lambda; r[2] = qmax; r[3] = accepted ? 1 : 0;
                }
                nRows++;
                if (qmax == 10 || rho == 0) break;
                if ((iniChi - currentChi) * 1e3 < iniChi) nBad++; else nBad = 0;
                if (nBad >= 3) break;
            }
        }
        nBadEdges = po_classify(F, &S);
        if (it == 2) robust = false;
        if (n < 10) break;
    }
    if (tid == 0) {
        A.inliers[f] = n - nBadEdges;
        if (A.nlog) A.nlog[f] = nRows;
        pose_to_Tcw32(S.pose, A.Tcw + 16 * f);
        if (A.pose64) pose_to_fp64(S.pose, A.pose64 + 7 * f);
    }
}

}  // namespace cslam

using namespace cslam;

// Both entry points: one CTA per frame on the optimizer's stream; the per-correspondence errors and levels are arena scratch of the call.
static int launch_pose_opt(cslam_optimizer* o, int nframes, size_t nCorr, PoseOptArgs A) {
    int rc;
    if ((rc = o->arena.take(&A.err, nCorr * 2)) || (rc = o->arena.take(&A.level, nCorr))) return rc;
    k_pose_opt<<<nframes, 256, 0, o->stream>>>(A); o->launches++;
    CSLAM_CUDA(cudaGetLastError());
    return CSLAM_OK;
}

// Both host entry points: every key point of a frame the optimizer runs on (>= 3 correspondences) must lie on a face, checked before anything
// is enqueued. The reference calls exit() in computeError there (include/g2o_cubemap_vertices_edges.h:52-58); the kernel would take it as the
// lower face. log / nlog (nframes x PO_LOG_ROWS x 4, nframes) may be null.
static int pose_opt_host(const char* fn, cslam_optimizer* o, int nframes, const int32_t* offset, float* Tcw, const float* Xw, const float* kp_xy,
                         const float* inv_sigma2, int face_w, int face_h, uint8_t* outlier, int32_t* inliers, double* pose_fp64, double* log, int32_t* nlog) {
    if (!o || nframes <= 0 || !offset || !Tcw || !inliers) { set_error("%s: bad argument", fn); return CSLAM_E_BADARG; }
    if (face_w != face_h || face_w <= 0) { set_error("cube faces must be square"); return CSLAM_E_BADARG; }
    for (int f = 0; f < nframes; f++) {
        if (offset[f + 1] - offset[f] < 3) continue;
        for (int e = offset[f]; e < offset[f + 1]; e++)
            if (face_of_pixel_f(kp_xy[2 * e], kp_xy[2 * e + 1], face_w, face_h) < 0) {
                set_error("%s: frame %d, correspondence %d: keypoint (%g,%g) is on no cube face (the reference calls exit() here)", fn, f, e - offset[f],
                          kp_xy[2 * e], kp_xy[2 * e + 1]);
                return CSLAM_E_BADARG;
            }
    }
    CSLAM_CUDA(cudaSetDevice(o->device));
    o->arena.reset();
    const int n = offset[nframes];
    PoseOptArgs A; std::memset(&A, 0, sizeof(A));
    int* d_off; float *d_T, *d_X, *d_kp, *d_w; uint8_t* d_out; int32_t* d_inl; double* d_p64;
    double* d_log = nullptr; int32_t* d_nlog = nullptr;
    int rc;
    if ((rc = o->arena.take(&d_off, nframes + 1)) || (rc = o->arena.take(&d_T, (size_t)nframes * 16)) || (rc = o->arena.take(&d_X, (size_t)n * 3)) || (rc = o->arena.take(&d_kp, (size_t)n * 2)) ||
        (rc = o->arena.take(&d_w, n)) || (rc = o->arena.take(&d_out, n)) || (rc = o->arena.take(&d_inl, nframes)) || (rc = o->arena.take(&d_p64, (size_t)nframes * 7))) return rc;
    // rows past a frame's count read 0
    if (log && ((rc = o->arena.take(&d_log, (size_t)nframes * PO_LOG_ROWS * 4, true)) || (rc = o->arena.take(&d_nlog, nframes)))) return rc;
    CSLAM_CUDA(cudaMemcpyAsync(d_off, offset, (nframes + 1) * 4, cudaMemcpyHostToDevice, o->stream));
    CSLAM_CUDA(cudaMemcpyAsync(d_T, Tcw, (size_t)nframes * 64, cudaMemcpyHostToDevice, o->stream));
    if (n) {
        CSLAM_CUDA(cudaMemcpyAsync(d_X, Xw, (size_t)n * 12, cudaMemcpyHostToDevice, o->stream));
        CSLAM_CUDA(cudaMemcpyAsync(d_kp, kp_xy, (size_t)n * 8, cudaMemcpyHostToDevice, o->stream));
        CSLAM_CUDA(cudaMemcpyAsync(d_w, inv_sigma2, (size_t)n * 4, cudaMemcpyHostToDevice, o->stream));
    }
    A.offset = d_off; A.Tcw = d_T; A.Xw = d_X; A.kpxy = d_kp; A.invSigma2 = d_w; A.faceW = face_w; A.faceH = face_h; A.outlier = d_out; A.inliers = d_inl;
    A.pose64 = d_p64; A.log = d_log; A.nlog = d_nlog;
    if ((rc = launch_pose_opt(o, nframes, n, A))) return rc;
    // frames with < 3 correspondences are returned untouched (src/Optimizer.cpp:133-134): copy back only the others
    std::vector<float> Tout((size_t)nframes * 16);
    CSLAM_CUDA(cudaMemcpyAsync(Tout.data(), d_T, Tout.size() * 4, cudaMemcpyDeviceToHost, o->stream));
    if (n && outlier) CSLAM_CUDA(cudaMemcpyAsync(outlier, d_out, n, cudaMemcpyDeviceToHost, o->stream));
    CSLAM_CUDA(cudaMemcpyAsync(inliers, d_inl, nframes * 4, cudaMemcpyDeviceToHost, o->stream));
    if (pose_fp64) CSLAM_CUDA(cudaMemcpyAsync(pose_fp64, d_p64, (size_t)nframes * 56, cudaMemcpyDeviceToHost, o->stream));
    if (log) {
        CSLAM_CUDA(cudaMemcpyAsync(log, d_log, (size_t)nframes * PO_LOG_ROWS * 4 * sizeof(double), cudaMemcpyDeviceToHost, o->stream));
        CSLAM_CUDA(cudaMemcpyAsync(nlog, d_nlog, (size_t)nframes * 4, cudaMemcpyDeviceToHost, o->stream));
    }
    if ((rc = o->sync())) return rc;
    for (int f = 0; f < nframes; f++) if (offset[f + 1] - offset[f] >= 3) std::memcpy(Tcw + 16 * f, Tout.data() + 16 * f, 64);
    return CSLAM_OK;
}

extern "C" int cslam_pose_optimization(cslam_optimizer* o, int nframes, const int32_t* offset, float* Tcw, const float* Xw, const float* kp_xy, const float* inv_sigma2,
                                       int face_w, int face_h, uint8_t* outlier, int32_t* inliers, double* pose_fp64) {
    return pose_opt_host("cslam_pose_optimization", o, nframes, offset, Tcw, Xw, kp_xy, inv_sigma2, face_w, face_h, outlier, inliers, pose_fp64, nullptr, nullptr);
}
extern "C" int cslam_pose_optimization_log(cslam_optimizer* o, int nframes, const int32_t* offset, float* Tcw, const float* Xw, const float* kp_xy,
                                           const float* inv_sigma2, int face_w, int face_h, uint8_t* outlier, int32_t* inliers, double* pose_fp64, double* log,
                                           int32_t* nlog) {
    if (!log || !nlog) { set_error("cslam_pose_optimization_log: bad argument"); return CSLAM_E_BADARG; }
    return pose_opt_host("cslam_pose_optimization_log", o, nframes, offset, Tcw, Xw, kp_xy, inv_sigma2, face_w, face_h, outlier, inliers, pose_fp64, log, nlog);
}

// Device-resident variant for pipelines (config 5): fixed stride, per-frame counts, all pointers on the device, asynchronous on the optimizer's stream.
extern "C" int cslam_pose_optimization_dev(cslam_optimizer* o, int nframes, int stride, const int32_t* count, float* Tcw, const float* Xw, const float* kp_xy, const float* inv_sigma2,
                                           int face_w, int face_h, uint8_t* outlier, int32_t* inliers) {
    if (!o || nframes <= 0 || stride <= 0 || !count || !Tcw || !Xw || !kp_xy || !inv_sigma2 || !outlier || !inliers) { set_error("cslam_pose_optimization_dev: bad argument"); return CSLAM_E_BADARG; }
    if (face_w != face_h || face_w <= 0) { set_error("cube faces must be square"); return CSLAM_E_BADARG; }
    CSLAM_CUDA(cudaSetDevice(o->device));
    o->arena.reset();
    PoseOptArgs A; std::memset(&A, 0, sizeof(A));
    A.count = count; A.stride = stride; A.Tcw = Tcw; A.Xw = Xw; A.kpxy = kp_xy; A.invSigma2 = inv_sigma2; A.faceW = face_w; A.faceH = face_h;
    A.outlier = outlier; A.inliers = inliers;
    return launch_pose_opt(o, nframes, (size_t)nframes * stride, A);
}
extern "C" void* cslam_optimizer_stream(const cslam_optimizer* o) { return o ? (void*)o->stream : nullptr; }
extern "C" int cslam_optimizer_sync(cslam_optimizer* o) { return o ? o->sync() : CSLAM_E_BADARG; }

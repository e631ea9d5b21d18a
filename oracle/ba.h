// ORACLE (test infrastructure, not product code).
// CPU restatement (fp64, flat arrays) of the reference's bundle-adjustment path:
//   Optimizer::PoseOptimization            src/Optimizer.cpp:48-190
//   Optimizer::LocalBundleAdjustment       src/Optimizer.cpp:192-451 (graph already collected: the caller passes
//                                          local KFs + fixed KFs, local MapPoints and their observations)
//   EdgeSE3ProjectXYZMultiPinhole[OnlyPose] include/g2o_cubemap_vertices_edges.h:43-134,
//                                          src/g2o_cubemap_vertices_edges.cpp:61-124,164-233
//   g2o slice: optimization_algorithm_levenberg.cpp:61-189, block_solver.hpp:354-604,
//              base_binary_edge.hpp:55-120, base_unary_edge.hpp:43-72, robust_kernel_impl.cpp:78-91,
//              base_edge.h:58-61,96-102, se3quat.h:56-110,217-257,280-285, types_six_dof_expmap.h:73-76,
//              types_sba.h:52-56, sparse_optimizer.cpp:100-114,166-267,354-435
//   Converter (float32 boundary)           src/Converter.cpp:41-120
// Eigen (un-vendored, >=3.1) supplies Quaterniond(R), toRotationMatrix, 3x3 inverse and the LDLT solves; the
// standard algorithms are restated here. No reference test pins these numbers: "parity unpinned"; the oracle
// is cross-checked against a numpy fp64 dense Gauss-Newton step in tests/test_oracle_ba.py.
#pragma once
#include <cfloat>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <vector>
#include "cam_model.h"

namespace orc {

struct Quat { double x, y, z, w; };
struct SE3 { Quat r; double t[3]; };

static inline void quat_normalize_rotation(Quat& q) {  // se3quat.h:280-285
    if (q.w < 0) { q.x = -q.x; q.y = -q.y; q.z = -q.z; q.w = -q.w; }
    double n = std::sqrt(q.x * q.x + q.y * q.y + q.z * q.z + q.w * q.w);
    q.x /= n; q.y /= n; q.z /= n; q.w /= n;
}
static inline Quat quat_from_matrix(const double m[3][3]) {  // Eigen quaternionbase_assign_impl<Matrix3>
    Quat q; double t = m[0][0] + m[1][1] + m[2][2];
    if (t > 0) {
        t = std::sqrt(t + 1.0); q.w = 0.5 * t; t = 0.5 / t;
        q.x = (m[2][1] - m[1][2]) * t; q.y = (m[0][2] - m[2][0]) * t; q.z = (m[1][0] - m[0][1]) * t;
    } else {
        int i = 0; if (m[1][1] > m[0][0]) i = 1; if (m[2][2] > m[i][i]) i = 2;
        int j = (i + 1) % 3, k = (j + 1) % 3;
        t = std::sqrt(m[i][i] - m[j][j] - m[k][k] + 1.0);
        double v[3]; v[i] = 0.5 * t; t = 0.5 / t;
        q.w = (m[k][j] - m[j][k]) * t; v[j] = (m[j][i] + m[i][j]) * t; v[k] = (m[k][i] + m[i][k]) * t;
        q.x = v[0]; q.y = v[1]; q.z = v[2];
    }
    return q;
}
static inline void quat_to_matrix(const Quat& q, double R[3][3]) {  // Eigen toRotationMatrix
    const double tx = 2 * q.x, ty = 2 * q.y, tz = 2 * q.z;
    const double twx = tx * q.w, twy = ty * q.w, twz = tz * q.w;
    const double txx = tx * q.x, txy = ty * q.x, txz = tz * q.x;
    const double tyy = ty * q.y, tyz = tz * q.y, tzz = tz * q.z;
    R[0][0] = 1 - (tyy + tzz); R[0][1] = txy - twz; R[0][2] = txz + twy;
    R[1][0] = txy + twz; R[1][1] = 1 - (txx + tzz); R[1][2] = tyz - twx;
    R[2][0] = txz - twy; R[2][1] = tyz + twx; R[2][2] = 1 - (txx + tyy);
}
static inline void quat_rotate(const Quat& q, const double v[3], double out[3]) {  // Eigen _transformVector
    double uv[3] = {q.y * v[2] - q.z * v[1], q.z * v[0] - q.x * v[2], q.x * v[1] - q.y * v[0]};
    uv[0] += uv[0]; uv[1] += uv[1]; uv[2] += uv[2];
    out[0] = v[0] + q.w * uv[0] + (q.y * uv[2] - q.z * uv[1]);
    out[1] = v[1] + q.w * uv[1] + (q.z * uv[0] - q.x * uv[2]);
    out[2] = v[2] + q.w * uv[2] + (q.x * uv[1] - q.y * uv[0]);
}
static inline Quat quat_mul(const Quat& a, const Quat& b) {
    Quat r;
    r.w = a.w * b.w - a.x * b.x - a.y * b.y - a.z * b.z;
    r.x = a.w * b.x + a.x * b.w + a.y * b.z - a.z * b.y;
    r.y = a.w * b.y + a.y * b.w + a.z * b.x - a.x * b.z;
    r.z = a.w * b.z + a.z * b.w + a.x * b.y - a.y * b.x;
    return r;
}
static inline void se3_map(const SE3& T, const double X[3], double out[3]) {
    quat_rotate(T.r, X, out); out[0] += T.t[0]; out[1] += T.t[1]; out[2] += T.t[2];
}
// Converter::toSE3Quat (src/Converter.cpp:41-51): float32 4x4 row-major -> SE3Quat(R,t)
static inline SE3 se3_from_Tcw32(const float* T) {
    double R[3][3];
    for (int i = 0; i < 3; i++) for (int j = 0; j < 3; j++) R[i][j] = (double)T[i * 4 + j];
    SE3 s; s.r = quat_from_matrix(R); quat_normalize_rotation(s.r);
    for (int i = 0; i < 3; i++) s.t[i] = (double)T[i * 4 + 3];
    return s;
}
static inline void se3_to_Tcw32(const SE3& s, float* T) {  // Converter::toCvMat(SE3Quat)
    double R[3][3]; quat_to_matrix(s.r, R);
    for (int i = 0; i < 3; i++) { for (int j = 0; j < 3; j++) T[i * 4 + j] = (float)R[i][j]; T[i * 4 + 3] = (float)s.t[i]; }
    T[12] = 0; T[13] = 0; T[14] = 0; T[15] = 1;
}
// SE3Quat::exp (se3quat.h:223-257), update = [omega, upsilon]
static inline SE3 se3_exp(const double* u) {
    const double w[3] = {u[0], u[1], u[2]}, up[3] = {u[3], u[4], u[5]};
    const double theta = std::sqrt(w[0] * w[0] + w[1] * w[1] + w[2] * w[2]);
    double O[3][3] = {{0, -w[2], w[1]}, {w[2], 0, -w[0]}, {-w[1], w[0], 0}};
    double O2[3][3];
    for (int i = 0; i < 3; i++) for (int j = 0; j < 3; j++) { double s = 0; for (int k = 0; k < 3; k++) s += O[i][k] * O[k][j]; O2[i][j] = s; }
    double R[3][3], V[3][3];
    if (theta < 0.00001) {
        for (int i = 0; i < 3; i++) for (int j = 0; j < 3; j++) { R[i][j] = (i == j) + O[i][j] + O2[i][j]; V[i][j] = R[i][j]; }
    } else {
        const double a = std::sin(theta) / theta, b = (1 - std::cos(theta)) / (theta * theta);
        const double c = (theta - std::sin(theta)) / std::pow(theta, 3);
        for (int i = 0; i < 3; i++) for (int j = 0; j < 3; j++) {
            R[i][j] = (i == j) + a * O[i][j] + b * O2[i][j];
            V[i][j] = (i == j) + b * O[i][j] + c * O2[i][j];
        }
    }
    SE3 s; s.r = quat_from_matrix(R);
    for (int i = 0; i < 3; i++) s.t[i] = V[i][0] * up[0] + V[i][1] * up[1] + V[i][2] * up[2];
    quat_normalize_rotation(s.r);
    return s;
}
static inline SE3 se3_mul(const SE3& a, const SE3& b) {  // se3quat.h:104-110
    SE3 r; double rt[3]; quat_rotate(a.r, b.t, rt);
    for (int i = 0; i < 3; i++) r.t[i] = a.t[i] + rt[i];
    r.r = quat_mul(a.r, b.r); quat_normalize_rotation(r.r);
    return r;
}

static inline void face_R_local(int face, double R[3][3]) {  // src/g2o_cubemap_vertices_edges.cpp:173-198
    static const double T[5][9] = {{1, 0, 0, 0, 1, 0, 0, 0, 1}, {0, 0, 1, 0, 1, 0, -1, 0, 0}, {0, 0, -1, 0, 1, 0, 1, 0, 0},
                                   {1, 0, 0, 0, 0, 1, 0, -1, 0}, {1, 0, 0, 0, 0, -1, 0, 1, 0}};
    for (int i = 0; i < 9; i++) R[i / 3][i % 3] = T[face][i];
}

struct EdgeObs { double mx, my, w; int face; };  // measurement in face, information scalar, face id
static inline EdgeObs make_obs(float kx, float ky, float invSigma2, int W, int H) {
    EdgeObs o; o.face = face_in_cubemap_f(kx, ky, W, H);
    const int i = (int)std::floor((double)kx / W), j = (int)std::floor((double)ky / H);  // GetPosInFace<double>
    o.mx = (double)kx - i * W; o.my = (double)ky - j * H; o.w = (double)invSigma2;
    return o;
}
// computeError: e = m_inface - multipinhole_project(T.map(X))  (fp64 -> float3 -> fp64 -> float)
static inline void edge_error(const EdgeObs& o, double f, const double Xc[3], double e[2]) {
    float u, v;
    rays_to_target_face(f, f, f, f, (float)Xc[0], (float)Xc[1], (float)Xc[2], o.face, u, v);
    e[0] = o.mx - (double)u; e[1] = o.my - (double)v;
}
// linearizeOplus: Jpose 2x6 (omega, upsilon), Jpt 2x3 (needs R of the pose)
static inline void edge_jacobians(int face, double f, const double Xc[3], const double Rcw[3][3], double Jp[2][6], double Jx[2][3]) {
    double Rl[3][3]; face_R_local(face, Rl);
    double L[3];
    for (int i = 0; i < 3; i++) L[i] = Rl[i][0] * Xc[0] + Rl[i][1] * Xc[1] + Rl[i][2] * Xc[2];
    double D[2][3] = {{f / L[2], 0, -f * L[0] / (L[2] * L[2])}, {0, f / L[2], -f * L[1] / (L[2] * L[2])}};
    double G[2][3];
    for (int i = 0; i < 2; i++) for (int j = 0; j < 3; j++) G[i][j] = -1.0 * (D[i][0] * Rl[0][j] + D[i][1] * Rl[1][j] + D[i][2] * Rl[2][j]);
    const double nS[3][3] = {{0, Xc[2], -Xc[1]}, {-Xc[2], 0, Xc[0]}, {Xc[1], -Xc[0], 0}};
    for (int i = 0; i < 2; i++) for (int j = 0; j < 3; j++) {
        Jp[i][j] = G[i][0] * nS[0][j] + G[i][1] * nS[1][j] + G[i][2] * nS[2][j];
        Jp[i][j + 3] = G[i][j];
        if (Rcw) Jx[i][j] = G[i][0] * Rcw[0][j] + G[i][1] * Rcw[1][j] + G[i][2] * Rcw[2][j];
    }
}
struct Huber { double delta, dsqr; };
static inline Huber make_huber() { Huber h; const float d = (float)std::sqrt(5.991); h.delta = (double)d; h.dsqr = h.delta * h.delta; return h; }
static inline void huber(const Huber& h, double e, double& rho0, double& rho1) {
    if (e <= h.dsqr) { rho0 = e; rho1 = 1.0; }
    else { const double s = std::sqrt(e); rho0 = 2 * s * h.delta - h.dsqr; rho1 = h.delta / s; }
}

// dense symmetric solve A x = b via LDL^T without pivoting (upper/lower both filled). Returns false on a zero /
// non-finite pivot (SimplicialLDLT's NumericalIssue) or, when requirePositive, on a negative pivot (LDLT::isPositive).
static inline bool ldlt_solve(std::vector<double> A, int n, const double* b, double* x, bool requirePositive) {
    std::vector<double> d(n);
    for (int j = 0; j < n; j++) {
        double dj = A[(size_t)j * n + j];
        for (int k = 0; k < j; k++) dj -= A[(size_t)j * n + k] * A[(size_t)j * n + k] * d[k];
        if (dj == 0.0 || !std::isfinite(dj)) return false;
        if (requirePositive && dj < 0) return false;
        d[j] = dj;
        for (int i = j + 1; i < n; i++) {
            double s = A[(size_t)i * n + j];
            for (int k = 0; k < j; k++) s -= A[(size_t)i * n + k] * A[(size_t)j * n + k] * d[k];
            A[(size_t)i * n + j] = s / dj;
        }
    }
    for (int i = 0; i < n; i++) { double s = b[i]; for (int k = 0; k < i; k++) s -= A[(size_t)i * n + k] * x[k]; x[i] = s; }
    for (int i = 0; i < n; i++) x[i] /= d[i];
    for (int i = n - 1; i >= 0; i--) { double s = x[i]; for (int k = i + 1; k < n; k++) s -= A[(size_t)k * n + i] * x[k]; x[i] = s; }
    return true;
}
static inline void inv3(const double* D, double* Di) {  // Eigen 3x3 inverse (cofactors / determinant)
    const double c00 = D[4] * D[8] - D[5] * D[7], c01 = D[5] * D[6] - D[3] * D[8], c02 = D[3] * D[7] - D[4] * D[6];
    const double det = D[0] * c00 + D[1] * c01 + D[2] * c02, id = 1.0 / det;
    Di[0] = c00 * id; Di[1] = (D[2] * D[7] - D[1] * D[8]) * id; Di[2] = (D[1] * D[5] - D[2] * D[4]) * id;
    Di[3] = c01 * id; Di[4] = (D[0] * D[8] - D[2] * D[6]) * id; Di[5] = (D[2] * D[3] - D[0] * D[5]) * id;
    Di[6] = c02 * id; Di[7] = (D[1] * D[6] - D[0] * D[7]) * id; Di[8] = (D[0] * D[4] - D[1] * D[3]) * id;
}

struct IterLog { double chi2, lambda; int trials; int accepted; };

// ------------------------------------------------------------------------------------------------ Local BA
struct LocalBA {
    int nKF, nMP, nE, W, H; double f;
    std::vector<SE3> pose; std::vector<uint8_t> fixed;
    std::vector<double> X;                       // nMP*3
    std::vector<int> eMP, eKF; std::vector<EdgeObs> obs;
    std::vector<double> err;                     // nE*2, "last computed" errors (g2o edge::_error)
    std::vector<int> level;                      // 0 active / 1 outlier
    bool robust = true; Huber hub = make_huber();
    const volatile uint8_t* stopFlag = nullptr;
    int stopAfterTrials = 0, trialsDone = 0;     // test hook: behave as if *stopFlag became non-zero right after trial k of the call (0 = off)
    std::vector<IterLog> log;
    std::vector<int> logRound, logStop;          // per log row: round (0, 1), why the iteration ended its round (0 none, 1 qmax == 10, 2 rho == 0, 3 nBad >= 3, 4 stop flag)
    // active set
    std::vector<int> poseIdx, ptIdx, actE; int nP = 0, nL = 0;
    // linear system
    std::vector<double> Hpp, Hll, Hpl, bp, bl, x; double lambda = -1, ni = 2; int nBad = 0;

    bool terminate() const { return (stopFlag && *stopFlag != 0) || (stopAfterTrials > 0 && trialsDone >= stopAfterTrials); }
    double chi2(int e) const { return obs[e].w * (err[2 * e] * err[2 * e] + err[2 * e + 1] * err[2 * e + 1]); }

    void initializeOptimization() {  // sparse_optimizer.cpp:206-267 + buildIndexMapping :166-190
        actE.clear(); poseIdx.assign(nKF, -1); ptIdx.assign(nMP, -1);
        std::vector<uint8_t> pAct(nKF, 0), lAct(nMP, 0);
        for (int e = 0; e < nE; e++) if (level[e] == 0) { actE.push_back(e); pAct[eKF[e]] = 1; lAct[eMP[e]] = 1; }
        nP = 0; for (int k = 0; k < nKF; k++) if (pAct[k] && !fixed[k]) poseIdx[k] = nP++;
        nL = 0; for (int l = 0; l < nMP; l++) if (lAct[l]) ptIdx[l] = nL++;
    }
    void computeActiveErrors() {
        for (int e : actE) { double Xc[3]; se3_map(pose[eKF[e]], &X[3 * eMP[e]], Xc); edge_error(obs[e], f, Xc, &err[2 * e]); }
    }
    double activeRobustChi2() const {
        double chi = 0;
        for (int e : actE) { double c = chi2(e); if (robust) { double r0, r1; huber(hub, c, r0, r1); chi += r0; } else chi += c; }
        return chi;
    }
    void buildSystem() {
        Hpp.assign((size_t)nP * 36, 0); Hll.assign((size_t)nL * 9, 0); Hpl.assign(actE.size() * 18, 0);
        bp.assign((size_t)nP * 6, 0); bl.assign((size_t)nL * 3, 0);
        for (size_t a = 0; a < actE.size(); a++) {
            const int e = actE[a], k = eKF[e], l = eMP[e], pi = poseIdx[k], li = ptIdx[l];
            double Xc[3], R[3][3], Jp[2][6], Jx[2][3];
            se3_map(pose[k], &X[3 * l], Xc); quat_to_matrix(pose[k].r, R);
            edge_jacobians(obs[e].face, f, Xc, R, Jp, Jx);
            double rho1 = 1.0;
            if (robust) { double r0; huber(hub, chi2(e), r0, rho1); }
            const double w = rho1 * obs[e].w;
            const double r[2] = {-w * err[2 * e], -w * err[2 * e + 1]};   // rho1 * (-omega * e)
            for (int i = 0; i < 3; i++) {
                bl[3 * li + i] += Jx[0][i] * r[0] + Jx[1][i] * r[1];
                for (int j = 0; j < 3; j++) Hll[9 * li + 3 * i + j] += w * (Jx[0][i] * Jx[0][j] + Jx[1][i] * Jx[1][j]);
            }
            if (pi >= 0) {
                for (int i = 0; i < 6; i++) {
                    bp[6 * pi + i] += Jp[0][i] * r[0] + Jp[1][i] * r[1];
                    for (int j = 0; j < 6; j++) Hpp[36 * pi + 6 * i + j] += w * (Jp[0][i] * Jp[0][j] + Jp[1][i] * Jp[1][j]);
                    for (int j = 0; j < 3; j++) Hpl[18 * a + 3 * i + j] += w * (Jp[0][i] * Jx[0][j] + Jp[1][i] * Jx[1][j]);
                }
            }
        }
    }
    double computeLambdaInit() const {   // std::max(fabs(H_jj), m) in index-mapping order: a NaN diagonal resets the maximum (last one: NaN)
        double m = 0;
        for (int p = 0; p < nP; p++) for (int j = 0; j < 6; j++) m = std::max(std::fabs(Hpp[36 * p + 7 * j]), m);
        for (int l = 0; l < nL; l++) for (int j = 0; j < 3; j++) m = std::max(std::fabs(Hll[9 * l + 4 * j]), m);
        return 1e-5 * m;
    }
    bool solve() {  // block_solver.hpp:354-486 with lambda already folded in by the caller's copies
        const int n = 6 * nP;
        std::vector<double> S((size_t)n * n, 0), g(bp), Dinv((size_t)nL * 9);
        for (int p = 0; p < nP; p++) for (int i = 0; i < 6; i++) for (int j = 0; j < 6; j++) {
            double v = Hpp[36 * p + 6 * i + j]; if (i == j) v += lambda; S[(size_t)(6 * p + i) * n + 6 * p + j] = v; }
        for (int l = 0; l < nL; l++) { double D[9]; for (int i = 0; i < 9; i++) D[i] = Hll[9 * l + i]; D[0] += lambda; D[4] += lambda; D[8] += lambda; inv3(D, &Dinv[9 * l]); }
        // group active edges by landmark
        std::vector<std::vector<int>> byL(nL);
        for (size_t a = 0; a < actE.size(); a++) if (poseIdx[eKF[actE[a]]] >= 0) byL[ptIdx[eMP[actE[a]]]].push_back((int)a);
        for (int l = 0; l < nL; l++) {
            const double* Di = &Dinv[9 * l];
            double db[3]; for (int i = 0; i < 3; i++) db[i] = Di[3 * i] * bl[3 * l] + Di[3 * i + 1] * bl[3 * l + 1] + Di[3 * i + 2] * bl[3 * l + 2];
            for (int a1 : byL[l]) {
                const int p1 = poseIdx[eKF[actE[a1]]]; const double* B1 = &Hpl[18 * (size_t)a1];
                double BD[18];
                for (int i = 0; i < 6; i++) for (int j = 0; j < 3; j++) BD[3 * i + j] = B1[3 * i] * Di[j] + B1[3 * i + 1] * Di[3 + j] + B1[3 * i + 2] * Di[6 + j];
                for (int i = 0; i < 6; i++) g[6 * p1 + i] -= B1[3 * i] * db[0] + B1[3 * i + 1] * db[1] + B1[3 * i + 2] * db[2];
                for (int a2 : byL[l]) {
                    const int p2 = poseIdx[eKF[actE[a2]]]; const double* B2 = &Hpl[18 * (size_t)a2];
                    for (int i = 0; i < 6; i++) for (int j = 0; j < 6; j++)
                        S[(size_t)(6 * p1 + i) * n + 6 * p2 + j] -= BD[3 * i] * B2[3 * j] + BD[3 * i + 1] * B2[3 * j + 1] + BD[3 * i + 2] * B2[3 * j + 2];
                }
            }
        }
        x.assign((size_t)n + 3 * nL, 0);
        if (n > 0 && !ldlt_solve(S, n, g.data(), x.data(), false)) return false;
        std::vector<double> cl(bl);
        for (size_t a = 0; a < actE.size(); a++) {
            const int p = poseIdx[eKF[actE[a]]]; if (p < 0) continue;
            const int l = ptIdx[eMP[actE[a]]]; const double* B = &Hpl[18 * a];
            for (int j = 0; j < 3; j++) { double s = 0; for (int i = 0; i < 6; i++) s += B[3 * i + j] * x[6 * p + i]; cl[3 * l + j] -= s; }
        }
        for (int l = 0; l < nL; l++) for (int i = 0; i < 3; i++)
            x[n + 3 * l + i] = Dinv[9 * l + 3 * i] * cl[3 * l] + Dinv[9 * l + 3 * i + 1] * cl[3 * l + 1] + Dinv[9 * l + 3 * i + 2] * cl[3 * l + 2];
        return true;
    }
    void update() {
        for (int k = 0; k < nKF; k++) if (poseIdx[k] >= 0) pose[k] = se3_mul(se3_exp(&x[6 * poseIdx[k]]), pose[k]);
        for (int l = 0; l < nMP; l++) if (ptIdx[l] >= 0) for (int i = 0; i < 3; i++) X[3 * l + i] += x[6 * nP + 3 * ptIdx[l] + i];
    }
    // OptimizationAlgorithmLevenberg::solve (one LM iteration). returns 0 OK, 1 Terminate
    int lmIteration(int iteration) {
        computeActiveErrors();
        double currentChi = activeRobustChi2(), tempChi = currentChi; const double iniChi = currentChi;
        buildSystem();
        if (iteration == 0) { lambda = computeLambdaInit(); ni = 2; nBad = 0; }
        double rho = 0; int qmax = 0; int accepted = 0;
        do {
            std::vector<SE3> poseBackup = pose; std::vector<double> Xbackup = X;   // push
            bool ok2 = solve();
            update();
            computeActiveErrors();
            tempChi = activeRobustChi2();
            if (!ok2) tempChi = DBL_MAX;
            rho = currentChi - tempChi;
            double scale = 0;
            for (int j = 0; j < 6 * nP; j++) scale += x[j] * (lambda * x[j] + bp[j]);
            for (int j = 0; j < 3 * nL; j++) scale += x[6 * nP + j] * (lambda * x[6 * nP + j] + bl[j]);
            scale += 1e-3;
            rho /= scale;
            if (rho > 0 && std::isfinite(tempChi)) {
                double alpha = 1. - std::pow((2 * rho - 1), 3);
                alpha = std::min(alpha, 2. / 3.);
                lambda *= std::max(1. / 3., alpha); ni = 2; currentChi = tempChi; accepted = 1;
            } else { lambda *= ni; ni *= 2; pose = poseBackup; X = Xbackup; }   // pop
            qmax++; trialsDone++;
        } while (rho < 0 && qmax < 10 && !terminate());
        log.push_back({currentChi, lambda, qmax, accepted}); logStop.push_back(0);
        if (qmax == 10 || rho == 0) { logStop.back() = qmax == 10 ? 1 : 2; return 1; }
        if ((iniChi - currentChi) * 1e3 < iniChi) nBad++; else nBad = 0;
        if (nBad >= 3) { logStop.back() = 3; return 1; }
        if (terminate()) logStop.back() = 4;
        return 0;
    }
    int optimize(int iterations) {  // sparse_optimizer.cpp:354-419
        if (nP + nL == 0) return -1;
        int n = 0; bool ok = true;
        for (int i = 0; i < iterations && !terminate() && ok; i++) { ok = (lmIteration(i) == 0); n++; }
        return n;
    }
    bool depthPositive(int e) const { double Xc[3]; se3_map(pose[eKF[e]], &X[3 * eMP[e]], Xc); return Xc[2] > 0.0; }
    // src/Optimizer.cpp:359-416 ; outlier[e]=1 for observations the reference would erase
    void run(uint8_t* outlier, int its1 = 5, int its2 = 10) {
        err.assign((size_t)nE * 2, 0); level.assign(nE, 0); robust = true; log.clear(); logRound.clear(); logStop.clear(); trialsDone = 0;
        for (int e = 0; e < nE; e++) outlier[e] = 0;
        if (terminate()) return;
        initializeOptimization(); optimize(its1);
        logRound.resize(log.size(), 0);
        bool bDoMore = !terminate();
        if (bDoMore) {
            for (int e = 0; e < nE; e++) if (chi2(e) > 5.991 || !depthPositive(e)) level[e] = 1;
            robust = false;
            initializeOptimization(); optimize(its2);
            logRound.resize(log.size(), 1);
        }
        for (int e = 0; e < nE; e++) if (chi2(e) > 5.991 || !depthPositive(e)) outlier[e] = 1;
    }
};

// ------------------------------------------------------------------------------------------------ PoseOptimization
struct PoseOpt {
    int n, W, H; double f;
    SE3 pose0, pose;
    std::vector<double> Xw; std::vector<EdgeObs> obs; std::vector<double> err; std::vector<int> level;
    bool robust = true; Huber hub = make_huber();
    std::vector<int> actE; double lambda = -1, ni = 2; int nBad = 0;
    double Hm[36], b[6], x[6];
    std::vector<IterLog> log;
    std::vector<int> logRound, logStop;          // per log row: round, why the iteration ended its round (0 none, 1 qmax == 10, 2 rho == 0, 3 nBad >= 3)
    std::vector<uint8_t> roundOutlier;           // 4 x n: the outlier flags after each round's classification
    double chi2(int e) const { return obs[e].w * (err[2 * e] * err[2 * e] + err[2 * e + 1] * err[2 * e + 1]); }
    void computeError(int e) { double Xc[3]; se3_map(pose, &Xw[3 * e], Xc); edge_error(obs[e], f, Xc, &err[2 * e]); }
    void computeActiveErrors() { for (int e : actE) computeError(e); }
    double activeRobustChi2() const {
        double chi = 0; for (int e : actE) { double c = chi2(e); if (robust) { double r0, r1; huber(hub, c, r0, r1); chi += r0; } else chi += c; } return chi;
    }
    void buildSystem() {
        std::memset(Hm, 0, sizeof(Hm)); std::memset(b, 0, sizeof(b));
        for (int e : actE) {
            double Xc[3], Jp[2][6]; se3_map(pose, &Xw[3 * e], Xc); edge_jacobians(obs[e].face, f, Xc, nullptr, Jp, nullptr);
            double rho1 = 1.0; if (robust) { double r0; huber(hub, chi2(e), r0, rho1); }
            const double w = obs[e].w;
            for (int i = 0; i < 6; i++) {
                b[i] -= rho1 * (Jp[0][i] * w * err[2 * e] + Jp[1][i] * w * err[2 * e + 1]);
                for (int j = 0; j < 6; j++) Hm[6 * i + j] += (rho1 * w) * (Jp[0][i] * Jp[0][j] + Jp[1][i] * Jp[1][j]);
            }
        }
    }
    int lmIteration(int iteration) {
        computeActiveErrors();
        double currentChi = activeRobustChi2(), tempChi = currentChi; const double iniChi = currentChi;
        buildSystem();
        if (iteration == 0) { double m = 0; for (int j = 0; j < 6; j++) m = std::max(std::fabs(Hm[7 * j]), m); lambda = 1e-5 * m; ni = 2; nBad = 0; }
        double rho = 0; int qmax = 0, accepted = 0;
        do {
            SE3 backup = pose;
            std::vector<double> A(Hm, Hm + 36); for (int j = 0; j < 6; j++) A[7 * j] += lambda;
            bool ok2 = ldlt_solve(A, 6, b, x, true);
            pose = se3_mul(se3_exp(x), pose);
            computeActiveErrors(); tempChi = activeRobustChi2();
            if (!ok2) tempChi = DBL_MAX;
            rho = currentChi - tempChi;
            double scale = 0; for (int j = 0; j < 6; j++) scale += x[j] * (lambda * x[j] + b[j]);
            scale += 1e-3; rho /= scale;
            if (rho > 0 && std::isfinite(tempChi)) {
                double alpha = 1. - std::pow((2 * rho - 1), 3); alpha = std::min(alpha, 2. / 3.);
                lambda *= std::max(1. / 3., alpha); ni = 2; currentChi = tempChi; accepted = 1;
            } else { lambda *= ni; ni *= 2; pose = backup; }
            qmax++;
        } while (rho < 0 && qmax < 10);
        log.push_back({currentChi, lambda, qmax, accepted}); logStop.push_back(0);
        if (qmax == 10 || rho == 0) { logStop.back() = qmax == 10 ? 1 : 2; return 1; }
        if ((iniChi - currentChi) * 1e3 < iniChi) nBad++; else nBad = 0;
        if (nBad >= 3) { logStop.back() = 3; return 1; }
        return 0;
    }
    // returns inliers; outlier[e] as mvbOutlier (src/Optimizer.cpp:133-189)
    int run(uint8_t* outlier) {
        err.assign((size_t)n * 2, 0); level.assign(n, 0); robust = true; log.clear(); logRound.clear(); logStop.clear(); pose = pose0;
        roundOutlier.assign((size_t)4 * n, 0);
        for (int e = 0; e < n; e++) outlier[e] = 0;
        for (int k = 0; k < 6; k++) x[k] = 0;
        if (n < 3) return 0;
        int nBadEdges = 0;
        for (int it = 0; it < 4; it++) {
            pose = pose0;
            actE.clear(); for (int e = 0; e < n; e++) if (level[e] == 0) actE.push_back(e);
            if (!actE.empty()) { bool ok = true; for (int i = 0; i < 10 && ok; i++) ok = (lmIteration(i) == 0); }
            logRound.resize(log.size(), it);
            nBadEdges = 0;
            for (int e = 0; e < n; e++) {
                if (outlier[e]) computeError(e);
                const float c = (float)chi2(e);
                if (c > 5.991f) { outlier[e] = 1; level[e] = 1; nBadEdges++; } else { outlier[e] = 0; level[e] = 0; }
                roundOutlier[(size_t)it * n + e] = outlier[e];
            }
            if (it == 2) robust = false;
            if (n < 10) break;
        }
        return n - nBadEdges;
    }
};

}  // namespace orc

// fp64 geometry shared by the bundle-adjustment kernels (host + device).
//   SE3Quat::map/exp/operator*/normalizeRotation   reference ThirdParty/g2o/g2o/types/se3quat.h:104-110,217-257,280-285
//   Eigen Quaterniond(Matrix3d) / toRotationMatrix  (un-vendored Eigen; standard algorithms restated)
//   EdgeSE3ProjectXYZMultiPinhole*                   reference src/g2o_cubemap_vertices_edges.cpp:61-124,164-233
//   CamModelGeneral::TransformRaysToTargetFace       reference src/CamModelGeneral.cpp:228-263 (float3 round trip!)
#pragma once
#include <cmath>
#include <cstdint>

#ifdef __CUDACC__
#define BA_HD __host__ __device__ __forceinline__
#else
#define BA_HD inline
#endif

namespace cslam {

struct Pose { double q[4]; double t[3]; };   // q = (x,y,z,w)

BA_HD void quat_normalize_rotation(double* q) {
    if (q[3] < 0) { q[0] = -q[0]; q[1] = -q[1]; q[2] = -q[2]; q[3] = -q[3]; }
    const double n = sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]);
    q[0] /= n; q[1] /= n; q[2] /= n; q[3] /= n;
}
BA_HD void quat_from_matrix(const double m[3][3], double* q) {
    double t = m[0][0] + m[1][1] + m[2][2];
    if (t > 0) {
        t = sqrt(t + 1.0); q[3] = 0.5 * t; t = 0.5 / t;
        q[0] = (m[2][1] - m[1][2]) * t; q[1] = (m[0][2] - m[2][0]) * t; q[2] = (m[1][0] - m[0][1]) * t;
    } else {
        int i = 0; if (m[1][1] > m[0][0]) i = 1; if (m[2][2] > m[i][i]) i = 2;
        const int j = (i + 1) % 3, k = (j + 1) % 3;
        t = sqrt(m[i][i] - m[j][j] - m[k][k] + 1.0);
        double v[3]; v[i] = 0.5 * t; t = 0.5 / t;
        q[3] = (m[k][j] - m[j][k]) * t; v[j] = (m[j][i] + m[i][j]) * t; v[k] = (m[k][i] + m[i][k]) * t;
        q[0] = v[0]; q[1] = v[1]; q[2] = v[2];
    }
}
BA_HD void quat_to_matrix(const double* q, double R[3][3]) {
    const double tx = 2 * q[0], ty = 2 * q[1], tz = 2 * q[2];
    const double twx = tx * q[3], twy = ty * q[3], twz = tz * q[3];
    const double txx = tx * q[0], txy = ty * q[0], txz = tz * q[0];
    const double tyy = ty * q[1], tyz = tz * q[1], tzz = tz * q[2];
    R[0][0] = 1 - (tyy + tzz); R[0][1] = txy - twz; R[0][2] = txz + twy;
    R[1][0] = txy + twz; R[1][1] = 1 - (txx + tzz); R[1][2] = tyz - twx;
    R[2][0] = txz - twy; R[2][1] = tyz + twx; R[2][2] = 1 - (txx + tyy);
}
BA_HD void quat_rotate(const double* q, const double* v, double* out) {
    double uv[3] = {q[1] * v[2] - q[2] * v[1], q[2] * v[0] - q[0] * v[2], q[0] * v[1] - q[1] * v[0]};
    uv[0] += uv[0]; uv[1] += uv[1]; uv[2] += uv[2];
    out[0] = v[0] + q[3] * uv[0] + (q[1] * uv[2] - q[2] * uv[1]);
    out[1] = v[1] + q[3] * uv[1] + (q[2] * uv[0] - q[0] * uv[2]);
    out[2] = v[2] + q[3] * uv[2] + (q[0] * uv[1] - q[1] * uv[0]);
}
BA_HD void pose_map(const Pose& T, const double* X, double* out) {
    quat_rotate(T.q, X, out); out[0] += T.t[0]; out[1] += T.t[1]; out[2] += T.t[2];
}
// Converter::toSE3Quat (reference src/Converter.cpp:41-51)
BA_HD Pose pose_from_Tcw32(const float* T) {
    double R[3][3];
    for (int i = 0; i < 3; i++) for (int j = 0; j < 3; j++) R[i][j] = (double)T[i * 4 + j];
    Pose p; quat_from_matrix(R, p.q); quat_normalize_rotation(p.q);
    for (int i = 0; i < 3; i++) p.t[i] = (double)T[i * 4 + 3];
    return p;
}
BA_HD void pose_to_Tcw32(const Pose& p, float* T) {
    double R[3][3]; quat_to_matrix(p.q, R);
    for (int i = 0; i < 3; i++) { for (int j = 0; j < 3; j++) T[i * 4 + j] = (float)R[i][j]; T[i * 4 + 3] = (float)p.t[i]; }
    T[12] = 0; T[13] = 0; T[14] = 0; T[15] = 1;
}
// the 7-double pose record of the fp64 outputs (pose_fp64): t, then q = (x, y, z, w)
BA_HD void pose_to_fp64(const Pose& p, double* r) {
    r[0] = p.t[0]; r[1] = p.t[1]; r[2] = p.t[2]; r[3] = p.q[0]; r[4] = p.q[1]; r[5] = p.q[2]; r[6] = p.q[3];
}
// estimate <- SE3Quat::exp(update) * estimate   (VertexSE3Expmap::oplusImpl), update = [omega, upsilon]
BA_HD Pose pose_oplus(const Pose& est, const double* u) {
    const double w[3] = {u[0], u[1], u[2]}, up[3] = {u[3], u[4], u[5]};
    const double theta = sqrt(w[0] * w[0] + w[1] * w[1] + w[2] * w[2]);
    const double O[3][3] = {{0, -w[2], w[1]}, {w[2], 0, -w[0]}, {-w[1], w[0], 0}};
    double O2[3][3];
    for (int i = 0; i < 3; i++) for (int j = 0; j < 3; j++) O2[i][j] = O[i][0] * O[0][j] + O[i][1] * O[1][j] + O[i][2] * O[2][j];
    double R[3][3], V[3][3];
    if (theta < 0.00001) {
        for (int i = 0; i < 3; i++) for (int j = 0; j < 3; j++) { R[i][j] = (i == j) + O[i][j] + O2[i][j]; V[i][j] = R[i][j]; }
    } else {
        const double a = sin(theta) / theta, b = (1 - cos(theta)) / (theta * theta), c = (theta - sin(theta)) / (theta * theta * theta);
        for (int i = 0; i < 3; i++) for (int j = 0; j < 3; j++) { R[i][j] = (i == j) + a * O[i][j] + b * O2[i][j]; V[i][j] = (i == j) + b * O[i][j] + c * O2[i][j]; }
    }
    Pose e; quat_from_matrix(R, e.q);
    for (int i = 0; i < 3; i++) e.t[i] = V[i][0] * up[0] + V[i][1] * up[1] + V[i][2] * up[2];
    quat_normalize_rotation(e.q);
    Pose r; double rt[3]; quat_rotate(e.q, est.t, rt);
    for (int i = 0; i < 3; i++) r.t[i] = e.t[i] + rt[i];
    const double* a = e.q; const double* b = est.q;
    r.q[3] = a[3] * b[3] - a[0] * b[0] - a[1] * b[1] - a[2] * b[2];
    r.q[0] = a[3] * b[0] + a[0] * b[3] + a[1] * b[2] - a[2] * b[1];
    r.q[1] = a[3] * b[1] + a[1] * b[3] + a[2] * b[0] - a[0] * b[2];
    r.q[2] = a[3] * b[2] + a[2] * b[3] + a[0] * b[1] - a[1] * b[0];
    quat_normalize_rotation(r.q);
    return r;
}

// Face rotation: rig -> face-local (cvtRigToFaces, reference include/CamModelGeneral.h:417-443 == R_local of the edges)
BA_HD void rig_to_face(int face, double x, double y, double z, double& lx, double& ly, double& lz) {
    switch (face) {
        case 0: lx = x; ly = y; lz = z; break;       // FRONT
        case 1: lx = z; ly = y; lz = -x; break;      // LEFT
        case 2: lx = -z; ly = y; lz = x; break;      // RIGHT
        case 3: lx = x; ly = z; lz = -y; break;      // UPPER
        default: lx = x; ly = -z; lz = y; break;     // LOWER
    }
}
// e = m_inface - multipinhole_project(Xc): Xc is cast to float3 first, the projection is evaluated in fp64 and stored as float
BA_HD void edge_error(int face, double f, double mx, double my, const double* Xc, double* e) {
    double lx, ly, lz;
    rig_to_face(face, (double)(float)Xc[0], (double)(float)Xc[1], (double)(float)Xc[2], lx, ly, lz);
    const float u = (float)(lx * f / lz + f), v = (float)(ly * f / lz + f);
    e[0] = mx - (double)u; e[1] = my - (double)v;
}
// G = -dudLocal * R_local (2x3); Jpose = G * [-[Xc]x | I]; Jpoint = G * R(q)
BA_HD void edge_G(int face, double f, const double* Xc, double G[2][3]) {
    double L[3]; rig_to_face(face, Xc[0], Xc[1], Xc[2], L[0], L[1], L[2]);
    const double iz = f / L[2], ax = -f * L[0] / (L[2] * L[2]), ay = -f * L[1] / (L[2] * L[2]);
    // D = [[iz,0,ax],[0,iz,ay]] ; R_local rows are signed unit vectors
    double Rl[3][3] = {{0, 0, 0}, {0, 0, 0}, {0, 0, 0}};
    switch (face) {
        case 0: Rl[0][0] = 1; Rl[1][1] = 1; Rl[2][2] = 1; break;
        case 1: Rl[0][2] = 1; Rl[1][1] = 1; Rl[2][0] = -1; break;
        case 2: Rl[0][2] = -1; Rl[1][1] = 1; Rl[2][0] = 1; break;
        case 3: Rl[0][0] = 1; Rl[1][2] = 1; Rl[2][1] = -1; break;
        default: Rl[0][0] = 1; Rl[1][2] = -1; Rl[2][1] = 1; break;
    }
    for (int j = 0; j < 3; j++) {
        G[0][j] = -1.0 * (iz * Rl[0][j] + ax * Rl[2][j]);
        G[1][j] = -1.0 * (iz * Rl[1][j] + ay * Rl[2][j]);
    }
}
BA_HD void edge_Jpose(const double G[2][3], const double* Xc, double Jp[2][6]) {
    const double nS[3][3] = {{0, Xc[2], -Xc[1]}, {-Xc[2], 0, Xc[0]}, {Xc[1], -Xc[0], 0}};
    for (int i = 0; i < 2; i++) for (int j = 0; j < 3; j++) {
        Jp[i][j] = G[i][0] * nS[0][j] + G[i][1] * nS[1][j] + G[i][2] * nS[2][j];
        Jp[i][j + 3] = G[i][j];
    }
}
// Huber delta of both optimizers: the reference's float thHuberMono = sqrt(5.991), widened to double
BA_HD double huber_delta() { return (double)(float)sqrt(5.991); }
// Huber (RobustKernelHuber::robustify)
BA_HD void huber(double delta, double dsqr, double e, double& rho0, double& rho1) {
    if (e <= dsqr) { rho0 = e; rho1 = 1.0; }
    else { const double s = sqrt(e); rho0 = 2 * s * delta - dsqr; rho1 = delta / s; }
}

}  // namespace cslam

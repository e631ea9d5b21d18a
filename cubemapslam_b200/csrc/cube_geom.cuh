// Cube-map geometry shared by the projection matchers (track.cu) and the LocalMapping feature operations (mapping.cu): the device-side
// window walk and projections, and the frame index both search.
#pragma once
#include "area_table.cuh"
#include "common.cuh"

namespace cslam {

// k_frame_index (track.cu) on the caller's stream, counted on the caller's launch counter: rays (optional) and the cell CSR of `nframes`
// frames of key points, kpStride <= maxStride (<= 65535: the CSR holds u16 positions and indices). prepare_frame_index() sets the kernel's
// shared-memory limit on the current device; every handle that launches it calls it once, at create.
int prepare_frame_index();
int frame_index(cudaStream_t stream, int64_t& launches, const cslam_keypoint* kps, const int32_t* n, int nframes, int kpStride, int faceW, int faceH, float* rays,
                uint16_t* cellStart, uint16_t* cellIdx, int maxStride = 4096);

// The GetFeaturesInArea window table in constant memory (without -rdc every translation unit that includes this holds its own copy)
static __constant__ AreaRect c_area[5][9][3] = AREA_TABLE_INIT;

// `Rcw * x + tcw` on CV_32F Mats: float products summed left to right, then (float)((double)t + (double)tcw). T: the top 3 x 4 of a
// row-major 4 x 4 Tcw.
__device__ __forceinline__ void transform_cw(const float* T, const float* x, float (&xc)[3]) {
#pragma unroll
    for (int i = 0; i < 3; i++) {
        float t = __fmul_rn(T[4 * i], x[0]);
        t = __fadd_rn(t, __fmul_rn(T[4 * i + 1], x[1]));
        t = __fadd_rn(t, __fmul_rn(T[4 * i + 2], x[2]));
        xc[i] = (float)((double)t + (double)T[4 * i + 3]);
    }
}

// Rectangle k of a GetFeaturesInArea window, clamped to its face: n cells (0 if the clamp leaves none); the ci-th in the reference's
// visiting order (ix major, iy minor) is cell(ci) of the 5 x 50 x 50 grid.
struct AreaCells {
    int face, x0, y0, ny, n;
    __device__ int cell(int ci) const { return (face * GRID_G + x0 + ci / ny) * GRID_G + y0 + ci % ny; }
};
// false: the window has no rectangle k (the table lists the used ones first)
__device__ __forceinline__ bool area_cells(const AreaQuery& aq, int k, AreaCells& r) {
    const AreaRect rc = c_area[aq.face][aq.caseRow][k];
    if (rc.face == FACE_NONE) return false;
    const int x0 = max(0, area_sym(aq, rc.x0)), x1 = min(GRID_G - 1, area_sym(aq, rc.x1));
    const int y0 = max(0, area_sym(aq, rc.y0)), y1 = min(GRID_G - 1, area_sym(aq, rc.y1));
    r.face = rc.face; r.x0 = x0; r.y0 = y0; r.ny = y1 - y0 + 1;
    r.n = (x0 > x1 || y0 > y1) ? 0 : (x1 - x0 + 1) * r.ny;
    return true;
}

// TransformRaysToCubemap (src/CamModelGeneral.cpp:95-154): ordered face tests, double pinhole, float result, in-face bounds, tile offset
__device__ __forceinline__ bool ray_to_cubemap(float x, float y, float z, int W, int H, float& up, float& vp) {
    int face; float lx, ly, lz;
    if (z > 0 && __fdiv_rn(x, z) <= 1 && __fdiv_rn(x, z) >= -1 && __fdiv_rn(y, z) <= 1 && __fdiv_rn(y, z) >= -1) { face = FACE_FRONT; lx = x; ly = y; lz = z; }
    else if (x > 0 && __fdiv_rn(y, x) <= 1 && __fdiv_rn(y, x) >= -1 && __fdiv_rn(z, x) <= 1 && __fdiv_rn(z, x) >= -1) { face = FACE_RIGHT; lx = -z; ly = y; lz = x; }
    else if (x < 0 && __fdiv_rn(y, -x) <= 1 && __fdiv_rn(y, -x) >= -1 && __fdiv_rn(z, -x) <= 1 && __fdiv_rn(z, -x) >= -1) { face = FACE_LEFT; lx = z; ly = y; lz = -x; }
    else if (y > 0 && __fdiv_rn(x, y) <= 1 && __fdiv_rn(x, y) >= -1 && __fdiv_rn(z, y) <= 1 && __fdiv_rn(z, y) >= -1) { face = FACE_LOWER; lx = x; ly = -z; lz = y; }
    else if (y < 0 && __fdiv_rn(x, -y) <= 1 && __fdiv_rn(x, -y) >= -1 && __fdiv_rn(z, -y) <= 1 && __fdiv_rn(z, -y) >= -1) { face = FACE_UPPER; lx = x; ly = z; lz = -y; }
    else { up = -1.0f; vp = -1.0f; return false; }   // the reference sets (-1, -1) here; a failed in-face test below leaves the face coordinates
    const double fx = W / 2.0, fy = H / 2.0;
    up = (float)__dadd_rn(__ddiv_rn(__dmul_rn((double)lx, fx), (double)lz), fx);
    vp = (float)__dadd_rn(__ddiv_rn(__dmul_rn((double)ly, fy), (double)lz), fy);
    if (up < 0 || up >= (float)W || vp < 0 || vp >= (float)H) return false;
    switch (face) {
        case FACE_FRONT: up = __fadd_rn(up, (float)W); vp = __fadd_rn(vp, (float)H); break;
        case FACE_RIGHT: up = __fadd_rn(up, (float)(2 * W)); vp = __fadd_rn(vp, (float)H); break;
        case FACE_LEFT: vp = __fadd_rn(vp, (float)H); break;
        case FACE_LOWER: up = __fadd_rn(up, (float)W); vp = __fadd_rn(vp, (float)(2 * H)); break;
        default: up = __fadd_rn(up, (float)W); break;
    }
    return true;
}

}  // namespace cslam

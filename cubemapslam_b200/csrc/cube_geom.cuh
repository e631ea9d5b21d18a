// Device-side cube-map geometry shared by the projection matchers (track.cu) and the LocalMapping feature operations (mapping.cu).
#pragma once
#include "area_table.cuh"

namespace cslam {

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

// Cube-face wrap-around of Frame::GetFeaturesInArea (reference src/Frame.cpp:251-716) as a TABLE: for every (face, overflow case) the up to three
// cell rectangles the reference visits, in visiting order, with each bound written as one of thirteen symbols (optionally mirrored, 49 - v).
// Host + device. The reference spells the same thing as ~470 lines of nested switch / if; both are checked against the compiled reference
// through the oracle (tests/test_oracle_frame_index.py, tests/test_track_tables.py).
#pragma once
#include <cmath>
#include <cstdint>

namespace cslam {

enum { FACE_FRONT = 0, FACE_LEFT = 1, FACE_RIGHT = 2, FACE_UPPER = 3, FACE_LOWER = 4, FACE_NONE = 0xff };
// canvas tile (column, row) of each face, in FACE_* order; the canvas is 3 x 3 faces and its four corner tiles belong to no face
static const int FACE_TILE_COL[5] = {1, 0, 2, 1, 1}, FACE_TILE_ROW[5] = {1, 1, 1, 0, 2};
static const int GRID_G = 50;   // CUBEFACE_GRID_COLS == CUBEFACE_GRID_ROWS (include/Frame.h:43-45)

// symbols: cell index of a window edge, in the centre's face (a b c d) or shifted by one face width / negated (the neighbour's frame)
enum { sZ = 0, sM = 1, sG = 2, sA = 3, sB = 4, sC = 5, sD = 6, sBW = 7, sDH = 8, sAW = 9, sCH = 10, sAN = 11, sCN = 12 };
#define AR_R(v) ((v) | 16)   // 49 - v
struct AreaRect { uint8_t face, x0, x1, y0, y1; };
#define AR_F FACE_FRONT
#define AR_L FACE_LEFT
#define AR_RT FACE_RIGHT
#define AR_U FACE_UPPER
#define AR_LO FACE_LOWER
#define AR_NONE {FACE_NONE, 0, 0, 0, 0}
// case rows: 0 window inside the face | 1 x inside, y overflow | 2 x inside, y underflow | 3 y inside, x overflow | 4 y inside, x underflow |
//            5 xO&yO | 6 xU&yO | 7 xO&yU | 8 xU&yU
#define AREA_TABLE_INIT                                                                                                                                   \
    {   /* FRONT */                                                                                                                                       \
        {{{AR_F, sA, sB, sC, sD}, AR_NONE, AR_NONE},                                                                                                    \
         {{AR_F, sA, sB, sC, sM}, {AR_LO, sA, sB, sZ, sDH}, AR_NONE},                                                                                   \
         {{AR_U, sA, sB, sCH, sM}, {AR_F, sA, sB, sZ, sD}, AR_NONE},                                                                                    \
         {{AR_F, sA, sM, sC, sD}, {AR_RT, sZ, sBW, sC, sD}, AR_NONE},                                                                                   \
         {{AR_L, sAW, sM, sC, sD}, {AR_F, sZ, sB, sC, sD}, AR_NONE},                                                                                    \
         {{AR_F, sA, sM, sC, sM}, {AR_RT, sZ, sBW, sC, sM}, {AR_LO, sA, sM, sZ, sDH}},                                                                  \
         {{AR_F, sZ, sB, sC, sM}, {AR_L, sAW, sM, sC, sM}, {AR_LO, sZ, sB, sZ, sDH}},                                                                   \
         {{AR_F, sA, sM, sZ, sD}, {AR_RT, sZ, sBW, sZ, sD}, {AR_U, sA, sM, AR_R(sCH), sM}},                                                             \
         {{AR_F, sZ, sB, sZ, sD}, {AR_L, AR_R(sAW), sM, sZ, sD}, {AR_U, sZ, sB, AR_R(sCH), sM}}},                                                       \
        /* LEFT */                                                                                                                                        \
        {{{AR_L, sA, sB, sC, sD}, AR_NONE, AR_NONE},                                                                                                    \
         {{AR_L, sA, sB, sC, sM}, {AR_LO, sZ, sDH, AR_R(sB), AR_R(sA)}, AR_NONE},                                                                       \
         {{AR_U, sZ, sCN, sA, sB}, {AR_L, sA, sB, sZ, sD}, AR_NONE},                                                                                    \
         {{AR_F, sZ, sBW, sC, sD}, {AR_L, sA, sM, sC, sD}, AR_NONE},                                                                                    \
         {{AR_L, sZ, sB, sC, sD}, AR_NONE, AR_NONE},                                                                                                    \
         {{AR_L, sA, sM, sC, sM}, {AR_F, sZ, sBW, sC, sM}, {AR_LO, sZ, sDH, sZ, AR_R(sA)}},                                                             \
         {{AR_L, sZ, sB, sC, sM}, {AR_LO, sZ, sDH, AR_R(sB), sM}, AR_NONE},                                                                             \
         {{AR_L, sA, sM, sZ, sD}, {AR_F, sZ, sBW, sZ, sD}, {AR_U, sZ, sCN, sA, sM}},                                                                    \
         {{AR_L, sZ, sB, sZ, sD}, {AR_U, sZ, sCN, sZ, sD}, AR_NONE}},                                                                                   \
        /* RIGHT */                                                                                                                                       \
        {{{AR_RT, sA, sB, sC, sD}, AR_NONE, AR_NONE},                                                                                                   \
         {{AR_RT, sA, sB, sC, sM}, {AR_LO, AR_R(sDH), sM, sA, sB}, AR_NONE},                                                                            \
         {{AR_U, sCH, sM, AR_R(sB), AR_R(sA)}, {AR_RT, sA, sB, sZ, sD}, AR_NONE},                                                                       \
         {{AR_RT, sA, sM, sC, sD}, AR_NONE, AR_NONE},                                                                                                   \
         {{AR_F, sAW, sM, sC, sD}, {AR_RT, sZ, sB, sC, sD}, AR_NONE},                                                                                   \
         {{AR_RT, sA, sM, sC, sM}, {AR_LO, AR_R(sDH), sM, sA, sM}, AR_NONE},                                                                            \
         {{AR_RT, sZ, sB, sC, sM}, {AR_F, AR_R(sAN), sM, sC, sM}, {AR_LO, AR_R(sDH), sM, sZ, sB}},                                                      \
         {{AR_RT, sA, sM, sZ, sD}, {AR_U, AR_R(sCN), sM, sZ, AR_R(sA)}, AR_NONE},                                                                       \
         {{AR_RT, sZ, sB, sZ, sD}, {AR_F, AR_R(sAN), sM, sZ, sD}, {AR_U, AR_R(sCN), sM, AR_R(sB), sM}}},                                                \
        /* UPPER */                                                                                                                                       \
        {{{AR_U, sA, sB, sC, sD}, AR_NONE, AR_NONE},                                                                                                    \
         {{AR_U, sA, sB, sC, sM}, {AR_F, sA, sB, sZ, sDH}, AR_NONE},                                                                                    \
         {{AR_LO, sA, sB, sZ, sD}, AR_NONE, AR_NONE},                                                                                                   \
         {{AR_U, sA, sM, sC, sD}, {AR_RT, AR_R(sD), AR_R(sC), sZ, sBW}, AR_NONE},                                                                       \
         {{AR_L, sC, sD, sZ, sAN}, {AR_U, sZ, sB, sC, sD}, AR_NONE},                                                                                    \
         {{AR_U, sA, sM, sC, sM}, {AR_RT, sZ, AR_R(sC), sZ, sBW}, {AR_F, sA, sM, sZ, sDH}},                                                             \
         {{AR_U, sZ, sB, sC, sM}, {AR_L, sC, sM, sZ, sAN}, {AR_F, sZ, sB, sZ, sDH}},                                                                    \
         {{AR_U, sA, sM, sZ, sD}, {AR_RT, AR_R(sD), sM, sZ, sD}, AR_NONE},                                                                              \
         {{AR_U, sZ, sB, sZ, sD}, {AR_L, sZ, sD, sZ, sAN}, AR_NONE}},                                                                                   \
        /* LOWER */                                                                                                                                       \
        {{{AR_LO, sA, sB, sC, sD}, AR_NONE, AR_NONE},                                                                                                   \
         {{AR_LO, sA, sB, sC, sM}, AR_NONE, AR_NONE},                                                                                                   \
         {{AR_F, sA, sB, sCH, sM}, {AR_LO, sA, sB, sZ, sD}, AR_NONE},                                                                                   \
         {{AR_LO, sA, sM, sC, sD}, {AR_RT, sC, sD, AR_R(sBW), sG}, AR_NONE},                                                                            \
         {{AR_L, AR_R(sD), AR_R(sC), sAW, sM}, {AR_LO, sZ, sB, sC, sD}, AR_NONE},                                                                       \
         {{AR_LO, sA, sM, sC, sM}, {AR_RT, sA, sM, AR_R(sBW), sM}, AR_NONE},                                                                            \
         {{AR_LO, sZ, sB, sC, sM}, {AR_L, sZ, AR_R(sC), AR_R(sAW), sM}, AR_NONE},                                                                       \
         {{AR_LO, sA, sM, sZ, sD}, {AR_RT, sZ, sD, AR_R(sBW), sG}, {AR_F, sA, sM, AR_R(sCN), sM}},                                                      \
         {{AR_LO, sZ, sB, sZ, sD}, {AR_L, AR_R(sAN), sM, AR_R(sAN), sG}, {AR_F, sZ, sB, AR_R(sCN), sM}}},                                               \
    }

struct AreaQuery { int face; int caseRow; int sym[13]; };

// FaceInCubemap (include/CamModelGeneral.h:458-470), the one definition of the face a canvas pixel lies on; -1: a corner tile or outside.
// It also stands for the cv::Point2f overload, which widens the float quotient to double: the quotients are IEEE-rounded here (nvcc's
// default -prec-div=true, plain IEEE float on the host) and compared with the exact constants 0..3, which widening does not change.
__host__ __device__ inline int face_of_pixel_f(float x, float y, int W, int H) {
    const float i = x / (float)W, j = y / (float)H;
    if (i >= 0 && i < 1 && j >= 1 && j < 2) return FACE_LEFT;
    if (i >= 1 && i < 2 && j >= 0 && j < 1) return FACE_UPPER;
    if (i >= 1 && i < 2 && j >= 1 && j < 2) return FACE_FRONT;
    if (i >= 1 && i < 2 && j >= 2 && j < 3) return FACE_LOWER;
    if (i >= 2 && i < 3 && j >= 1 && j < 2) return FACE_RIGHT;
    return -1;
}
// GetPosInFace<double>: the position of canvas coordinate x inside its face of width W
__host__ __device__ inline double pos_in_face(float x, int W) { return (double)x - floor((double)x / W) * W; }

// classifies the search window [x-r, x+r] x [y-r, y+r] (src/Frame.cpp:256-286) and evaluates the thirteen symbols; false: centre on no face
__host__ __device__ inline bool area_query(float x, float y, float r, int W, int H, float inv, AreaQuery& q) {
    q.face = face_of_pixel_f(x, y, W, H);
    if (q.face < 0) return false;
    const int cornerX = (int)x / W * W, cornerY = (int)y / H * H;
    const float xIn = x - (float)cornerX, yIn = y - (float)cornerY;
    const float xs = xIn - r, xe = xIn + r, ys = yIn - r, ye = yIn + r;
    const bool xU = xs < 0, xO = xe > (float)(W - 1), yU = ys < 0, yO = ye > (float)(H - 1);
    const bool xInF = !xO && !xU, yInF = !yO && !yU;
    if (xInF && yInF) q.caseRow = 0;
    else if (xInF) q.caseRow = yO ? 1 : 2;
    else if (yInF) q.caseRow = xO ? 3 : 4;
    else q.caseRow = (xO && yO) ? 5 : (xU && yO) ? 6 : (xO && yU) ? 7 : 8;
    q.sym[sZ] = 0; q.sym[sM] = GRID_G - 1; q.sym[sG] = GRID_G;
    q.sym[sA] = (int)floorf(xs * inv); q.sym[sB] = (int)floorf(xe * inv); q.sym[sC] = (int)floorf(ys * inv); q.sym[sD] = (int)floorf(ye * inv);
    q.sym[sBW] = (int)floorf((xe - (float)W) * inv); q.sym[sDH] = (int)floorf((ye - (float)H) * inv);
    q.sym[sAW] = (int)floorf((xs + (float)W) * inv); q.sym[sCH] = (int)floorf((ys + (float)H) * inv);
    q.sym[sAN] = (int)floorf((-xs) * inv); q.sym[sCN] = (int)floorf((-ys) * inv);
    return true;
}
__host__ __device__ inline int area_sym(const AreaQuery& q, uint8_t s) { const int v = q.sym[s & 15]; return (s & 16) ? GRID_G - 1 - v : v; }

}  // namespace cslam

"""Scenes for Optimizer::PoseOptimization (and LocalBA's classification) at their thresholds, stops, seams and degenerate systems, shared by
tests/test_oracle_pose_limits.py (CPU, oracle) and tests/test_gpu_pose_limits.py (GPU against the oracle). Every scene is a list of frames
(Tcw 4x4 float32, Xw n x 3, kpxy n x 2, inv_sigma2 n), built at the face widths of WIDTHS.

Stationary threshold frames. The prior is the identity and the geometry dyadic: a MapPoint at face-local d*(a, b, 1) with a, b multiples of
1/8 and d a power of two projects to exactly (a*f + f, b*f + f), f = W/2, so every error and Jacobian entry is exact. Each frame has zero-
residual correspondences on all five faces and one pair of correspondences to one MapPoint with errors (+1, 0) and (-1, 0): their gradient
contributions cancel exactly in any summation order (the two edges are separate threads of the kernel, so no FMA joins them), b = 0, the
step is 0, rho = 0 and every round stops after one rejected trial with the pose bit-unchanged. The pair's weight is its chi2 exactly:
5.991f is an inlier for PoseOptimization's float compare and an outlier for LocalBA's double compare; one float ulp above is an outlier for
both, one ulp below an inlier for both. A fourth pair has errors (+-1, +-0.25) and a chi2 that is exact in double, above 5.991f, and
rounds to 5.991f: an inlier only through PoseOptimization's float cast. LocalBA's scene uses the same technique with every key frame fixed, plus camera depths 0 (an
outlier with zero residual), -0.5 and +2^-4.

Seams. face_of_pixel_f takes the face from a float quotient and pos_in_face the position from a double floor. They cannot disagree at any
face width: for a float x just below a seam k*W, the gap to the seam is at least 2^-24 of k*W (x and k*W share a binade or x is in the one
below), while the float quotient x / W rounds up to k only within half an ulp of k, at most 2^-24.58 of k. seam_disagreements() checks it
exhaustively for the floats within SEAM_ULPS ulps of every seam at every width of WIDTHS (the CPU test asserts that it finds none); the seam
frames put key points on the ulp-adjacent floats on both sides of every seam of the front face anyway.

Degenerate systems. A frame with every weight 0 (H = 0 and lambda = 0: every 6x6 solve fails, qmax reaches 10) and a frame with one
correspondence exactly on its face's plane (lz = 0, an infinite error). The kernel zeroes x on a failed solve and skips the update; g2o's
LinearSolverDense leaves x as it was and the update applies it. The two agree as long as no solve of the frame has succeeded before the
failure, which holds for these frames (the CPU test checks that every row of their logs is a rejected trial); no scene here reaches a failure
after a success. The oracle's zero-pivot rule stands in for Eigen's LDLT::isPositive, which cannot be pinned here.

Stale errors. An inlier is classified with the error of the last computeActiveErrors, at the last trial pose, even a rejected one; only
outliers get a fresh error at the final pose (src/Optimizer.cpp:156-163). The two poses differ only when the final round's last iteration
ends on ten rejected trials that moved the pose. No scene here reaches an inlier whose chi2 straddles 5.991f between those poses: a seeded
search over 20 000 random frames (3 to 40 correspondences, priors 5 to 60 degrees off, up to 60 % outliers) found none. The rule is pinned on the other side: outliers that become
inliers again in a later round (schedule frames) need their fresh error."""
import math

import numpy as np

from cubemapslam_b200 import synth

WIDTHS = (650, 450, 610)
TILES = {0: (1, 1), 1: (0, 1), 2: (2, 1), 3: (1, 0), 4: (1, 2)}     # face -> (column, row) of the canvas: front, left, right, upper, lower
CHI2_TH = np.float32(5.991)
PAIR_WEIGHTS = (CHI2_TH, np.nextafter(CHI2_TH, np.float32(np.inf)), np.nextafter(CHI2_TH, np.float32(0)))
# a pair with errors (+-1, +-0.25): its chi2 = w * 17/16 is exact in double, above 5.991f and rounds to 5.991f, an inlier only after the float cast
ROUND_PAIR = (np.float32(5.991 / 1.0625), 0.25)
SEAM_ULPS = 64


def local_to_rig(face, lx, ly, lz):
    """Inverse of the face rotation rig_to_face (lx, ly, lz are face-local)."""
    return {0: (lx, ly, lz), 1: (-lz, ly, lx), 2: (lz, ly, -lx), 3: (lx, -lz, ly), 4: (lx, lz, -ly)}[face]


def canvas_of(face, a, b, W):
    """Canvas pixel of the face-local direction (a, b, 1): exact for dyadic a, b."""
    f = W / 2.0
    c, r = TILES[face]
    return c * W + a * f + f, r * W + b * f + f


def frame(Xw, kp, w, Tcw=None):
    return dict(Tcw=np.eye(4, dtype=np.float32) if Tcw is None else np.asarray(Tcw, np.float32), Xw=np.asarray(Xw, np.float32).reshape(-1, 3),
                kpxy=np.asarray(kp, np.float32).reshape(-1, 2), inv_sigma2=np.asarray(w, np.float32))


def zero_residual(W, n_per_face=3, scale=(1.0, 2.0, 4.0)):
    """Exact zero-residual correspondences, n_per_face on each of the five faces."""
    X, kp = [], []
    ab = ((-0.5, 0.25), (0.375, -0.625), (0.75, 0.5), (-0.125, -0.875))
    for face in range(5):
        for j in range(n_per_face):
            a, b = ab[j % len(ab)]
            d = scale[(face + j) % len(scale)]
            X.append(local_to_rig(face, d * a, d * b, d)); kp.append(canvas_of(face, a, b, W))
    return X, kp


STATIONARY_PAIRS = tuple((wp, 0.0) for wp in PAIR_WEIGHTS) + (ROUND_PAIR,)     # (weight, error in v) of each stationary frame's pair


def stationary_frames(W):
    """One frame per pair of STATIONARY_PAIRS; the pair is correspondences 7 and 8 (adjacent, so two threads of one warp)."""
    out = []
    for wp, ev in STATIONARY_PAIRS:
        X, kp = zero_residual(W)
        w = [1.0] * len(X)
        u, v = canvas_of(0, 0.5, 0.25, W)
        X[7:7] = [local_to_rig(0, 0.5, 0.25, 1.0)] * 2
        kp[7:7] = [(u + 1, v + ev), (u - 1, v - ev)]
        w[7:7] = [wp, wp]
        out.append(frame(X, kp, w))
    return out


def local_ba_scene(W):
    """LocalBA with every key frame fixed (key frames 0 and 1 share the identity pose). MapPoints 0..2: the weight pairs of PAIR_WEIGHTS,
    seen by key frames 0 (+1 px) and 1 (-1 px); MapPoints 3..5: zero residual at camera depth 0, -0.5 and +2^-4 (right face); the rest zero
    residual on all faces. expected: the outlier flag of every edge."""
    pts, eMP, eKF, kp, w, expected = [], [], [], [], [], []
    for i, wp in enumerate(PAIR_WEIGHTS):
        a, b = (0.5, 0.25 - 0.125 * i)
        u, v = canvas_of(0, a, b, W)
        pts.append(local_to_rig(0, a, b, 1.0))
        for k, du in ((0, 1.0), (1, -1.0)):
            eMP.append(i); eKF.append(k); kp.append((u + du, v)); w.append(wp); expected.append(i != 2)
    for depth in (0.0, -0.5, 0.0625):                  # rig Xc = (1, 0.25, depth) on the right face: lx = -depth, lz = 1
        a = -depth
        pts.append((1.0, 0.25, depth)); eMP.append(len(pts) - 1); eKF.append(0); kp.append(canvas_of(2, a, 0.25, W)); w.append(1.0)
        expected.append(depth <= 0)
    X, k0 = zero_residual(W)
    for x, k in zip(X, k0):
        pts.append(x); eMP.append(len(pts) - 1); eKF.append(len(pts) % 2); kp.append(k); w.append(1.0); expected.append(x[2] <= 0)   # rig depth
    return dict(Tcw=np.stack([np.eye(4, dtype=np.float32)] * 2), kf_fixed=np.ones(2, np.uint8), pts=np.array(pts, np.float32),
                eMP=np.array(eMP, np.int32), eKF=np.array(eKF, np.int32), kpxy=np.array(kp, np.float32), inv_sigma2=np.array(w, np.float32),
                faceW=W, faceH=W, expected=np.array(expected, np.uint8))


def rotated(q, deg, axis):
    T = q["Tcw"].astype(np.float64)
    ax = np.asarray(axis, np.float64); ax = ax / np.linalg.norm(ax)
    T[:3, :3] = synth._rodrigues(ax * math.radians(deg)) @ T[:3, :3]
    q = dict(q); q["Tcw"] = T.astype(np.float32)
    return q


SCHEDULE_SIZES = (3, 9, 10, 11, 256, 257, 4096)
SCHEDULE_OUTLIERS = (0.0, 0.15, 0.5)


def schedule_frames(W):
    """Random frames (synth.pose_problem) with priors rotated 10 to 40 degrees, so that the 10-iteration budget binds and trials get rejected,
    at every size of SCHEDULE_SIZES and outlier rate of SCHEDULE_OUTLIERS; the last frame's prior is 86 degrees off, so its first round
    loses every edge."""
    out = []
    for k, fr in enumerate(SCHEDULE_OUTLIERS):
        for j, n in enumerate(SCHEDULE_SIZES):
            q = synth.pose_problem(n=n, faceW=W, seed=500 + 10 * k + j, outlier_frac=fr, radius=1.5)
            out.append(frame(q["Xw"], q["kpxy"], q["inv_sigma2"], rotated(q, 10 + 30 * ((j + k) % 4) / 3, (1, 2 - j % 3, 0.5 * k))["Tcw"]))
    q = synth.pose_problem(n=300, faceW=W, seed=31, outlier_frac=0.0, radius=1.5)
    out.append(frame(q["Xw"], q["kpxy"], q["inv_sigma2"], rotated(q, 86, (0, 1, 0))["Tcw"]))
    return out


def seam_floats(W):
    """The floats within SEAM_ULPS ulps of every seam k*W (k = 1, 2, 3) of the canvas."""
    out = []
    for k in (1, 2, 3):
        s = np.float32(k * W)
        lo, hi = s, s
        for _ in range(SEAM_ULPS):
            lo = np.nextafter(lo, np.float32(0)); hi = np.nextafter(hi, np.float32(np.inf))
        a = np.arange(lo.view(np.int32), hi.view(np.int32) + 1, dtype=np.int32).view(np.float32)
        out.append(a)
    return np.concatenate(out)


def seam_disagreements(W):
    """Floats near the seams where face_of_pixel_f's float quotient and pos_in_face's double floor put x in different columns."""
    x = seam_floats(W)
    col_f = np.floor(x / np.float32(W)).astype(np.int64)                       # float quotient, compared with the integers 0..3
    col_d = np.floor(x.astype(np.float64) / W).astype(np.int64)
    return x[col_f != col_d]


def seam_frames(W):
    """Front-face key points one ulp inside each of its four seams (and on the seam itself, which belongs to the front face on its left and
    upper side), with MapPoints on their rays at depth 2 and 4; plus the matching points one ulp outside, on the left / right / upper /
    lower faces. Each frame also has zero-residual correspondences; the second frame's prior is 3 degrees off."""
    lo, hi = np.float32(W), np.float32(2 * W)
    below = lambda s: float(np.nextafter(s, np.float32(0)))
    above = lambda s: float(np.nextafter(s, np.float32(np.inf)))
    mid = 1.5 * W + 0.25
    pts = [(lo, mid), (above(lo), mid), (below(hi), mid), (mid, lo), (mid, above(lo)), (mid, below(hi)),       # front face
           (below(lo), mid), (hi, mid), (above(hi), mid), (mid, below(lo)), (mid, hi), (mid, above(hi))]       # left, right, right, upper, lower, lower
    X, kp = zero_residual(W)
    w = [1.0] * len(X)
    for i, (x, y) in enumerate(pts):
        ray = synth._pixel_to_ray(float(x), float(y), W)
        X.append(tuple(ray * (2.0 + 2.0 * (i % 2)))); kp.append((x, y)); w.append(1.0)
    fr = frame(X, kp, w)
    return [fr, frame(X, kp, w, rotated(fr, 3.0, (0.3, 1.0, -0.2))["Tcw"])]


def degenerate_frames(W):
    """Every weight 0 (H = 0, lambda = 0: every solve fails); one correspondence exactly on its face's plane (lz = 0: infinite error)."""
    X, kp = zero_residual(W)
    zero_w = frame(X, kp, [0.0] * len(X), rotated(frame(X, kp, [0.0] * len(X)), 5.0, (0, 1, 0))["Tcw"])
    X2, kp2 = list(X), list(kp)
    X2[4] = local_to_rig(1, 0.5, 0.25, 0.0)                 # on the left face's plane
    plane = frame(X2, kp2, [1.0] * len(X2), rotated(frame(X2, kp2, [1.0] * len(X2)), 2.0, (1, 0, 0))["Tcw"])
    return [zero_w, plane]


def off_face_batch(W):
    """Four frames; frame 2's correspondence 17 lies in the canvas's top-left corner tile (no face)."""
    frames = [frame(*zero_residual(W), [1.0] * 15) for _ in range(4)]
    X, kp = zero_residual(W, n_per_face=4)
    kp[17] = (10.0, 10.0)
    frames[2] = frame(X, kp, [1.0] * len(X))
    return frames


def batch(frames):
    """Concatenate frames for one host call with ragged offsets."""
    off = np.cumsum([0] + [len(q["Xw"]) for q in frames]).astype(np.int32)
    cat = lambda k: np.concatenate([q[k] for q in frames]) if off[-1] else np.zeros((0,) + frames[0][k].shape[1:], np.float32)
    return dict(Tcw=np.stack([q["Tcw"] for q in frames]), Xw=cat("Xw"), kpxy=cat("kpxy"), inv_sigma2=cat("inv_sigma2"), offset=off)


def all_frames(W):
    """Every PoseOptimization scene at width W, in one list, with a name per frame."""
    named = []
    named += [("stationary_%d" % i, q) for i, q in enumerate(stationary_frames(W))]
    named += [("schedule_%d" % i, q) for i, q in enumerate(schedule_frames(W))]
    named += [("seam_%d" % i, q) for i, q in enumerate(seam_frames(W))]
    named += [("degenerate_%d" % i, q) for i, q in enumerate(degenerate_frames(W))]
    return named

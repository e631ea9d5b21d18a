"""Scenes for Optimizer::LocalBundleAdjustment at the rules of its LM loop, shared by tests/test_oracle_local_ba_limits.py (CPU, oracle) and
tests/test_gpu_local_ba_limits.py (GPU against the oracle): the qmax == 10, rho == 0, nBad >= 3 and stop-flag ends of a round, trial loops
that end on a rejected trial, second rounds whose active set shrinks, NaN and infinite chi2, and reduced solves that fail. Every scene is a
dict of LocalBundleAdjustment's arguments (plus its1 / its2 / stop_after_trials where they differ from the reference's 5 / 10 / off), built
at the face widths of pose_limits_scenes.WIDTHS with its dyadic helpers.

Stationary scenes. Every key frame sits at the identity; key frames 0 and 2 are free, 1 is fixed. The zero-residual MapPoints of
zero_residual() are seen by all three. For each free key frame k and each weight of PAIR_WEIGHTS, two MapPoints at the same dyadic position
are seen by k with errors (+1, 0) / (-1, 0) and by key frame 1 with the opposite errors: every gradient term has an exact negative partner in
the same vertex, so b = 0 in any summation order, the Schur solve returns x = 0 exactly and rho == 0 ends both rounds after one trial. The
5.991f-weighted pairs are outliers of the double compare and leave round 2; poses and points stay bit-identical to the input.

Degenerate systems. A MapPoint at rig (0.5, 0.25, 0) seen through a front-face key point lies on the front face's plane: its error is
infinite. Seen only by a fixed key frame it makes its Hll NaN, so computeLambdaInit's std::max order matters: NaN when it is the last active
vertex (lambda NaN for the whole round), the maximum over the vertices after it otherwise (first: the free pose's diagonal drops out).
Seen by a free key frame, the NaN reaches S and every reduced solve fails; with an infinite currentChi, rho = (inf - DBL_MAX) / scale ends each
trial loop after its first, rejected trial. Every weight 0 gives H = 0 and lambda = 0: Dinv is NaN, every solve fails, qmax == 10 ends both
rounds. The zero-weight-round-2 scene (conflicting()) moves its landmarks in round 1 and then loses every weighted edge, so round 2 fails ten
solves after the landmarks had a step: a kernel that applied a step from a failed solve would classify from errors of a state the LM loop
never visits.
The oracle's pivot rule (a zero or non-finite pivot fails) stands in for SimplicialLDLT's, which cannot be pinned without Eigen; no scene
here has a pivot that is finite, non-zero and rejected by Eigen.
"""
import math

import numpy as np

from cubemapslam_b200 import synth
from tests.pose_limits_scenes import PAIR_WEIGHTS, WIDTHS, canvas_of, local_to_rig, zero_residual  # noqa: F401  (WIDTHS re-exported)

PLANE = ((0.5, 0.25, 0.0), (0, 0.5, 0.25))      # rig position on the front face's plane, and the (face, a, b) of its key point


def problem(Tcw, fixed, pts, eMP, eKF, kp, w, W, **kw):
    p = dict(Tcw=np.asarray(Tcw, np.float32).reshape(-1, 4, 4), kf_fixed=np.asarray(fixed, np.uint8), pts=np.asarray(pts, np.float32).reshape(-1, 3),
             eMP=np.asarray(eMP, np.int32), eKF=np.asarray(eKF, np.int32), kpxy=np.asarray(kp, np.float32).reshape(-1, 2),
             inv_sigma2=np.asarray(w, np.float32), faceW=W, faceH=W)
    p.update(kw)
    return p


def args(p):
    return (p["Tcw"], p["kf_fixed"], p["pts"], p["eMP"], p["eKF"], p["kpxy"], p["inv_sigma2"], p["faceW"], p["faceH"])


def kwargs(p):
    return {k: p[k] for k in ("its1", "its2", "stop_after_trials") if k in p}


class Builder:
    def __init__(self, nKF):
        self.pts, self.eMP, self.eKF, self.kp, self.w = [], [], [], [], []
        self.T = np.stack([np.eye(4, dtype=np.float32)] * nKF)

    def point(self, X, obs):
        """obs: (key frame, canvas key point, weight) per edge."""
        self.pts.append(X)
        for k, kp, w in obs:
            self.eMP.append(len(self.pts) - 1); self.eKF.append(k); self.kp.append(kp); self.w.append(w)
        return len(self.pts) - 1

    def zero(self, W, kfs, w=1.0):
        for X, kp in zip(*zero_residual(W)):
            self.point(X, [(k, kp, w) for k in kfs])

    def build(self, fixed, W, **kw):
        return problem(self.T, fixed, self.pts, self.eMP, self.eKF, self.kp, self.w, W, **kw)


def stationary(W):
    b = Builder(3)
    b.zero(W, (0, 1, 2))
    for k in (0, 2):
        for i, wp in enumerate(PAIR_WEIGHTS):
            a, c = 0.5 - 0.25 * k, 0.25 - 0.125 * i
            u, v = canvas_of(0, a, c, W)
            X = local_to_rig(0, a, c, 1.0)
            for s in (1.0, -1.0):
                b.point(X, [(k, (u + s, v), wp), (1, (u - s, v), wp)])
    return b.build((0, 1, 0), W)


def plane_fixed(W, where):
    """Key frame 0 free and 1 cm off, key frame 1 fixed; the face-plane MapPoint seen only by key frame 1, placed first, in the middle or
    last in vertex order."""
    b = Builder(2)
    X, kp = zero_residual(W)
    at = {"first": 0, "middle": len(X) // 2, "last": len(X)}[where]
    for i in range(len(X) + 1):
        if i == at:
            b.point(PLANE[0], [(1, canvas_of(*PLANE[1], W), 1.0)])
        if i < len(X):
            b.point(X[i], [(0, kp[i], 1.0), (1, kp[i], 1.0)])
    b.T[0, 0, 3] = 0.01
    return b.build((0, 1), W)


def plane_free(W):
    """The face-plane MapPoint seen by the free key frame 0: NaN in S, every reduced solve fails."""
    b = Builder(2)
    b.zero(W, (0, 1))
    b.point(PLANE[0], [(0, canvas_of(*PLANE[1], W), 1.0)])
    b.T[0, 0, 3] = 0.01
    return b.build((0, 1), W)


def zero_weight(W):
    """Every weight 0: H = 0, lambda = 0, every solve fails; both rounds end on qmax == 10."""
    b = Builder(2)
    b.zero(W, (0, 1), w=0.0)
    b.T[0, 0, 3] = 0.01
    return b.build((0, 1), W)


def conflicting(W, zero_weight_points=True):
    """Key frame 0 free and 2 cm off, key frames 1, 2 and 3 fixed at the identity. Every weighted MapPoint is seen by 1, 2 and 3 at 40 px
    from a centre 10 px right of its projection, in three directions 120 degrees apart: round 1 moves the points to the centre and every
    weighted edge ends an outlier. With the zero-weight MapPoints (seen by key frames 0 and 1), round 2 keeps only zero-weight edges:
    H = 0, lambda = 0 and ten failed solves after the landmarks had a step. Without them every edge is an outlier and round 2 has nothing
    to optimize."""
    b = Builder(4)
    if zero_weight_points:
        b.zero(W, (0, 1), w=0.0)
    X, kp = zero_residual(W)
    for x, (u, v) in zip(X, kp):
        b.point(x, [(k, (u + 10.0 + 40.0 * math.cos(2 * math.pi * k / 3), v + 40.0 * math.sin(2 * math.pi * k / 3)), 1.0) for k in (1, 2, 3)])
    b.T[0, 0, 3] = 0.02
    return b.build((0, 1, 1, 1), W)


def sparse_vertices(W):
    """A MapPoint with a single edge, and a free key frame (2) that sees one MapPoint; key frame 0 free and rotated 1 degree."""
    b = Builder(3)
    b.zero(W, (0, 1))
    X, kp = zero_residual(W)
    b.point(X[3], [(0, kp[3], 1.0)])
    b.point(X[5], [(2, kp[5], 1.0), (1, kp[5], 1.0)])
    p = b.build((0, 1, 0), W)
    p["Tcw"][0] = rotated(p["Tcw"][0], 1.0, (0, 1, 0.3))
    return p


def lost_keyframe(W):
    """Key frames 0 and 1 fixed, 2 and 3 free and 1 cm off; the zero-residual MapPoints are seen by 0, 1 and 3 (key frame 1 with a residual
    floor of half a pixel, so that round 2 ends on nBad >= 3 well above rounding). Key frame 2 sees only the MapPoints at rig depth <= 0:
    its every edge fails the depth test after round 1, and the number of free poses drops from 2 to 1 between the rounds."""
    b = Builder(4)
    X, kp = zero_residual(W)
    for i, (x, (u, v)) in enumerate(zip(X, kp)):
        n = (0.5 * (-1) ** i, 0.25 * (-1) ** (i // 2))
        b.point(x, [(0, (u, v), 1.0), (1, (u + n[0], v + n[1]), 1.0), (3, (u, v), 1.0)] + ([(2, (u, v), 1.0)] if x[2] <= 0 else []))
    b.T[2, 0, 3] = 0.01; b.T[3, 1, 3] = 0.01
    return b.build((1, 1, 0, 0), W, its1=2)


def rotated(T, deg, axis, shift=(0, 0, 0)):
    T = np.asarray(T, np.float64).copy()
    ax = np.asarray(axis, np.float64); ax = ax / np.linalg.norm(ax)
    T[:3, :3] = synth._rodrigues(ax * math.radians(deg)) @ T[:3, :3]
    T[:3, 3] += shift
    return T.astype(np.float32)


def perturbed(p, deg, shift, seed):
    """Every free key frame's prior rotated by deg about a seeded axis and moved by shift (m) along another."""
    rng = np.random.default_rng(seed)
    p = dict(p); T = p["Tcw"].copy()
    for k in np.flatnonzero(p["kf_fixed"] == 0):
        T[k] = rotated(T[k], deg, rng.normal(size=3), shift * rng.normal(size=3) / math.sqrt(3))
    p["Tcw"] = T
    return p


SCHEDULE_ITS = ((5, 10), (0, 10), (5, 0), (1, 1))
# (seed, degrees, metres, outlier fraction). Priors much further off (12 or 25 degrees at these sizes) end in a flat valley where the sign of
# rho in the last iterations is decided by rounding, so a GPU summation order and the oracle's part ways there: not a test of the LM rules.
SCHEDULE = ((70, 4.0, 0.05, 0.1), (200, 8.0, 0.1, 0.3), (200, 0.3, 0.003, 0.0))


def window(W, seed, deg, shift, outliers):
    """A 5-key-frame synth.ba_problem window (key frame 0 fixed) whose free priors are rotated by deg and moved by shift."""
    p = synth.ba_problem(nKF=5, nMP=60, kmin=2, kmax=4, faceW=W, seed=seed, radius=1.5, outlier_frac=outliers)
    p["kf_fixed"][0] = 1
    return perturbed(p, deg, shift, seed + 100)


def schedule(W):
    """Windows with priors rotated and moved far enough that the 5 + 10 budget binds, trials get rejected and nBad >= 3 ends rounds (the
    last window starts 0.3 degrees off and stalls within round 1); each at every (its1, its2) of SCHEDULE_ITS."""
    out = []
    for j, sc in enumerate(SCHEDULE):
        p = window(W, *sc)
        for its in SCHEDULE_ITS:
            out.append(("schedule_%d_%d_%d" % (j, its[0], its[1]), problem(*args(p)[:7], W, its1=its[0], its2=its[1])))
    return out


# Stop flag raised after trial k. HOOKS run on window SCHEDULE[1]: after an accepted trial of round 1, inside round 2, and past the call's last
# trial (no effect).
HOOKS = (("accepted", 2), ("round2", 7), ("past_end", 1000))
# The rejected-trial stop. A MapPoint 5 cm in front of the rig, seen by key frame 0 (free, 1 cm off) at its projection and by key frame 1
# (fixed) 20 px to the right: its depth is barely constrained, and the third trial of round 1 overshoots and is rejected, far from
# convergence. The stop after it skips round 2, and the classification reads that rejected trial's errors. The weight of the MapPoint's key
# frame 1 edge (edge STRADDLE_EDGE, per face width) puts its chi2 above 5.991 at the rejected trial's state and below it at the restored
# state (by 20 % or more either way), so a classification from recomputed errors gets this edge wrong.
STRADDLE_EDGE, STRADDLE_K = 31, 3
STRADDLE_W = {650: 0.935064971446991, 450: 0.23564250767230988, 610: 0.7405559420585632}


def rejected_stop(W):
    b = Builder(2)
    b.zero(W, (0, 1))
    u, v = canvas_of(0, 0.5, 0.25, W)
    b.point(local_to_rig(0, 0.025, 0.0125, 0.05), [(0, (u, v), 1.0), (1, (u + 20.0, v), STRADDLE_W[W])])
    b.T[0, 0, 3] = 0.01
    return b.build((0, 1), W, stop_after_trials=STRADDLE_K)


def stop_scenes(W):
    p = window(W, *SCHEDULE[1])
    out = [("stop_%s" % name, problem(*args(p)[:7], W, stop_after_trials=k)) for name, k in HOOKS]
    out.append(("stop_rejected", rejected_stop(W)))
    return out


def all_scenes(W):
    named = [("stationary", stationary(W))]
    named += [("plane_fixed_%s" % where, plane_fixed(W, where)) for where in ("first", "middle", "last")]
    named += [("plane_free", plane_free(W)), ("zero_weight", zero_weight(W)), ("zero_weight_round2", conflicting(W)),
              ("all_outliers", conflicting(W, False)), ("lost_keyframe", lost_keyframe(W)),
              ("sparse_vertices", sparse_vertices(W))]
    named += schedule(W)
    named += stop_scenes(W)
    return named

"""The tracking kernels (cubemapslam_b200/csrc/track.cu) at the rules random scenes do not reach. Every answer is compared with the oracle,
exactly, through the host entries and the _dev entries (rows past every count filled with garbage), at face widths 650, 450 and 610 (not a
multiple of 50). The scenes are built here from synth.tracking_pair plus hand-placed key points and descriptors; test_scenes_reach_every_case
checks on the oracle's answers alone that each case is really there, and tests/test_oracle_projection.py / tests/test_oracle_frame_index.py
pin the oracle to the compiled reference on the scenes the reference can take.

k_frame_index (index_frames):
  key points on the face seams (x or y == W, 2W), the largest float below each seam (at W = 650, x = 1949.9999 lands in cell column
  150 % 50 = 0 of the right face), exact cell edges and the float below them; corner tiles, negative coordinates and >= 3W (zero ray, no
  cell); one cell holding 300 key points in shuffled slot order (listed ascending); n = 0, n = 257, n = stride = 4096, a count past the
  stride (clamped); ragged frames in one launch.
k_search_by_projection, mode 0 (last frame; last_batch) and mode 1 (local map; local_batch):
  ties at the least distance in one cell, across 32-cell chunks of one rectangle and across seam rectangles ("cell", "cells", "chunks",
  "rects": the first visited wins, never the lowest index or lane); mode 1: a tie at one level (ratio-rejected), at two levels (accepted),
  at distance 0 (accepted), a second best after the best (the else-if branch) and a second best equal to it at the best's level;
  TH_HIGH at 100 / 101; bestDist == nnratio * bestDist2 in float for nnratio 0.6, 0.75, 0.8, 0.9 (accepted) and one over (rejected);
  the window edge |kx - u| == radius (out) and one ulp inside (in); the level gates minL - 1 / maxL + 1; viewCos == float(0.998) (radius
  2.5: the float exceeds the double 0.998) and the float below it (radius 4); th = 1.0 and the float above it (radius_pair);
  mode 0 projection (proj_pair, TcwCur = I): camera z == cosFovTh (kept) and the float below (skipped), |x| == |z| and |y| == |z| rays
  (u or v == W is rejected, 0 is kept), points behind the camera inside and outside the field of view;
  taken slots: a slot holding an observed MapPoint is skipped, a slot matched by an observation-less MapPoint is taken again;
  rotation histogram (ori_pairs): a slot listed twice whose first / second / both listings fall in dropped bins, rotations at the rounding
  halves 6 + 12k (C round, half away from zero), a difference just below 0 that wraps to bin 30 = bin 0, 354 degrees, four equal bins (the
  first three win), max2 / max3 exactly 0.1 * max1 (kept) and below it (dropped);
  sizes (size_pairs): nQ = 0, no valid query, nQ = 13 (rounds of 8), nQ = nCur = 4096, more queries than features; mode 1 with 12 levels
  at factor 1.1.
k_gather_pose_inputs (gather_frames): ray z == cosFovTh (kept) and the float below (dropped), slots holding -1 and -2, 255 / 256 / 257 /
  4096 correspondences, and the rays == nullptr form."""
import ctypes as C

import numpy as np
import pytest

from cubemapslam_b200 import synth

G = 50                                                         # grid cells per face side
TILE = {0: (1, 1), 1: (0, 1), 2: (2, 1), 3: (1, 0), 4: (1, 2)}   # face -> canvas tile (column, row)
POPC = np.array([bin(i).count("1") for i in range(256)], np.int32)
F32 = np.float32
GARBAGE = 0xAB
TIE_DIST = 20
TH_LAST, TH_LOCAL = 15.0, 3.0
NNRATIOS = (0.6, 0.75, 0.8, 0.9)
WIDTHS = (650, 450, 610)


# ----------------------------------------------------------------------------------------------------------------- helpers
def KP():
    from oracle import KP_DTYPE
    return KP_DTYPE


def hamming(a, b):
    return int(POPC[np.bitwise_xor(a, b)].sum())


def flipped(d, bits):
    out = d.copy()
    for b in bits:
        out[b >> 3] ^= np.uint8(1 << (b & 7))
    return out


def cos_fov_th(fov_deg=190.0):
    """CamModelGeneral::SetCosFovTh: float argument, double cos, float result (every camera of the reference's settings has fov 190)."""
    a = F32(fov_deg) / F32(2) * (F32(3.1415926535897932384626) / F32(180))
    return F32(np.cos(np.float64(a)))


def level_tables(nlevels=8, factor=1.2):
    sc = np.ones(nlevels, F32)
    for lv in range(1, nlevels):
        sc[lv] = sc[lv - 1] * F32(factor)
    return sc, (F32(1.0) / (sc * sc)).astype(F32)


def cell_of(x, y, W):
    """Frame::PosInGrid on a 3W-wide canvas: (face, column, row), face None off the five faces."""
    x, y = F32(x), F32(y)
    face = {(0, 1): 1, (1, 0): 3, (1, 1): 0, (1, 2): 4, (2, 1): 2}.get((int(np.floor(x / F32(W))), int(np.floor(y / F32(W)))))
    inv = F32(3 * G) / F32(3 * W)
    return face, int(x * inv) % G, int(y * inv) % G


def ref_safe(x, y, W):
    """The reference's debug build asserts in PosInGrid when the key point's cell corner lies on another face than the key point."""
    x, y = F32(x), F32(y)
    f = cell_of(x, y, W)[0]
    inv = F32(3 * G) / F32(3 * W); ln = F32(3 * W) / F32(3 * G)
    return f is not None and cell_of(F32(int(x * inv) * ln), F32(int(y * inv) * ln), W)[0] == f


def visit_cells(oracle, u, v, r, W):
    """The cells GetFeaturesInArea visits, in its order: (rectangle, position in the rectangle, face, column, row)."""
    out = []
    for k, (f, x0, x1, y0, y1) in enumerate(oracle.area_rects(u, v, r, W, W)):
        x0, x1, y0, y1 = max(0, x0), min(G - 1, x1), max(0, y0), min(G - 1, y1)
        ci = 0
        for ix in range(x0, x1 + 1):
            for iy in range(y0, y1 + 1):
                out.append((k, ci, int(f), ix, iy)); ci += 1
    return out


def point_in_cell(f, ix, iy, u, v, W, margin=0.6, far=False):
    """The point of cell (f, ix, iy) nearest to (u, v) (farthest with far=True), `margin` pixels inside the cell."""
    cl = W / G; c, rw = TILE[f]
    x0, y0 = c * W + ix * cl + margin, rw * W + iy * cl + margin
    x1, y1 = x0 + cl - 2 * margin, y0 + cl - 2 * margin
    if far:
        x, y = (x0 if abs(x0 - u) > abs(x1 - u) else x1), (y0 if abs(y0 - v) > abs(y1 - v) else y1)
    else:
        x, y = min(max(float(u), x0), x1), min(max(float(v), y0), y1)
    return (F32(x), F32(y)) if cell_of(x, y, W) == (f, ix, iy) else None


def in_window(x, y, u, v, r):
    return abs(F32(x) - F32(u)) < r and abs(F32(y) - F32(v)) < r


def ratio_pair(nn):
    """(a, b), a <= 100 < 256, with a == nnratio * b exactly in float: the ratio test's boundary."""
    out = [(a, b) for b in range(110, 1, -1) for a in range(0, 101) if F32(F32(nn) * F32(b)) == F32(a)]
    return max(out)


def garbage(shape, dtype):
    dtype = np.dtype(dtype)
    return np.full(tuple(shape) + (dtype.itemsize,), GARBAGE, np.uint8).view(dtype)[..., 0].copy()


def bits(a):
    return np.ascontiguousarray(a).view(np.uint8)


def to_dev(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a).reshape(-1).view(np.uint8).copy()).cuda()


def from_dev(t, like):
    return t.cpu().numpy().view(like.dtype).reshape(like.shape)


# ----------------------------------------------------------------------------------------------------------------- search scenes
class Pair:
    """One frame of a batched projection search: the searched key points, and the queries (mode 0: LastFrame features with their
    MapPoints, seen through TcwCur = I; mode 1: local MapPoints with projection, predicted level and viewing cosine). `cases` lists the
    hand-placed queries with the final match value they must leave in their key points' slots (`want`: slot -> value, -1 none)."""

    def __init__(self, oracle, W, mode, seed=0):
        self.oracle, self.W, self.mode = oracle, W, mode
        self.rng = np.random.default_rng(900 + seed)
        self.k, self.d, self.taken = [], [], []
        self.q = []
        self.cases = []
        self.used = []

    def desc(self):
        return self.rng.integers(0, 256, 32, dtype=np.uint8)

    def add_kp(self, x, y, oct_, d, angle=0.0, taken=0):
        self.k.append((float(x), float(y), 31.0, float(angle), 0.0, int(oct_), -1)); self.d.append(d); self.taken.append(int(taken))
        return len(self.k) - 1

    def add_q(self, d, oct_=0, X=(0, 0, 1), angle=0.0, uv=(0, 0), vcos=0.99, obs=1, valid=1):
        self.q.append(dict(d=d, oct=int(oct_), X=np.asarray(X, F32), angle=F32(angle), uv=uv, vcos=F32(vcos), obs=int(obs), valid=int(valid)))
        return len(self.q) - 1

    def mp_at(self, tx, ty, oct_, d=None, vcos=0.99, obs=1, angle=0.0, depth=5.0):
        """A query projecting at canvas pixel (u, v) near (tx, ty): (index, u, v, descriptor)."""
        d = self.desc() if d is None else d
        if self.mode == 0:
            X = (synth._pixel_to_ray(float(tx), float(ty), self.W) * depth).astype(F32)
            uv, face = self.oracle.ray_to_cubemap(X, self.W, self.W)
            assert face[0] >= 0
            u, v = F32(uv[0, 0]), F32(uv[0, 1])
            return self.add_q(d, oct_, X=X, angle=angle, obs=obs), u, v, d
        u, v = F32(tx), F32(ty)
        return self.add_q(d, oct_, uv=(u, v), vcos=vcos, obs=obs), u, v, d

    def radius(self, oct_, th, scale, vcos=0.99):
        if self.mode == 0:
            return F32(F32(th) * scale[oct_])
        r = F32(2.5 if np.float64(F32(vcos)) > 0.998 else 4.0)
        if F32(th) != F32(1.0):
            r = F32(r * F32(th))
        return F32(r * scale[oct_])

    def case(self, kind, q, want, **kw):
        self.cases.append(dict(kind=kind, q=q, want=want, **kw))

    def background(self, n, seed, keep_out=90.0):
        """synth.tracking_pair's current frame and its queries, none within keep_out pixels of a hand-placed case."""
        s = synth.tracking_pair(seed, n=n, faceW=self.W)
        far = lambda x, y: all((x - a) ** 2 + (y - b) ** 2 > max(keep_out, e) ** 2 for a, b, e in self.used)
        for i, kp in enumerate(s["kCur"]):
            if far(kp["x"], kp["y"]):
                self.add_kp(kp["x"], kp["y"], kp["octave"], s["dCur"][i], kp["angle"], s["curTaken"][i])
        if self.mode == 0:
            uv, face = self.oracle.ray_to_cubemap(s["Xw"], self.W, self.W)
            for i in range(len(s["Xw"])):
                if face[i] < 0 or far(*uv[i]):
                    self.add_q(s["dLast"][i], s["kLast"]["octave"][i], X=s["Xw"][i], angle=s["kLast"]["angle"][i], obs=s["mpObs"][i], valid=s["hasMP"][i])
        else:
            rng = np.random.default_rng(seed)
            for i in np.nonzero(s["src"] >= 0)[0]:
                u, v = F32(s["kCur"]["x"][i] + rng.normal(0, 2)), F32(s["kCur"]["y"][i] + rng.normal(0, 2))
                if far(u, v):
                    self.add_q(s["dLast"][s["src"][i]], int(np.clip(s["kCur"]["octave"][i] + rng.integers(0, 2), 0, 7)), uv=(u, v),
                               vcos=rng.choice(np.array([0.9999, 0.99, 0.7], F32)), obs=int(rng.random() < 0.9), valid=int(rng.random() < 0.9))

    def arrays(self):
        K = KP()
        k = np.array(self.k, K) if self.k else np.zeros(0, K)
        d = np.stack(self.d) if self.d else np.zeros((0, 32), np.uint8)
        n = len(self.q)
        kl = np.zeros(n, K); kl["x"] = kl["y"] = 1.5 * self.W; kl["size"] = 31; kl["class_id"] = -1
        kl["octave"] = [q["oct"] for q in self.q]; kl["angle"] = [q["angle"] for q in self.q]
        return dict(k=k, d=d, taken=np.array(self.taken, np.uint8), kl=kl, valid=np.array([q["valid"] for q in self.q], np.uint8),
                    Xw=np.array([q["X"] for q in self.q], F32).reshape(-1, 3), dq=np.array([q["d"] for q in self.q], np.uint8).reshape(-1, 32),
                    obs=np.array([q["obs"] for q in self.q], np.int32), proj=np.array([q["uv"] for q in self.q], F32).reshape(-1, 2),
                    level=kl["octave"].astype(np.int32), vcos=np.array([q["vcos"] for q in self.q], F32), T=np.eye(4, dtype=F32), W=self.W)


def spots(W, step, corner=False, margin=70):
    """Candidate query pixels: face interiors on a lattice, or 2..8 px inside every face corner."""
    out = []
    for f, (c, r) in TILE.items():
        if corner:
            for ox in (0, 1):
                for oy in (0, 1):
                    for dx, dy in ((3.1, 3.3), (5.2, 2.4), (2.3, 6.1), (6.6, 5.7), (1.7, 1.9), (4.4, 7.3)):
                        out.append((c * W + (W - dx if ox else dx), r * W + (W - dy if oy else dy)))
        else:
            for x in np.arange(margin, W - margin, step):
                for y in np.arange(margin, W - margin, step):
                    out.append((c * W + x, r * W + y))
    return out


class Spots:
    def __init__(self, P, sep):
        self.P, self.sep = P, sep
        self.it = iter(spots(P.W, 23.0))

    def free(self, x, y):
        return all((x - a) ** 2 + (y - b) ** 2 > max(self.sep, e) ** 2 for a, b, e in self.P.used)

    def next(self):
        for x, y in self.it:
            if self.free(x, y):
                self.P.used.append((x, y, self.sep))
                return x, y
        raise AssertionError("out of spots")


def near(P, u, v, dx, dy):
    """A key point position (dx, dy) pixels from (u, v), in the same cell as (u, v)."""
    f, ix, iy = cell_of(u, v, P.W)
    return point_in_cell(f, ix, iy, u + dx, v + dy, P.W)


def tie_kinds(P, u, v, r, oct_):
    """Pairs of reachable cells (earlier, later in the visiting order) for each tie arrangement, the later one on a lower lane."""
    reach = []
    for k, ci, f, ix, iy in visit_cells(P.oracle, u, v, r, P.W):
        p = point_in_cell(f, ix, iy, u, v, P.W)
        if p is not None and in_window(p[0], p[1], u, v, r):
            reach.append((k, ci, f, ix, iy, p))
    kinds = {}
    for a, p in enumerate(reach):
        for q in reach[a + 1:]:
            if p[0] == q[0] and p[1] // 32 == q[1] // 32 and p[1] != q[1]:
                kinds.setdefault("cells", (p, q))
            if p[0] == q[0] and p[1] // 32 < q[1] // 32 and q[1] % 32 < p[1] % 32:
                kinds.setdefault("chunks", (p, q))
            if p[0] == 1 and q[0] == 2 and q[1] % 32 < p[1] % 32:
                kinds.setdefault("rects", (p, q))
    return kinds


def add_ties(P, th, scale, lvl, late_lvl):
    """The four tie arrangements at TIE_DIST around level-lvl queries (radius 43-54 px: 7 x 7 cells and more). The later-visited tied key
    point is appended first (octave late_lvl) and twelve fillers precede the earlier one in its cell, so the winner is neither the lowest
    index nor the lowest lane."""
    want = {"cells": 1, "chunks": 1, "rects": 1, "cell": 1}
    r = P.radius(lvl, th, scale)
    for corner in (True, False):
        for tx, ty in spots(P.W, 37.0, corner):
            if not any(want.values()):
                break
            if not all((tx - a) ** 2 + (ty - b) ** 2 > (2.2 * r) ** 2 for a, b, _ in P.used):
                continue
            save = len(P.q)
            q, u, v, D = P.mp_at(tx, ty, lvl)
            kinds = tie_kinds(P, u, v, r, lvl)
            kind = next((k for k in (("rects",) if corner else ("chunks", "cells")) if want[k] and k in kinds), None)
            if kind is None and want["cell"] and not corner and near(P, u, v, 0.5, 0.2) is not None:
                kind = "cell"
            if kind is None:
                del P.q[save:]
                continue
            want[kind] -= 1; P.used.append((tx, ty, r + 40))
            b = P.rng.permutation(256)
            if kind == "cell":
                pts = [near(P, u, v, dx, dy) for dx, dy in ((0.5, 0.2), (-0.4, 0.6), (0.3, -0.5))]
                kps = [P.add_kp(x, y, (lvl, late_lvl, lvl)[i], flipped(D, b[TIE_DIST * i:TIE_DIST * (i + 1)])) for i, (x, y) in enumerate(pts)]
                expect = kps[0]
            else:
                p, qq = kinds[kind]
                late = P.add_kp(*qq[5], late_lvl, flipped(D, b[:TIE_DIST]))
                for _ in range(12):
                    P.add_kp(*point_in_cell(*p[2:5], u, v, P.W, far=True), lvl, P.desc())
                expect = P.add_kp(*p[5], lvl, flipped(D, b[TIE_DIST:2 * TIE_DIST]))
                kps = [late, expect]
            P.case(kind, q, {s: (q if s == expect else -1) for s in kps}, u=u, v=v, r=r, lvl=lvl, kps=kps, dist=TIE_DIST)
    assert not any(want.values()), want


def add_local_rules(P, sp, D_of, nn):
    """Mode 1, level 0 (radius 12 px): ties at one level, at distance 0, the else-if branch, a second best equal to it, the ratio boundary."""
    a, b = ratio_pair(nn)
    accept = lambda x, y: not (F32(x) > F32(F32(nn) * F32(y)))
    rules = [("tie_same_level", ((20, 0), (20, 0)), None), ("tie_zero", ((0, 0), (0, 0)), 0), ("tie_two_levels", ((20, 1), (20, 0)), 0),
             ("else_if", ((30, 0), (31, 0)), None), ("second_equal", ((30, 1), (31, 0), (31, 1)), 0),
             ("ratio_equal", ((a, 0), (b, 0)), 0 if accept(a, b) else None), ("ratio_over", ((a + 1, 0), (b, 0)), None)]
    for kind, ks, win in rules:
        tx, ty = sp.next()
        q, u, v, D = P.mp_at(tx, ty, 1 if kind in ("tie_two_levels", "second_equal") else 0)
        bt = P.rng.permutation(256); kps = []
        for j, (dist, oct_) in enumerate(ks):
            x, y = near(P, u, v, (0.3, -0.4, 0.2)[j], (0.2, 0.3, -0.5)[j])
            kps.append(P.add_kp(x, y, oct_, flipped(D, bt[:dist]) if j == 0 else flipped(D, bt[200 - dist:200] if dist else [])))
        exp = None if win is None else kps[win]
        P.case(kind, q, {s: (q if s == exp else -1) for s in kps}, u=u, v=v, kps=kps)


def add_common(P, sp, th, scale):
    """Both modes: TH_HIGH, the window edge, the level gates, taken slots."""
    for dist in (100, 101):
        tx, ty = sp.next()
        q, u, v, D = P.mp_at(tx, ty, 0)
        s = P.add_kp(*near(P, u, v, 0.4, -0.3), 0, flipped(D, P.rng.permutation(256)[:dist]))
        P.case("th_%d" % dist, q, {s: q if dist == 100 else -1}, kps=[s])
    # the window edge at level 0: the best key point exactly at the radius on one axis (out) or one ulp inside (in)
    variants = [(ax, sg, ulp) for ulp in (False, True) for ax in (0, 1) for sg in (1, -1)]
    for ax, sg, ulp in variants:
        while True:
            tx, ty = sp.next()
            save = len(P.q)
            q, u, v, D = P.mp_at(tx, ty, 0)
            r = P.radius(0, th, scale)
            c = (u, v)[ax]; e = F32(c + F32(sg) * r)
            if abs(F32(e - c)) == r:
                break
            del P.q[save:]
        if ulp:
            e = np.nextafter(e, c)
        x, y = (e, v) if ax == 0 else (u, e)
        bt = P.rng.permutation(256)
        inside = P.add_kp(u + F32(0.25 * r * -sg * (ax == 0)), v + F32(0.25 * r * -sg * (ax == 1)), 0, flipped(D, bt[:30]))
        edge = P.add_kp(x, y, 0, flipped(D, bt[30:40]))
        exp = edge if ulp else inside
        P.case("ulp_inside" if ulp else "edge", q, {inside: q if exp == inside else -1, edge: q if exp == edge else -1}, u=u, v=v, r=r, kps=[inside, edge])
    # level gates: (octave, distance) around a query at octave / level lvl; the gate drops the better descriptors
    gates = {0: {(0, 0): ((2, 5), (1, 10), (0, 20)), (0, 3): ((1, 5), (5, 6), (4, 10), (2, 12))},
             1: {(1, 0): ((1, 5), (0, 20)), (1, 3): ((1, 5), (4, 6), (2, 10), (3, 20))}}
    for (_, lvl), ks in gates[P.mode].items():
        tx, ty = sp.next()
        q, u, v, D = P.mp_at(tx, ty, lvl)
        bt = P.rng.permutation(256); kps = []
        for j, (o, dist) in enumerate(ks):
            kps.append(P.add_kp(*near(P, u, v, 0.3 * np.cos(j * 1.7), 0.3 * np.sin(j * 1.7)), o, flipped(D, bt[:dist])))
        best = min((dist, s) for s, (o, dist) in zip(kps, ks) if lvl - 1 <= o <= (lvl + 1 if P.mode == 0 else lvl))[1]
        P.case("level", q, {s: q if s == best else -1 for s in kps}, lvl=lvl, kps=kps)
    # taken: the best slot holds an observed MapPoint; an observation-less query's slot taken again by a later query
    tx, ty = sp.next()
    q, u, v, D = P.mp_at(tx, ty, 0)
    bt = P.rng.permutation(256)
    s0 = P.add_kp(*near(P, u, v, 0.2, 0.3), 0, flipped(D, bt[:5]), taken=1)
    s1 = P.add_kp(*near(P, u, v, -0.3, 0.2), 0, flipped(D, bt[5:25]))
    P.case("taken", q, {s0: -1, s1: q}, kps=[s0, s1])
    tx, ty = sp.next()
    qa, u, v, D = P.mp_at(tx, ty, 0, obs=0)
    qb = P.mp_at(tx, ty, 0, d=D, obs=1, depth=7.0)[0]
    qc = P.mp_at(tx, ty, 0, d=D, obs=1, depth=9.0)[0]
    bt = P.rng.permutation(256)
    s0 = P.add_kp(*near(P, u, v, 0.1, 0.1), 0, flipped(D, bt[:5]))
    s1 = P.add_kp(*near(P, u, v, -0.2, 0.3), 0, flipped(D, bt[5:20]))
    P.case("retaken", qb, {s0: qb, s1: qc}, kps=[s0, s1], first=qa, later=qc)


def main_pair(oracle, W, mode, nn=0.8, seed=0):
    """Ties, thresholds, window edges, level gates, taken slots (and in mode 1 the ratio rules), among synth.tracking_pair's features."""
    P = Pair(oracle, W, mode, seed)
    scale, _ = level_tables()
    th = TH_LAST if mode == 0 else TH_LOCAL
    add_ties(P, th, scale, 7, 7 if mode == 0 else 6)
    sp = Spots(P, 60.0)
    add_common(P, sp, th, scale)
    if mode == 1:
        add_local_rules(P, sp, None, nn)
        for kind, vc in (("vcos_998", F32(0.998)), ("vcos_below", np.nextafter(F32(0.998), F32(0))), ("vcos_9999", F32(0.9999))):
            tx, ty = sp.next()
            q, u, v, D = P.mp_at(tx, ty, 0, vcos=vc)
            bt = P.rng.permutation(256)
            a = P.add_kp(u + F32(9.5), v + F32(0.2), 0, flipped(D, bt[:10]))      # inside radius 12, outside radius 7.5
            b = P.add_kp(u + F32(0.4), v - F32(0.3), 0, flipped(D, bt[10:40]))
            exp = a if np.float64(vc) <= 0.998 else b
            P.case(kind, q, {a: q if exp == a else -1, b: q if exp == b else -1}, kps=[a, b], vcos=vc)
    P.background(1500, seed)
    return P


def radius_pair(oracle, W, th):
    """Mode 1, th = 1.0 (radius 2.5, no factor) or the float above 1.0 (radius 2.5000002): a key point exactly 2.5 px away."""
    P = Pair(oracle, W, 1, 7)
    P.th = th
    sp = Spots(P, 40.0)
    scale, _ = level_tables()
    for ax in (0, 1):
        while True:
            tx, ty = sp.next()
            save = len(P.q)
            q, u, v, D = P.mp_at(tx, ty, 0, vcos=0.9999)
            c = (u, v)[ax]; e = F32(c + F32(2.5))
            if F32(e - c) == F32(2.5):
                break
            del P.q[save:]
        x, y = (e, v) if ax == 0 else (u, e)
        bt = P.rng.permutation(256)
        a = P.add_kp(x, y, 0, flipped(D, bt[:10]))
        b = P.add_kp(u - F32(0.5), v - F32(0.5), 0, flipped(D, bt[10:40]))
        exp = a if F32(th) != F32(1.0) else b
        P.case("th_one" if exp == b else "th_above_one", q, {a: q if exp == a else -1, b: q if exp == b else -1}, kps=[a, b],
               r=P.radius(0, th, scale, 0.9999))
    return P


def proj_pair(oracle, W, cth):
    """Mode 0 through TcwCur = I: camera z at the field-of-view threshold, rays on the face seams, points behind the camera."""
    P = Pair(oracle, W, 0, 8)
    below = np.nextafter(cth, F32(-1))
    pts = [("fov_keep", (1, 0.2, cth), True), ("fov_skip", (1, -0.35, below), False), ("seam_x_pos", (2, 0.3, 2), False),
           ("seam_x_neg", (-2, -0.3, 2), True), ("seam_y_pos", (0.3, 2, 2), False), ("seam_y_neg", (-0.3, -2, 2), True),
           ("behind_keep", (1, -0.1, -0.05), True), ("behind_skip", (1, 0.3, -0.5), False)]
    for kind, X, kept in pts:
        X = np.array(X, F32)
        D = P.desc()
        q = P.add_q(D, 0, X=X)
        uv, face = oracle.ray_to_cubemap(X, W, W)
        u, v = float(uv[0, 0]), float(uv[0, 1])
        if kind == "seam_x_pos":
            u, v = 2 * W + 0.4, W + v          # where u == W would land (column 0 of the right face)
        elif kind == "seam_y_pos":
            u, v = W + u, 2 * W + 0.4          # v == W: row 0 of the lower face
        else:
            assert face[0] >= 0, kind
        s = P.add_kp(F32(u + 0.3), F32(v + 0.2), 0, flipped(D, P.rng.permutation(256)[:10]))
        P.case(kind, q, {s: q if kept else -1}, kps=[s], X=X)
    return P


def rot_bin(a, b):
    """The rotation-histogram bin of a match: float difference wrapped into [0, 360), times 1/12 in float, C round (half away from zero)."""
    rot = F32(F32(a) - F32(b))
    if rot < 0:
        rot = F32(rot + F32(360))
    p = F32(rot * (F32(1) / F32(12)))
    return int(np.floor(p + 0.5)) % 30


def ori_pairs(oracle, W):
    """Mode 0, one histogram per pair: (scenario, {bin or rotation: count}, extra cases). Every query has its own key point 60 px from the
    others (radius 15); rotation = last angle - current angle."""
    out = []
    scen = [("halves", {1: 10, 3: 10, 5: 10}, ("rot6", "rot30", "rot54"), ()),
            ("dominant0", {0: 16}, ("wrap", "rot354", "rot342", "double_first_out", "double_second_out", "double_both_out"), (29, 7, 9, 11, 13)),
            ("four_equal", {2: 5, 4: 5, 6: 5, 8: 5}, (), (8,)),
            ("max2_tenth", {0: 20, 5: 2, 9: 1}, (), (9,)),
            ("max3_tenth", {0: 20, 5: 4, 9: 2, 12: 1}, (), (12,)),
            ("max2_below", {0: 30, 5: 2, 9: 2}, (), (5, 9))]
    for si, (name, bins, extra, drop) in enumerate(scen):
        P = Pair(oracle, W, 0, 20 + si)
        P.name = name
        sp = Spots(P, 45.0)

        def one(last_angle, cur_angle, kind, obs=1):
            tx, ty = sp.next()
            q, u, v, D = P.mp_at(tx, ty, 0, angle=last_angle, obs=obs)
            s = P.add_kp(*near(P, u, v, 0.3, 0.2), 0, flipped(D, P.rng.permutation(256)[:10]), angle=cur_angle)
            P.case(kind, q, {s: -1 if rot_bin(last_angle, cur_angle) in drop else q}, kps=[s], rot=(F32(last_angle), F32(cur_angle)))
            return q, s
        for b, n in bins.items():
            for _ in range(n):
                one(F32(12 * b), 0.0, "bin%d" % b)
        for kind in extra:
            if kind.startswith("rot"):
                one(F32(int(kind[3:])), 0.0, kind)
            elif kind == "wrap":
                one(F32(10.0), np.nextafter(F32(10.0), F32(11.0)), kind)
            else:
                first_bin, second_bin = {"double_first_out": (7, 0), "double_second_out": (0, 9), "double_both_out": (11, 13)}[kind]
                tx, ty = sp.next()
                qa, u, v, D = P.mp_at(tx, ty, 0, angle=F32(12 * first_bin), obs=0)
                qb = P.mp_at(tx, ty, 0, d=D, angle=F32(12 * second_bin), obs=1, depth=7.0)[0]
                s = P.add_kp(*near(P, u, v, 0.3, 0.2), 0, flipped(D, P.rng.permutation(256)[:10]))
                P.case(kind, qb, {s: -1}, kps=[s], first=qa, bins=(first_bin, second_bin))
        out.append(P)
    return out


def size_pairs(oracle, W, mode):
    """No queries, no valid query, 13 queries, 4096 queries on 4096 features, more queries than features."""
    out = []
    for kind, n, nk, nq in (("nq0", 300, None, 0), ("none_valid", 300, None, None), ("nq13", 0, None, None), ("full", 4096, 4096, 4096), ("more_q", 3000, 600, None)):
        P = Pair(oracle, W, mode, 40 + len(out))
        P.name = kind
        if kind == "nq13":
            sp = Spots(P, 45.0)
            for _ in range(13):
                tx, ty = sp.next()
                q, u, v, D = P.mp_at(tx, ty, 0)
                P.add_kp(*near(P, u, v, 0.3, 0.2), 0, flipped(D, P.rng.permutation(256)[:10]))
        else:
            P.background(4600 if kind == "full" else n, 40 + len(out))
            if nk is not None:
                del P.k[nk:], P.d[nk:], P.taken[nk:]
                assert len(P.k) == nk
            if kind == "full":
                while len(P.q) < 4096:
                    P.q.append(dict(P.q[len(P.q) % 500]))
                del P.q[4096:]
            if kind == "none_valid":
                for q in P.q:
                    q["valid"] = 0
            if nq == 0:
                P.q = []
        out.append(P)
    return out


def last_batch(oracle, W):
    cth = cos_fov_th()
    return [main_pair(oracle, W, 0), proj_pair(oracle, W, cth)] + ori_pairs(oracle, W) + size_pairs(oracle, W, 0)


def local_batch(oracle, W, nn):
    return [main_pair(oracle, W, 1, nn=nn, seed=1)] + size_pairs(oracle, W, 1)


def stack(pairs, pad=0):
    """Pad the pairs' arrays to common strides (+pad rows) with garbage: the batched layout of the host and _dev entries."""
    K = KP()
    A = [p.arrays() for p in pairs]
    P = len(A)
    cs = max(1, max(len(a["k"]) for a in A)) + pad; qs = max(1, max(len(a["kl"]) for a in A)) + pad
    cs, qs = min(cs, 4096), min(qs, 4096)
    out = dict(k=garbage((P, cs), K), d=garbage((P, cs, 32), np.uint8), taken=garbage((P, cs), np.uint8), kl=garbage((P, qs), K),
               valid=garbage((P, qs), np.uint8), Xw=garbage((P, qs, 3), F32), dq=garbage((P, qs, 32), np.uint8), obs=garbage((P, qs), np.uint8),
               proj=garbage((P, qs, 2), F32), level=garbage((P, qs), np.int32), vcos=garbage((P, qs), F32),
               T=np.stack([a["T"] for a in A]), nC=np.array([len(a["k"]) for a in A], np.int32), nQ=np.array([len(a["kl"]) for a in A], np.int32))
    for i, a in enumerate(A):
        n, m = len(a["k"]), len(a["kl"])
        out["k"][i, :n] = a["k"]; out["d"][i, :n] = a["d"]; out["taken"][i, :n] = a["taken"]
        for key in ("kl", "valid", "Xw", "dq", "proj", "level", "vcos"):
            out[key][i, :m] = a[key]
        out["obs"][i, :m] = a["obs"] > 0
    return A, out


def oracle_search(oracle, a, mode, cth=None, check_ori=True, nn=0.8, th=None, nlevels=8, factor=1.2):
    scale, _ = level_tables(nlevels, factor)
    g = oracle.FrameGrid(a["k"], a["W"], a["W"])
    if mode == 0:
        return g.search_by_projection_last(a["d"], a["T"], scale, a["kl"], a["valid"], a["Xw"], a["dq"], a["obs"], a["taken"], cth, TH_LAST if th is None else th,
                                           check_ori)
    return g.search_by_projection_local(a["d"], scale, a["valid"], a["proj"], a["level"], a["vcos"], a["dq"], a["obs"], a["taken"], TH_LOCAL if th is None else th, nn)


# ----------------------------------------------------------------------------------------------------------------- frame index scenes
def seam_points(W):
    """Key points on the seams, the float below each seam, exact cell edges and the float below them, plus off-face points."""
    Wf = F32(W)
    xs = []
    for k in (1, 2, 3):
        s = F32(k * W)
        xs += [s, np.nextafter(s, F32(0))]
    inv = F32(3 * G) / F32(3 * W)
    for c in (1, 7, 25, 49, 51, 74, 99, 101, 149):          # the first float of cell column c, and the float below it
        x = F32(c * W / G)
        while int(x * inv) >= c:
            x = np.nextafter(x, F32(0))
        while int(x * inv) < c:
            x = np.nextafter(x, F32(1e9))
        xs += [x, np.nextafter(x, F32(0))]
    mids = [F32(0.5 * W + 0.37), F32(1.5 * W + 0.41), F32(2.5 * W - 0.29)]
    pts = [(x, y) for x in xs for y in mids] + [(y, x) for x in xs for y in mids]
    off = [(F32(3.0), F32(4.0)), (F32(2 * W + 10.5), F32(2 * W + 20.25)), (F32(W - 0.5), F32(0.5)), (F32(2.5 * W), F32(2.9 * W)),
           (F32(-0.5), F32(1.5 * W)), (F32(1.5 * W), F32(-1e-3)), (F32(3 * W), F32(1.5 * W)), (F32(1.5 * W), F32(3 * W)), (F32(5 * W), F32(1.2 * W)),
           (F32(-3 * W), F32(-2 * W))]
    return pts + off


def index_frames(W, with_off=True, seed=0):
    """(key points, count) of a ragged batch: seams and cell edges (+ off-face points), a 300-key-point cell in shuffled slot order,
    n = 0, n = 257, n = 4096 = stride, and a count past the stride."""
    K = KP()
    rng = np.random.default_rng(seed)

    def kps(pts):
        k = np.zeros(len(pts), K); k["size"] = 31; k["class_id"] = -1
        k["x"] = [p[0] for p in pts]; k["y"] = [p[1] for p in pts]; k["octave"] = rng.integers(0, 8, len(pts))
        return k

    def on_faces(n):
        pts = []
        while len(pts) < n:
            c, r = TILE[int(rng.integers(0, 5))]
            pts.append((c * W + rng.uniform(0, W), r * W + rng.uniform(0, W)))
        return pts
    sp = [p for p in seam_points(W) if with_off or ref_safe(p[0], p[1], W)]
    f0 = kps([sp[i] for i in rng.permutation(len(sp))])
    cl = W / G
    crowd = [(W + 20 * cl + rng.uniform(0.05, cl - 0.05), W + 31 * cl + rng.uniform(0.05, cl - 0.05)) for _ in range(300)]
    f1 = kps([p for i, p in sorted(zip(rng.permutation(1000), crowd + on_faces(700)))])
    frames = [(f0, len(f0)), (f1, 1000), (kps([]), 0), (kps(on_faces(257)), 257), (kps(on_faces(4096)), 4096)]
    k5 = kps(on_faces(4096))
    frames.append((k5, 5000))                                  # clamped to the stride
    return frames


# ----------------------------------------------------------------------------------------------------------------- gather scenes
def pose_inputs_reference(match, kps, rays, Xw_last, inv_level_sigma2, cos_fov):
    """The correspondence loop of Optimizer::PoseOptimization: features in slot order, a feature whose ray leaves the field of view
    skipped, only slots holding a MapPoint taken, the world point of that MapPoint and mvInvLevelSigma2[kp.octave] as the weight."""
    Xw, kp, w = [], [], []
    for i in range(len(kps)):
        if rays is not None and rays[i, 2] < cos_fov:
            continue
        if match[i] >= 0:
            Xw.append(Xw_last[match[i]]); kp.append((kps["x"][i], kps["y"][i])); w.append(inv_level_sigma2[kps["octave"][i]])
    return np.array(Xw, F32).reshape(-1, 3), np.array(kp, F32).reshape(-1, 2), np.array(w, F32)


def gather_frames(oracle, W, cth):
    """(kCur, match, rays, Xw_last) per frame: 255, 256, 257 and 4096 correspondences, a frame mixing -1 / -2 slots with rays at exactly
    cosFovTh and the float below it, and an empty frame."""
    K = KP()
    rng = np.random.default_rng(3)
    out = []
    for kind, n, nm in (("c255", 600, 255), ("c256", 256, 256), ("c257", 1000, 257), ("c4096", 4096, 4096), ("mixed", 3000, None), ("empty", 0, 0)):
        k = np.zeros(n, K); k["size"] = 31; k["class_id"] = -1; k["octave"] = rng.integers(0, 8, n)
        for i in range(n):
            c, r = TILE[int(rng.integers(0, 5))]
            k["x"][i], k["y"][i] = c * W + rng.uniform(0, W), r * W + rng.uniform(0, W)
        rays = oracle.key_point_rays(k, W, W)[0]
        rays[:, 2] = np.maximum(rays[:, 2], F32(0.0))              # every ray inside the field of view but the ones placed below
        nl = 3500
        Xw = rng.normal(0, 3, (nl, 3)).astype(F32)
        match = np.full(n, -1, np.int32)
        if nm is None:
            match[:] = np.where(rng.random(n) < 0.6, rng.choice([-1, -2], n), rng.integers(0, nl, n))
            z = rng.permutation(n)
            rays[z[:40], 2] = cth                                   # kept
            rays[z[40:80], 2] = np.nextafter(cth, F32(-1))          # dropped
            match[z[:80]] = rng.integers(0, nl, 80)
        else:
            match[rng.permutation(n)[:nm]] = rng.integers(0, nl, nm)
            match[match < 0] = rng.choice([-1, -2], int((match < 0).sum()))
        out.append(dict(kind=kind, k=k, match=match, rays=rays, Xw=Xw))
    return out


# ----------------------------------------------------------------------------------------------------------------- the cases are reached
def test_scenes_reach_every_case(oracle):
    """On the oracle's answers alone, at every face width: each hand-placed case leaves the match it was built for, ties are won by the
    first visited key point (neither the lowest index nor the lowest lane) across a chunk boundary and across seam rectangles, the window
    edge is exact, the ratio boundary is exact in float, viewCos(0.998) selects radius 2.5, the projections sit exactly on the field-of-view
    threshold and the seams, the histogram lists a slot twice and clears it, the rotation halves round away from zero, four equal bins keep
    the first three; the frame index puts 1949.9999 in column 0 of the right face and leaves off-face points in no cell."""
    cth = cos_fov_th()
    scale, _ = level_tables()
    for W in WIDTHS:
        seen = set()
        for mode in (0, 1):
            batches = [last_batch(oracle, W)] if mode == 0 else [local_batch(oracle, W, nn) for nn in NNRATIOS] + [[radius_pair(oracle, W, th)] for th in (1.0, np.nextafter(F32(1), F32(2)))]
            for bi, pairs in enumerate(batches):
                for P in pairs:
                    a = P.arrays()
                    th = getattr(P, "th", None)
                    nn = NNRATIOS[bi] if mode == 1 and bi < len(NNRATIOS) else 0.8
                    nmo, mo = oracle_search(oracle, a, mode, cth, True, nn, th)
                    for c in P.cases:
                        for s, want in c["want"].items():
                            assert mo[s] == want, (W, mode, c["kind"], s, mo[s], want)
                        seen.add((mode, c["kind"]))
                        if c["kind"] in ("cells", "chunks", "rects", "cell"):
                            g = oracle.FrameGrid(a["k"], W, W)
                            start, idx = g.csr()
                            order = [i for i in g.features_in_area(c["u"], c["v"], c["r"], c["lvl"] - 1, c["lvl"] + (1 if mode == 0 else 0))]
                            dists = [hamming(a["dq"][c["q"]], a["d"][i]) for i in order]
                            tied = [i for i, dd in zip(order, dists) if dd == min(dists)]
                            assert len(tied) >= 2 and min(dists) == TIE_DIST and mo[tied[0]] == c["q"], c["kind"]
                            if c["kind"] != "cell":
                                assert tied[0] != min(tied)
                                visits = {(f, ix, iy): (k, ci) for k, ci, f, ix, iy in visit_cells(oracle, c["u"], c["v"], c["r"], W)}
                                where = [visits[cell_of(a["k"]["x"][i], a["k"]["y"][i], W)] for i in tied[:2]]
                                (k0, c0), (k1, c1) = where
                                if c["kind"] == "chunks":
                                    assert k0 == k1 and c0 // 32 < c1 // 32 and c1 % 32 < c0 % 32, where
                                if c["kind"] == "rects":
                                    assert (k0, k1) == (1, 2) and c1 % 32 < c0 % 32, where
                        if c["kind"] in ("edge", "ulp_inside"):
                            e = c["kps"][1]
                            d = max(abs(F32(a["k"]["x"][e]) - c["u"]), abs(F32(a["k"]["y"][e]) - c["v"]))
                            assert (d == c["r"]) == (c["kind"] == "edge") and d <= c["r"]
                        if c["kind"] == "ratio_equal":
                            da, db = (hamming(a["dq"][c["q"]], a["d"][s]) for s in c["kps"])
                            assert F32(F32(nn) * F32(db)) == F32(da)
                        if c["kind"] in ("th_one", "th_above_one"):
                            e = c["kps"][0]
                            assert max(abs(F32(a["k"]["x"][e]) - F32(a["proj"][c["q"], 0])), abs(F32(a["k"]["y"][e]) - F32(a["proj"][c["q"], 1]))) == F32(2.5)
                        if c["kind"] == "retaken":
                            assert a["obs"][c["first"]] == 0 and mo[c["kps"][0]] == c["q"]
                            alone = np.where(np.isin(np.arange(len(a["valid"])), [c["q"], c["later"]]), 0, a["valid"]).astype(np.uint8)
                            _, m1 = oracle_search(oracle, dict(a, valid=alone), mode, cth, True, nn)
                            assert m1[c["kps"][0]] == c["first"]              # the observation-less query matched the slot first
                        if c["kind"] in ("fov_keep", "fov_skip"):
                            assert (c["X"][2] == cth) == (c["kind"] == "fov_keep") and (c["X"][2] < cth) == (c["kind"] == "fov_skip")
                        if c["kind"] in ("seam_x_pos", "seam_y_pos", "seam_x_neg", "seam_y_neg"):
                            uv, f = oracle.ray_to_cubemap(c["X"], W, W)
                            ax = 0 if "_x_" in c["kind"] else 1
                            if c["kind"].endswith("pos"):
                                assert f[0] == -1 and uv[0, ax] == W
                            else:
                                assert f[0] >= 0 and uv[0, ax] == W
                        if c["kind"].startswith("double"):
                            s = c["kps"][0]
                            _, m0 = oracle_search(oracle, a, 0, cth, False)
                            assert m0[s] == c["q"] and mo[s] == -1 and (c["kind"] != "double_first_out" or c["bins"][1] == 0)
                        if c["kind"] in ("rot6", "rot30", "rot54"):
                            la, ca = c["rot"]
                            p = F32(F32(la - ca) * (F32(1) / F32(12)))
                            assert p - np.floor(p) == 0.5 and int(np.floor(p)) % 2 == 0 and mo[c["kps"][0]] == c["q"]   # rintf would pick the even bin
                        if c["kind"] == "wrap":
                            la, ca = c["rot"]
                            assert F32(la - ca) < 0 and F32(F32(la - ca) + F32(360)) == F32(360)
                    if getattr(P, "name", "") == "four_equal":
                        assert all(mo[c["kps"][0]] == -1 for c in P.cases if c["kind"] == "bin8") and all(mo[c["kps"][0]] >= 0 for c in P.cases if c["kind"] == "bin2")
                    if getattr(P, "name", "") in ("max2_tenth", "max3_tenth"):
                        assert F32(F32(0.1) * F32(20)) == F32(2)
                        assert all(mo[c["kps"][0]] >= 0 for c in P.cases if c["kind"] in ("bin5", "bin9") and P.name == "max3_tenth" or c["kind"] == "bin5")
                    if getattr(P, "name", "") == "max2_below":
                        assert all(mo[c["kps"][0]] == -1 for c in P.cases if c["kind"] in ("bin5", "bin9"))
                    if getattr(P, "name", "") == "nq13":
                        assert nmo == 13
                    if getattr(P, "name", "") == "full":
                        assert len(a["k"]) == len(a["kl"]) == 4096 and nmo > 1000
        kinds0 = {k for m, k in seen if m == 0}; kinds1 = {k for m, k in seen if m == 1}
        assert {"cell", "cells", "chunks", "rects", "th_100", "th_101", "edge", "ulp_inside", "level", "taken", "retaken", "fov_keep", "fov_skip", "seam_x_pos",
                "seam_x_neg", "seam_y_pos", "seam_y_neg", "behind_keep", "behind_skip", "rot6", "rot30", "rot54", "wrap", "rot354", "rot342", "double_first_out",
                "double_second_out", "double_both_out"} <= kinds0, kinds0
        assert {"cell", "cells", "chunks", "rects", "tie_same_level", "tie_zero", "tie_two_levels", "else_if", "second_equal", "ratio_equal", "ratio_over",
                "vcos_998", "vcos_below", "th_one", "th_above_one", "level", "taken", "retaken"} <= kinds1, kinds1
        # the frame index
        f0 = index_frames(W)[0][0]
        rays, faces = oracle.key_point_rays(f0, W, W)
        start, idx = oracle.FrameGrid(f0, W, W).csr()
        listed = set(idx.tolist())
        for i in range(len(f0)):
            c = cell_of(f0["x"][i], f0["y"][i], W)
            if c[0] is None:
                assert i not in listed and not rays[i].any() and faces[i] == -1
            else:
                cell = (c[0] * G + c[1]) * G + c[2]
                assert i in idx[start[cell]:start[cell + 1]]
        assert sum(cell_of(x, y, W)[0] is None for x, y in zip(f0["x"], f0["y"])) >= 10
        assert W != 650 or sum(not ref_safe(x, y, W) and cell_of(x, y, W)[0] is not None for x, y in zip(f0["x"], f0["y"])) >= 2
    x = np.nextafter(F32(1950), F32(0))
    assert cell_of(x, F32(975.41), 650) == (2, 0, 25) and not ref_safe(x, F32(975.41), 650)
    f1 = index_frames(650)[1][0]
    start, idx = oracle.FrameGrid(f1, 650, 650).csr()
    big = int(np.argmax(np.diff(start)))
    assert start[big + 1] - start[big] == 300


# ----------------------------------------------------------------------------------------------------------------- GPU parity
@pytest.fixture(scope="module")
def trk():
    from cubemapslam_b200.tracker import Tracker
    t = Tracker(max_frames=16, max_features=4096)
    yield t
    t.close()


def check_search(oracle, A, nm, m, mode, pairs, **kw):
    for i, (a, P) in enumerate(zip(A, pairs)):
        n = len(a["k"])
        nmo, mo = oracle_search(oracle, a, mode, **kw)
        got = np.where(m[i, :n] == -2, -1, m[i, :n])
        assert nm[i] == nmo and np.array_equal(got, mo), (i, getattr(P, "name", ""), nm[i], nmo, np.nonzero(got != mo)[0][:5])


def run_last(trk, S, W, cth, ori, path):
    import torch
    P = len(S["nC"]); cs, qs = S["k"].shape[1], S["kl"].shape[1]
    if path == "host":
        return trk.SearchByProjection_last(S["k"], S["d"], S["T"], S["kl"], S["valid"], S["Xw"], S["dq"], S["obs"], S["taken"], W, W, cth, TH_LAST, ori,
                                           nCur=S["nC"], nLast=S["nQ"])
    d = {k: to_dev(v) for k, v in dict(k=S["k"], d=S["d"], nC=S["nC"], taken=S["taken"], T=S["T"], kl=S["kl"], nQ=S["nQ"], valid=S["valid"], Xw=S["Xw"],
                                       dq=S["dq"], obs=S["obs"], cst=garbage((P, 12501), np.uint16), cid=garbage((P, cs), np.uint16),
                                       match=garbage((P, cs), np.int32), nm=garbage((P,), np.int32)).items()}
    a = {k: v.data_ptr() for k, v in d.items()}
    torch.cuda.synchronize()
    trk.frame_index_dev(a["k"], a["nC"], P, cs, W, W, None, a["cst"], a["cid"])
    trk.search_by_projection_last_dev(P, a["k"], a["d"], a["nC"], cs, a["cst"], a["cid"], a["taken"], a["T"], a["kl"], a["nQ"], qs, a["valid"], a["Xw"], a["dq"], a["obs"],
                                      W, W, cth, TH_LAST, int(ori), a["match"], a["nm"])
    trk.sync()
    match = from_dev(d["match"], garbage((P, cs), np.int32)); nm = from_dev(d["nm"], garbage((P,), np.int32))
    for i in range(P):
        assert (bits(match[i, S["nC"][i]:]) == GARBAGE).all(), i              # nothing written past the count
    return nm, match


def run_local(trk, S, W, th, nn, path, nlevels=8, factor=1.2):
    import torch
    from cubemapslam_b200._capi import check, lib, ptr
    P = len(S["nC"]); cs, qs = S["k"].shape[1], S["kl"].shape[1]
    if path == "host":
        return trk.SearchByProjection_local(S["k"], S["d"], S["valid"], S["proj"], S["level"], S["vcos"], S["dq"], S["obs"], S["taken"], W, W, th, nn, factor, nlevels,
                                            nF=S["nC"], nMP=S["nQ"])
    d = {k: to_dev(v) for k, v in dict(k=S["k"], d=S["d"], nC=S["nC"], taken=S["taken"], nQ=S["nQ"], valid=S["valid"], proj=S["proj"], level=S["level"], vcos=S["vcos"],
                                       dq=S["dq"], obs=S["obs"], cst=garbage((P, 12501), np.uint16), cid=garbage((P, cs), np.uint16),
                                       match=garbage((P, cs), np.int32), nm=garbage((P,), np.int32)).items()}
    a = {k: v.data_ptr() for k, v in d.items()}
    torch.cuda.synchronize()
    trk.frame_index_dev(a["k"], a["nC"], P, cs, W, W, None, a["cst"], a["cid"])
    check(lib().cslam_search_by_projection_local_dev(trk._h, P, ptr(a["k"]), ptr(a["d"]), ptr(a["nC"]), cs, ptr(a["cst"]), ptr(a["cid"]), ptr(a["taken"]), ptr(a["nQ"]), qs,
                                                     ptr(a["valid"]), ptr(a["proj"]), ptr(a["level"]), ptr(a["vcos"]), ptr(a["dq"]), ptr(a["obs"]), W, W, C.c_float(th),
                                                     C.c_float(nn), C.c_float(factor), nlevels, ptr(a["match"]), ptr(a["nm"])))
    trk.sync()
    match = from_dev(d["match"], garbage((P, cs), np.int32)); nm = from_dev(d["nm"], garbage((P,), np.int32))
    for i in range(P):
        assert (bits(match[i, S["nC"][i]:]) == GARBAGE).all(), i
    return nm, match


@pytest.mark.gpu
@pytest.mark.parametrize("path", ["host", "dev"])
@pytest.mark.parametrize("W", WIDTHS)
def test_frame_index_limits(oracle, trk, W, path):
    import torch
    frames = index_frames(W)
    Fn = len(frames); stride = 4096
    k = garbage((Fn, stride), KP()); n = np.array([c for _, c in frames], np.int32)
    for i, (kk, _) in enumerate(frames):
        k[i, :len(kk)] = kk
    if path == "host":
        rays, cs, ci = trk.frame_index(k, W, W, n=n)
    else:
        d = {key: to_dev(v) for key, v in dict(k=k, n=n, rays=garbage((Fn, stride, 3), F32), cs=garbage((Fn, 12501), np.uint16), ci=garbage((Fn, stride), np.uint16)).items()}
        torch.cuda.synchronize()
        trk.frame_index_dev(d["k"].data_ptr(), d["n"].data_ptr(), Fn, stride, W, W, d["rays"].data_ptr(), d["cs"].data_ptr(), d["ci"].data_ptr())
        trk.sync()
        rays, cs, ci = from_dev(d["rays"], garbage((Fn, stride, 3), F32)), from_dev(d["cs"], garbage((Fn, 12501), np.uint16)), from_dev(d["ci"], garbage((Fn, stride), np.uint16))
    for i in range(Fn):
        m = min(n[i], stride)
        kk = k[i, :m]
        r_o, _ = oracle.key_point_rays(kk, W, W)
        start, idx = oracle.FrameGrid(kk, W, W).csr()
        assert np.array_equal(bits(rays[i, :m]), bits(r_o)), i
        assert np.array_equal(cs[i].astype(np.int64), start.astype(np.int64)), i
        assert np.array_equal(ci[i, :len(idx)].astype(np.int64), idx.astype(np.int64)), i
        if path == "dev":
            assert (bits(rays[i, m:]) == GARBAGE).all() and (bits(ci[i, len(idx):]) == GARBAGE).all(), i


@pytest.mark.gpu
@pytest.mark.parametrize("path", ["host", "dev"])
@pytest.mark.parametrize("W", WIDTHS)
def test_search_last_limits(oracle, trk, W, path):
    cth = cos_fov_th()
    pairs = last_batch(oracle, W)
    A, S = stack(pairs, pad=7)
    for ori in (True, False):
        nm, m = run_last(trk, S, W, cth, ori, path)
        check_search(oracle, A, nm, m, 0, pairs, cth=cth, check_ori=ori)


@pytest.mark.gpu
@pytest.mark.parametrize("path", ["host", "dev"])
@pytest.mark.parametrize("nn", NNRATIOS)
@pytest.mark.parametrize("W", WIDTHS)
def test_search_local_limits(oracle, trk, W, nn, path):
    pairs = local_batch(oracle, W, nn)
    A, S = stack(pairs, pad=5)
    nm, m = run_local(trk, S, W, TH_LOCAL, nn, path)
    check_search(oracle, A, nm, m, 1, pairs, nn=nn)


@pytest.mark.gpu
@pytest.mark.parametrize("path", ["host", "dev"])
@pytest.mark.parametrize("th", [1.0, float(np.nextafter(F32(1), F32(2)))])
def test_search_local_radius_factor(oracle, trk, th, path):
    for W in WIDTHS:
        pairs = [radius_pair(oracle, W, th)]
        A, S = stack(pairs, pad=3)
        nm, m = run_local(trk, S, W, th, 0.8, path)
        check_search(oracle, A, nm, m, 1, pairs, nn=0.8, th=th)


@pytest.mark.gpu
@pytest.mark.parametrize("path", ["host", "dev"])
def test_search_local_12_levels(oracle, trk, path):
    """A pyramid of 12 levels at factor 1.1 (the reference scenes fix 8 at 1.2): predicted levels up to 11."""
    pairs = [main_pair(oracle, 650, 1, seed=3)]
    rng = np.random.default_rng(5)
    for q in pairs[0].q:
        q["oct"] = int(rng.integers(0, 12))
    for i in range(len(pairs[0].k)):
        x = pairs[0].k[i]
        pairs[0].k[i] = x[:5] + (int(rng.integers(0, 12)),) + x[6:]
    A, S = stack(pairs, pad=3)
    nm, m = run_local(trk, S, 650, TH_LOCAL, 0.8, path, nlevels=12, factor=1.1)
    check_search(oracle, A, nm, m, 1, pairs, nn=0.8, nlevels=12, factor=1.1)
    assert nm[0] > 100


@pytest.mark.gpu
@pytest.mark.parametrize("with_rays", [True, False])
def test_gather_pose_inputs_limits(oracle, trk, with_rays):
    import torch
    W = 650
    cth = cos_fov_th()
    _, invs2 = level_tables()
    fr = gather_frames(oracle, W, cth)
    P = len(fr); cs, ls = 4096, 3500
    k, match, rays, Xw = garbage((P, cs), KP()), garbage((P, cs), np.int32), garbage((P, cs, 3), F32), garbage((P, ls, 3), F32)
    n = np.array([len(f["k"]) for f in fr], np.int32)
    for i, f in enumerate(fr):
        k[i, :n[i]] = f["k"]; match[i, :n[i]] = f["match"]; rays[i, :n[i]] = f["rays"]; Xw[i] = f["Xw"]
    gX, gkp, gw, cnt = garbage((P, cs, 3), F32), garbage((P, cs, 2), F32), garbage((P, cs), F32), garbage((P,), np.int32)
    d = {key: to_dev(v) for key, v in dict(k=k, match=match, rays=rays, Xw=Xw, n=n, invs2=invs2, gX=gX, gkp=gkp, gw=gw, cnt=cnt).items()}
    torch.cuda.synchronize()
    trk.gather_pose_inputs_dev(P, d["match"].data_ptr(), d["k"].data_ptr(), d["n"].data_ptr(), cs, d["rays"].data_ptr() if with_rays else None, cth,
                               d["Xw"].data_ptr(), ls, d["invs2"].data_ptr(), d["gX"].data_ptr(), d["gkp"].data_ptr(), d["gw"].data_ptr(), d["cnt"].data_ptr())
    trk.sync()
    gX, gkp, gw, cnt = from_dev(d["gX"], gX), from_dev(d["gkp"], gkp), from_dev(d["gw"], gw), from_dev(d["cnt"], cnt)
    sizes = {}
    for i, f in enumerate(fr):
        X_o, kp_o, w_o = pose_inputs_reference(f["match"], f["k"], f["rays"] if with_rays else None, f["Xw"], invs2, cth)
        c = len(X_o); sizes[f["kind"]] = c
        assert cnt[i] == c, (f["kind"], cnt[i], c)
        assert np.array_equal(bits(gX[i, :c]), bits(X_o)) and np.array_equal(bits(gkp[i, :c]), bits(kp_o)) and np.array_equal(bits(gw[i, :c]), bits(w_o)), f["kind"]
        assert (bits(gX[i, c:]) == GARBAGE).all() and (bits(gw[i, c:]) == GARBAGE).all(), f["kind"]
    assert [sizes[k] for k in ("c255", "c256", "c257", "c4096", "empty")] == [255, 256, 257, 4096, 0]
    mixed = fr[4]
    kept = (mixed["match"] >= 0) & (mixed["rays"][:, 2] == cth); dropped = (mixed["match"] >= 0) & (mixed["rays"][:, 2] < cth)
    assert kept.sum() >= 30 and dropped.sum() >= 30 and (mixed["match"] == -2).sum() > 500 and (mixed["match"] == -1).sum() > 500
    assert sizes["mixed"] == (mixed["match"] >= 0).sum() - (dropped.sum() if with_rays else 0)

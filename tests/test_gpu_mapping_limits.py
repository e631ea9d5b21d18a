"""The LocalMapping kernels (cubemapslam_b200/csrc/mapping.cu) at the rules random scenes do not reach: Fuse's first-least-distance order
across cells, 32-cell chunks and seam rectangles, complement-only windows (distance 256 is no match), the strict window edge, seam and
behind-the-camera projections, the level gates and level counts, the size limits; ComputeDistinctiveDescriptors' first-least-median rule
across warps and past the shared-memory staging; SearchForTriangulation at face width 450, with a zero camera centre and with the epipole
on a face seam. Every answer is compared with the oracle, exactly. The scenes are built here from synth.mapping_pair plus hand-placed key
points and descriptors; test_scenes_reach_every_case checks, on the oracle's answers alone, that each case is really there, and
tests/test_oracle_mapping.py pins the oracle to the compiled reference on the scenes that have a reference counterpart."""
import os

import numpy as np
import pytest

from cubemapslam_b200 import synth

G = 50                                                         # grid cells per face side
TILE = {0: (1, 1), 1: (0, 1), 2: (2, 1), 3: (1, 0), 4: (1, 2)}   # face -> canvas tile (column, row)
POPC = np.array([bin(i).count("1") for i in range(256)], np.int32)
TIE_DIST = 20
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "refcalls_oracle_mapping.npz")
F32 = np.float32


# ----------------------------------------------------------------------------------------------------------------- geometry
def hamming(a, b):
    return int(POPC[np.bitwise_xor(a, b)].sum())


def flipped(d, bits):
    out = d.copy()
    for b in bits:
        out[b >> 3] ^= np.uint8(1 << (b & 7))
    return out


def transform(T, X):
    """`Rcw * x + tcw` as the reference's CV_32F gemm evaluates it (oracle/frame_index.h fi_transform)."""
    T = np.asarray(T, F32).reshape(4, 4); X = np.asarray(X, F32)
    out = np.empty(3, F32)
    for i in range(3):
        t = T[i, 0] * X[0]
        t = t + T[i, 1] * X[1]
        t = t + T[i, 2] * X[2]
        out[i] = F32(np.float64(t) + np.float64(T[i, 3]))
    return out


def project(oracle, T, X, W):
    uv, face = oracle.ray_to_cubemap(transform(T, X), W, W)
    return F32(uv[0, 0]), F32(uv[0, 1]), int(face[0])


def cell_of(x, y, W):
    """Frame::PosInGrid on a 3W-wide canvas: (face, column, row), face None off the five faces."""
    x, y = F32(x), F32(y)
    face = {(0, 1): 1, (1, 0): 3, (1, 1): 0, (1, 2): 4, (2, 1): 2}.get((int(np.floor(x / F32(W))), int(np.floor(y / F32(W)))))
    inv = F32(3 * G) / F32(3 * W)
    return face, int(x * inv) % G, int(y * inv) % G


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


def gated(kx, ky, oct_, u, v, lvl, r, isg):
    """Fuse's window, level and chi2 tests in the reference's float arithmetic."""
    kx, ky, u, v = F32(kx), F32(ky), F32(u), F32(v)
    if not (abs(kx - u) < r and abs(ky - v) < r) or oct_ < lvl - 1 or oct_ > lvl:
        return False
    ex = u - kx; ey = v - ky
    return float((ex * ex + ey * ey) * isg[oct_]) <= 5.99


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


# ----------------------------------------------------------------------------------------------------------------- Fuse scenes
class FuseScene:
    """A key frame (synth.mapping_pair's current frame plus hand-placed key points) and MapPoints placed to project at chosen pixels.
    `cases` lists the hand-placed MapPoints: kind, index, projection, radius, level, its key points and the expected answer."""

    def __init__(self, oracle, W, th, seed=0, nlevels=8, clear=()):
        s = synth.mapping_pair(seed, n=1500, faceW=W)
        self.oracle, self.W, self.th, self.T = oracle, W, F32(th), s["TcwCur"]
        self.scale, self.isg = s["scale"][:nlevels].copy(), s["inv_level_sigma2"][:nlevels].copy()
        self.rng = np.random.default_rng(500 + seed)
        keep = np.ones(len(s["kCur"]), bool)
        for cx, cy in clear:   # no stray key point near these pixels
            keep &= (s["kCur"]["x"] - cx) ** 2 + (s["kCur"]["y"] - cy) ** 2 > 14 ** 2
        self.kps = [tuple(k) for k in s["kCur"][keep].tolist()]; self.desc = list(s["dCur"][keep])
        self.Xw, self.level, self.dMP, self.valid = [], [], [], []
        self.cases = []
        self.base = s

    def add_kp(self, x, y, oct_, d):
        self.kps.append((float(x), float(y), 31.0, float(self.rng.uniform(0, 360)), 0.0, int(oct_), -1)); self.desc.append(d)
        return len(self.kps) - 1

    def add_mp(self, tx, ty, lvl, depth=5.0):
        """A MapPoint projecting near canvas pixel (tx, ty) at predicted level lvl: (index, u, v, radius, descriptor), or None off the faces."""
        ray = synth._pixel_to_ray(float(tx), float(ty), self.W)
        if ray is None:
            return None
        T = self.T.astype(np.float64)
        X = (T[:3, :3].T @ (ray * depth - T[:3, 3])).astype(F32)
        u, v, face = project(self.oracle, self.T, X, self.W)
        if face < 0:
            return None
        d = self.rng.integers(0, 256, 32, dtype=np.uint8)
        self.Xw.append(X); self.level.append(lvl); self.dMP.append(d); self.valid.append(1)
        return len(self.Xw) - 1, u, v, F32(self.th * self.scale[lvl]), d

    def add_background(self, n):
        """n of the pair's own MapPoints (true correspondences and misses), levels near their key points' octaves."""
        s = self.base; nl = len(self.scale)
        for m in self.rng.choice(len(s["Xw"]), n, replace=False):
            self.Xw.append(s["Xw"][m]); self.dMP.append(s["dLast"][m]); self.valid.append(int(self.rng.random() < 0.9))
            self.level.append(int(np.clip(s["kLast"]["octave"][m] + self.rng.integers(-1, 2), 0, nl - 1)))

    def arrays(self):
        from oracle import KP_DTYPE
        k = np.array(self.kps, KP_DTYPE) if self.kps else np.zeros(0, KP_DTYPE)
        d = np.stack(self.desc) if self.desc else np.zeros((0, 32), np.uint8)
        return dict(kKF=k, dKF=d, Tcw=self.T, valid=np.array(self.valid, np.uint8), Xw=np.array(self.Xw, F32).reshape(-1, 3),
                    level=np.array(self.level, np.int32), dMP=np.array(self.dMP, np.uint8).reshape(-1, 32), th=float(self.th), scale=self.scale,
                    isg=self.isg, W=self.W)

    def kobs(self):
        """Key points of the observing key frame of the reference's scene: MapPoint m seen by key point m at octave = its level."""
        from oracle import KP_DTYPE
        a = self.arrays(); k = np.zeros(len(a["Xw"]), KP_DTYPE)
        k["x"], k["y"], k["size"], k["octave"], k["class_id"] = self.W * 1.5, self.W * 1.5, 31, a["level"], -1
        return k

    def reachable(self, u, v, r, lvl):
        """Visited cells holding a point that passes every gate at octave lvl: [(rectangle, position, face, column, row, (x, y))]."""
        out = []
        for k, ci, f, ix, iy in visit_cells(self.oracle, u, v, r, self.W):
            p = point_in_cell(f, ix, iy, u, v, self.W)
            if p is not None and gated(p[0], p[1], lvl, u, v, lvl, r, self.isg):
                out.append((k, ci, f, ix, iy, p))
        return out


def tie_kinds(reach):
    """Pairs of reachable cells (earlier, later in the visiting order) for each tie arrangement; the later one sits on a lower lane where
    that is what tells the arrangements apart."""
    kinds = {}
    for a, p in enumerate(reach):
        for q in reach[a + 1:]:
            if p[0] == q[0] and p[1] // 32 == q[1] // 32:
                kinds.setdefault("cells", (p, q))
            if p[0] == q[0] and p[1] // 32 < q[1] // 32 and q[1] % 32 < p[1] % 32:
                kinds.setdefault("chunks", (p, q))
            if p[0] == 1 and q[0] == 2 and q[1] % 32 < p[1] % 32:
                kinds.setdefault("rects", (p, q))
    return kinds


def _spots(W, corner, step):
    """Candidate MapPoint pixels: face interiors on a lattice, or 2..8 px inside every face corner."""
    out = []
    for f, (c, r) in TILE.items():
        if corner:
            for ox in (0, 1):
                for oy in (0, 1):
                    for dx, dy in ((3.1, 3.3), (5.2, 2.4), (2.3, 6.1), (6.6, 5.7), (1.7, 1.9), (4.4, 7.3)):
                        out.append((c * W + (W - dx if ox else dx), r * W + (W - dy if oy else dy)))
        else:
            for x in np.arange(60, W - 60, step):
                for y in np.arange(60, W - 60, step):
                    out.append((c * W + x, r * W + y))
    return out


def tie_scene(oracle, W=650, per_kind=3, seed=0):
    """th = 12 at level 7: 7-8 x 7-8-cell windows. Five tie arrangements at TIE_DIST, complement-only windows and complement + 255 windows
    at levels 0 and 7, and background MapPoints. Tied key points are appended later-visited first, so the first visited is never the
    lowest index outside one cell; twelve fillers precede the earlier candidate in its cell, so its position within its chunk is high."""
    lvl = 7
    comp_spots = [(W + 100 + 110 * i, 2 * W + 200 + 120 * (i % 2)) for i in range(4)] + [(2 * W + 150 + 110 * i, W + 500) for i in range(3)]
    S = FuseScene(oracle, W, 12.0, seed=seed, clear=comp_spots)
    used = list(comp_spots)

    def free(x, y):
        return all((x - a) ** 2 + (y - b) ** 2 > 40 ** 2 for a, b in used)

    want = {"cells": per_kind, "chunks": per_kind, "rects": per_kind, "cell": per_kind}
    for corner in (True, False):
        for tx, ty in _spots(W, corner, 37.0):
            if not any(want.values()):
                break
            if not free(tx, ty):
                continue
            mp = S.add_mp(tx, ty, lvl)
            if mp is None:
                continue
            m, u, v, r, D = mp
            kinds = tie_kinds(S.reachable(u, v, r, lvl))
            kind = next((k for k in (("rects",) if corner else ("chunks", "cells")) if want[k] and k in kinds), None)
            if kind is None and want["cell"] and not corner:
                kind = "cell"
            if kind is None:
                S.Xw.pop(); S.level.pop(); S.dMP.pop(); S.valid.pop()
                continue
            want[kind] -= 1; used.append((tx, ty))
            bits = S.rng.permutation(256)
            if kind == "cell":
                f, ix, iy = cell_of(u, v, W)
                pts = [point_in_cell(f, ix, iy, u + dx, v + dy, W) for dx, dy in ((0.5, 0.2), (-0.4, 0.6), (0.3, -0.5))]
                kps = [S.add_kp(x, y, lvl, flipped(D, bits[TIE_DIST * i:TIE_DIST * (i + 1)])) for i, (x, y) in enumerate(pts)]
                expect = kps[0]
            else:
                p, q = kinds[kind]
                late = S.add_kp(*q[5], lvl, flipped(D, bits[:TIE_DIST]))
                for _ in range(12):
                    S.add_kp(*point_in_cell(*p[2:5], u, v, W, far=True), lvl, S.rng.integers(0, 256, 32, dtype=np.uint8))
                early = S.add_kp(*p[5], lvl, flipped(D, bits[TIE_DIST:2 * TIE_DIST]))
                kps, expect = [late, early], early
            S.cases.append(dict(kind=kind, m=m, u=u, v=v, r=r, lvl=lvl, kps=kps, expect=expect, dist=TIE_DIST))
    assert not any(want.values()), want
    # complement-only windows and complement + 255 windows (either order), at level 0 (one cell) and level 7
    for i, (tx, ty) in enumerate(comp_spots):
        lv = 0 if i % 2 == 0 else lvl
        m, u, v, r, D = S.add_mp(tx, ty, lv)
        offs = ((0.4, 0.3), (-0.5, 0.2), (0.1, -0.6)) if lv == 0 else ((3.0, 2.0), (-4.0, 1.0), (1.0, -5.5))
        octs = (lv, lv, lv) if lv == 0 else (lv, lv - 1, lv)
        kind = ("complement", "complement", "mixed_after", "mixed_before")[i % 4] if i < 4 else ("complement", "mixed_after", "mixed_before")[i - 4]
        near = ~D if kind == "complement" else flipped(~D, [int(S.rng.integers(0, 256))])
        kps = []
        for j, ((dx, dy), o) in enumerate(zip(offs, octs)):
            d = near if (kind == "mixed_after" and j == 1) or (kind == "mixed_before" and j == 0) else ~D
            kps.append(S.add_kp(u + dx, v + dy, o, d))
        expect = -1 if kind == "complement" else kps[1 if kind == "mixed_after" else 0]
        S.cases.append(dict(kind=kind, m=m, u=u, v=v, r=r, lvl=lv, kps=kps, expect=expect, dist=256 if expect < 0 else 255))
    S.add_background(300)
    return S


def edge_scene(oracle, th, W=650):
    """Level 0, radius th (1 or 2, exact in float32 at any canvas position): a key point at exactly |kp - centre| == radius on one axis
    with the best descriptor, which the strict window test drops, or one ulp inside, which it keeps; a worse key point inside the window."""
    S = FuseScene(oracle, W, th, seed=3)
    cl = W // G
    spots = [(c * W + (ix + 0.5) * cl, r * W + (iy + 0.5) * cl) for (c, r) in TILE.values() for ix in (6, 24, 42) for iy in (8, 30)]
    variants = [(ax, sg, ulp) for ulp in (False, True) for ax in (0, 1) for sg in (1, -1)]
    for i, (tx, ty) in enumerate(spots):
        ax, sg, ulp = variants[i % len(variants)]
        m, u, v, r, D = S.add_mp(tx, ty, 0)
        assert r == th
        c = (u, v)[ax]
        e = F32(c + F32(sg) * r)
        if ulp:
            e = np.nextafter(e, c)
        assert (abs(e - c) == r) != ulp
        x, y = (e, v) if ax == 0 else (u, e)
        bits = S.rng.permutation(256)
        inside = S.add_kp(u + F32(0.25 * r * -sg * (ax == 0)), v + F32(0.25 * r * -sg * (ax == 1)), 0, flipped(D, bits[:30]))
        edge = S.add_kp(x, y, 0, flipped(D, bits[30:40]))
        S.cases.append(dict(kind="ulp_inside" if ulp else "edge", m=m, u=u, v=v, r=r, lvl=0, kps=[inside, edge], expect=edge if ulp else inside,
                            dist=10 if ulp else 30))
    S.add_background(200)
    return S


def level_scene(oracle, nlevels):
    """th = 3. Predicted level 0, 1, the middle and the last; key points at octave lvl - 2 .. lvl + 1 around the projection, the ones the
    level gate drops holding the better descriptors. Plus complement-only windows at the first and the last level."""
    S = FuseScene(oracle, 650, 3.0, seed=4, nlevels=nlevels)
    lvls = sorted({0, min(1, nlevels - 1), nlevels // 2, nlevels - 1})
    spots = [(650 + 80 + 120 * i, 650 + 90 + 130 * j) for j in range(4) for i in range(4)] + [(1300 + 100 + 150 * i, 650 + 200) for i in range(3)]
    dist = {-2: 5, -1: 10, 0: 20, 1: 3}
    for i, (tx, ty) in enumerate(spots):
        lv = lvls[i % len(lvls)]
        m, u, v, r, D = S.add_mp(tx, ty, lv)
        bits = S.rng.permutation(256)
        kps = {}
        for j, o in enumerate((-2, -1, 0, 1)):
            if lv + o >= 0:
                kps[o] = S.add_kp(u + F32(0.3 * np.cos(j * 1.7)), v + F32(0.3 * np.sin(j * 1.7)), lv + o, flipped(D, bits[:dist[o]]))
        S.cases.append(dict(kind="level", m=m, u=u, v=v, r=r, lvl=lv, kps=list(kps.values()), expect=kps[-1] if -1 in kps else kps[0],
                            dist=dist[-1] if -1 in kps else dist[0]))
    S.add_background(300)
    return S


def crowded_scene(oracle):
    """4096 key points, 40 of them in one cell around a MapPoint's projection (level 0): the least distance on the 35th and the 38th."""
    S = FuseScene(oracle, 650, 3.0, seed=5, clear=[(981.5, 981.5)])
    m, u, v, r, D = S.add_mp(981.5, 981.5, 0)
    bits = S.rng.permutation(256)
    first = len(S.kps)
    for j in range(40):
        a = 2 * np.pi * j / 40
        d = flipped(D, bits[:15]) if j in (34, 37) else flipped(D, bits[:40 + j])
        S.add_kp(u + F32(1.2 * np.cos(a)), v + F32(1.2 * np.sin(a)), 0, d)
    assert len({cell_of(*k[:2], 650) for k in S.kps[first:]}) == 1
    S.cases.append(dict(kind="crowded", m=m, u=u, v=v, r=r, lvl=0, kps=list(range(first, first + 40)), expect=first + 34, dist=15))
    while len(S.kps) < 4096:
        c, rw = TILE[int(S.rng.integers(0, 5))]
        S.add_kp(c * 650 + S.rng.uniform(0.5, 649.5), rw * 650 + S.rng.uniform(0.5, 649.5), int(S.rng.integers(0, 8)), S.rng.integers(0, 256, 32, dtype=np.uint8))
    S.add_background(600)
    return S


def face_boundary_points():
    """synth.mapping_pair(5)'s MapPoints, five in six moved onto a face seam or behind the camera (identity pose). Returns the pair, Xw
    and the placement kind of every MapPoint. TransformRaysToCubemap leaves in-face coordinates (no tile offset) when its in-face test
    fails, and Fuse only asks IsInImage of them (src/ORBMatcher.cpp:1150-1154)."""
    s = synth.mapping_pair(5, n=1200, faceW=650)
    rng = np.random.default_rng(11)
    Xw = s["Xw"].copy(); n = len(Xw)
    d = rng.uniform(2.0, 9.0, n).astype(F32); y = rng.uniform(-0.9, 0.9, n).astype(F32) * d
    k = np.arange(n) % 6
    Xw[k == 0] = np.stack([d, y, d], 1)[k == 0]           # x / z == 1: front test passes, u == W fails the in-face test
    Xw[k == 1] = np.stack([-d, y, d], 1)[k == 1]          # x / z == -1
    Xw[k == 2] = np.stack([y, d, d], 1)[k == 2]           # y / z == 1
    Xw[k == 3] = np.stack([d, y, -d], 1)[k == 3]          # behind: right face, z / x == -1
    Xw[k == 4] = 0                                        # the origin: no face at all -> (-1, -1)
    return s, Xw, k


def seam_scene(oracle):
    """face_boundary_points() with the valid / level arrays the reference produced for them (test_oracle_mapping.test_fuse_on_face_boundaries),
    plus a close key point next to every valid seam or behind-the-camera MapPoint's projection."""
    s, Xw, k = face_boundary_points()
    rng = np.random.default_rng(12)
    rec = np.load(GOLD)
    valid, level = rec["fuse_face_boundaries/1"], rec["fuse_face_boundaries/2"]
    uv, face = oracle.ray_to_cubemap(Xw, 650, 650)
    kps = [tuple(x) for x in s["kCur"].tolist()]; desc = list(s["dCur"])
    for m in np.nonzero((valid == 1) & (k < 4))[0]:
        u, v = uv[m]
        if 0 <= u < 1950 and 0 <= v < 1950 and cell_of(u + 0.3, v + 0.3, 650)[0] is not None:
            kps.append((float(u + F32(0.3)), float(v + F32(0.3)), 31.0, 0.0, 0.0, int(level[m]), -1))
            desc.append(flipped(s["dLast"][m], rng.permutation(256)[:12]))
    from oracle import KP_DTYPE
    return dict(kKF=np.array(kps, KP_DTYPE), dKF=np.stack(desc), Tcw=np.eye(4, dtype=F32), valid=valid, Xw=Xw, level=level, dMP=s["dLast"], th=4.0,
                scale=s["scale"], isg=s["inv_level_sigma2"], W=650, kind=k, face=face, uv=uv)


def oracle_fuse(oracle, a):
    g = oracle.FrameGrid(a["kKF"], a["W"], a["W"])
    return g.fuse_search(a["dKF"], a["Tcw"], a["scale"], a["isg"], a["valid"], a["Xw"], a["level"], a["dMP"], a["th"])


# ----------------------------------------------------------------------------------------------------------------- distinctive sets
def tie_set(rng, N, rows):
    """N descriptors whose least median is shared by exactly `rows`: row i in rows is base ^ one bit of its own, the others base ^ ~30
    noise bits that avoid those bits. Every tied row sees the same distances (0, 2 to the other tied rows, w + 1 to a noisy row of weight w),
    a noisy row sees about 2w to the other noisy ones, so the tied rows' median is the least."""
    base = rng.integers(0, 256, 32, dtype=np.uint8)
    own = rng.choice(256, len(rows), replace=False)
    free = np.setdiff1d(np.arange(256), own)
    d = np.stack([flipped(base, rng.choice(free, int(rng.integers(24, 40)), replace=False)) for _ in range(N)])
    for i, b in zip(rows, own):
        d[i] = flipped(base, [b])
    return d


TIE_SETS = [(40, (0, 17)), (40, (31, 35)), (40, (32, 33, 39)), (200, (31, 150)), (200, (32, 64)), (200, (127, 190)), (200, (128, 129)),
            (200, (129, 199)), (1024, (1023,)), (1024, (127, 1023)), (1025, (1023, 1024)), (1025, (1024,)), (3000, (1024, 2999)), (3000, (129, 2000))]


def distinctive_sets(seed=0, max_n=None):
    """Tie sets, all-identical sets, random sets of every N in 1..3 and 127..129 and of small even N."""
    rng = np.random.default_rng(seed)
    sets = [tie_set(rng, N, rows) for N, rows in TIE_SETS if max_n is None or N <= max_n]
    for N in (1, 2, 3, 127, 128, 129, 1025):
        if max_n is None or N <= max_n:
            sets.append(np.repeat(rng.integers(0, 256, (1, 32), dtype=np.uint8), N, axis=0))
    for N in (1, 2, 3, 127, 128, 129, 2, 4, 4, 6, 6, 8, 8, 10, 12, 16) * 4:
        base = rng.integers(0, 256, 32, dtype=np.uint8)
        sets.append(np.stack([flipped(base, rng.choice(256, int(rng.integers(0, 90)), replace=False)) for _ in range(N)]))
    return sets


def medians(d, k=None):
    """Every row's median distance (vDists[0.5 * (N - 1)], or the k-th order statistic)."""
    N = len(d)
    D = POPC[d[:, None, :] ^ d[None, :, :]].sum(axis=2)
    return np.sort(D, axis=1)[:, int(0.5 * (N - 1)) if k is None else k]


def pack(sets, rng, lead=0, empty_every=3):
    """Concatenate sets with empty points between them and `lead` unused rows before the first."""
    rows = [rng.integers(0, 256, (lead, 32), dtype=np.uint8)]; off = [lead]; where = []
    for i, d in enumerate(sets):
        if i % empty_every == 1:
            off.append(off[-1])
        where.append(len(off) - 1); rows.append(d); off.append(off[-1] + len(d))
    return np.concatenate(rows), np.array(off, np.int32), where


# ----------------------------------------------------------------------------------------------------------------- triangulation pairs
def triangulation_pairs(oracle, W=450):
    """Three synthetic pairs at face width W, a pure rotation (Tcw2 = I, Ow1 = 0 exactly, so C2 = 0, the epipole is (-1, -1) and E12 = 0)
    and a pair whose KF1 centre puts the epipole on a face seam next to true matches of KF2 (x / z = 1 on the front face: the in-face test
    fails and the epipole keeps in-face coordinates)."""
    ps = []
    for p in range(3):
        s = synth.mapping_pair(30 + p, n=1200, faceW=W)
        T1 = s["TcwCur"].astype(np.float64)
        ps.append(dict(s=s, Ow=(-T1[:3, :3].T @ T1[:3, 3]).astype(F32), T2=s["TcwLast"], E=s["E12"]))
    s = synth.mapping_pair(33, n=1200, faceW=W)
    ps.append(dict(s=s, Ow=np.zeros(3, F32), T2=np.eye(4, dtype=F32), E=np.zeros((3, 3), F32)))
    s = synth.mapping_pair(34, n=1200, faceW=W)
    rays1, _ = oracle.key_point_rays(s["kCur"], W, W); rays2, _ = oracle.key_point_rays(s["kLast"], W, W)
    T1 = s["TcwCur"].astype(np.float64); Ow = (-T1[:3, :3].T @ T1[:3, 3]).astype(F32)
    _, m = oracle.search_for_triangulation(s["kCur"], s["dCur"], rays1, s["hasMPCur"], s["nodeCur"], s["kLast"], s["dLast"], rays2, s["hasMPObs"], s["nodeObs"], Ow,
                                           s["TcwLast"], s["E12"], s["scale"], s["level_sigma2"], W, W, False)
    # the matched KF2 key point nearest to the upper face's left edge x = W: put the epipole (W, y) 2 px from it
    i2 = m[m >= 0]; k2 = s["kLast"][i2]
    up = (k2["y"] < W) & (k2["x"] >= W) & (k2["x"] < 2 * W)
    j = np.argmin(np.where(up, k2["x"], np.inf))
    y = (float(k2["y"][j]) + 2.0 - W / 2.0) / (W / 2.0)
    ps.append(dict(s=s, Ow=np.array([1.0, y, 1.0], F32), T2=np.eye(4, dtype=F32), E=s["E12"]))
    return ps


def oracle_triangulation(oracle, p, W, ori):
    s = p["s"]
    ra, _ = oracle.key_point_rays(s["kCur"], W, W); rb, _ = oracle.key_point_rays(s["kLast"], W, W)
    return oracle.search_for_triangulation(s["kCur"], s["dCur"], ra, s["hasMPCur"], s["nodeCur"], s["kLast"], s["dLast"], rb, s["hasMPObs"], s["nodeObs"], p["Ow"],
                                           p["T2"], p["E"], s["scale"], s["level_sigma2"], W, W, ori)


# ----------------------------------------------------------------------------------------------------------------- fixtures
@pytest.fixture(scope="module")
def scenes(oracle):
    return dict(ties=tie_scene(oracle), edge1=edge_scene(oracle, 1.0), edge2=edge_scene(oracle, 2.0),
                levels={nl: level_scene(oracle, nl) for nl in (1, 4, 8)}, seam=seam_scene(oracle))


@pytest.fixture(scope="module")
def mapper():
    from cubemapslam_b200.mapper import Mapper
    m = Mapper()
    yield m
    m.close()


def gpu_fuse(mapper, a):
    return mapper.FuseSearch(a["kKF"], a["dKF"], a["Tcw"], a["valid"], a["Xw"], a["level"], a["dMP"], a["th"], a["scale"], a["isg"], a["W"], a["W"])


def check_fuse(oracle, mapper, S):
    a = S.arrays() if isinstance(S, FuseScene) else S
    bi, bd = oracle_fuse(oracle, a)
    gi, gd = gpu_fuse(mapper, a)
    bad = np.nonzero((gi != bi) | (gd != bd))[0]
    assert len(bad) == 0, "%d MapPoints differ, first %d: gpu (%d, %d) oracle (%d, %d)" % (len(bad), bad[0], gi[bad[0]], gd[bad[0]], bi[bad[0]], bd[bad[0]])
    for c in getattr(S, "cases", ()):
        assert (bi[c["m"]], bd[c["m"]]) == (c["expect"], c["dist"]), c
    return bi, bd


# ----------------------------------------------------------------------------------------------------------------- the cases are reached
def test_scenes_reach_every_case(oracle):
    """On the oracle's answers alone: ties across a chunk boundary and across seam rectangles whose winner is neither the lowest index nor
    the lowest lane nor the first within its chunk, complement-only windows, key points exactly at the radius that the window drops, seam
    and behind-the-camera MapPoints that stay valid and match, least-median ties first at rows >= 32 and >= 128, N = 1024 and 1025, even N
    where vDists[0.5 * (N - 1)] and vDists[N / 2] choose different rows, an epipole on a seam that rejects a match (-1, -1) would keep."""
    S = tie_scene(oracle); a = S.arrays()
    g = oracle.FrameGrid(a["kKF"], 650, 650)
    start, idx = g.csr()
    bi, bd = oracle_fuse(oracle, a)
    seen = set()
    for c in S.cases:
        m, u, v, r, lvl = c["m"], c["u"], c["v"], c["r"], c["lvl"]
        order = [i for i in g.features_in_area(u, v, r) if gated(a["kKF"]["x"][i], a["kKF"]["y"][i], a["kKF"]["octave"][i], u, v, lvl, r, S.isg)]
        dists = [hamming(a["dMP"][m], a["dKF"][i]) for i in order]
        assert bi[m] == c["expect"] and bd[m] == c["dist"], c
        if c["kind"] == "complement":
            assert len(order) >= 2 and set(dists) == {256}
        elif c["kind"].startswith("mixed"):
            assert sorted(dists) == [255] + [256] * (len(dists) - 1)
        else:
            tied = [i for i, dd in zip(order, dists) if dd == min(dists)]
            assert len(tied) >= 2 and tied[0] == c["expect"]
            if c["kind"] != "cell":
                assert tied[0] != min(tied)
                # rectangle, position in it, lane and position within its chunk of each tied key point, from the oracle's grid
                visits = {(f, ix, iy): (k, ci) for k, ci, f, ix, iy in visit_cells(oracle, u, v, r, 650)}
                where = []
                for i in tied[:2]:
                    f, ix, iy = cell_of(a["kKF"]["x"][i], a["kKF"]["y"][i], 650)
                    k, ci = visits[(f, ix, iy)]
                    chunk = [cc for (kk, cc) in visits.values() if kk == k and cc // 32 == ci // 32 and cc < ci]
                    before = sum(start[(ff * G + xx) * G + yy + 1] - start[(ff * G + xx) * G + yy] for (ff, xx, yy), (kk, cc) in visits.items() if kk == k and cc in chunk)
                    cell = (f * G + ix) * G + iy
                    where.append((k, ci, ci % 32, before + list(idx[start[cell]:start[cell + 1]]).index(i)))
                (k0, c0, l0, p0), (k1, c1, l1, p1) = where
                if c["kind"] == "chunks":
                    assert k0 == k1 and c0 // 32 < c1 // 32 and l1 < l0 and p1 < p0, where
                if c["kind"] == "rects":
                    assert (k0, k1) == (1, 2) and l1 < l0 and p1 < p0, where
        seen.add(c["kind"])
    assert seen == {"cell", "cells", "chunks", "rects", "complement", "mixed_after", "mixed_before"}, seen
    # the window edge: exactly at the radius on one axis, in a visited cell, and dropped; one ulp inside kept
    for th in (1.0, 2.0):
        E = edge_scene(oracle, th); a = E.arrays(); g = oracle.FrameGrid(a["kKF"], 650, 650)
        for c in E.cases:
            edge = c["kps"][1]; kx, ky = a["kKF"]["x"][edge], a["kKF"]["y"][edge]
            d = max(abs(kx - c["u"]), abs(ky - c["v"]))
            assert d == c["r"] if c["kind"] == "edge" else 0 < c["r"] - d <= np.spacing(max(kx, ky))
            assert cell_of(kx, ky, 650) in {(f, ix, iy) for _, _, f, ix, iy in visit_cells(oracle, c["u"], c["v"], c["r"], 650)}
            assert (edge in g.features_in_area(c["u"], c["v"], c["r"])) == (c["kind"] == "ulp_inside")
    # seams and behind the camera: the in-face test fails, IsInImage passes, the MapPoint is valid and finds its key point
    a = seam_scene(oracle)
    bi, bd = oracle_fuse(oracle, a)
    for kind in (0, 2, 3):
        sel = (a["kind"] == kind) & (a["valid"] == 1) & (a["face"] < 0)
        assert sel.sum() > 20 and (bd[sel] <= 50).sum() > 20, kind
    # distinctive descriptors: first tied rows at >= 32 and >= 128, the global-memory sizes, and the order statistic deciding
    firsts, sizes = set(), set()
    for d in distinctive_sets(max_n=1025):
        N = len(d); sizes.add(N)
        med = medians(d); best = oracle.distinctive_descriptors(d, np.array([0, N], np.int32))[0]
        least = np.nonzero(med == med.min())[0]
        assert best == least[0]
        if len(least) > 1:
            firsts.add(int(least[0]))
    assert {0, 31, 32, 127, 128, 129, 1023} <= firsts, sorted(firsts)
    assert {1, 2, 3, 127, 128, 129, 1024, 1025} <= sizes
    flips = sum(int(np.argmin(medians(d)) != np.argmin(medians(d, len(d) // 2))) for d in distinctive_sets() if 2 <= len(d) <= 16 and len(d) % 2 == 0)
    assert flips >= 3, flips
    # triangulation: the seam epipole keeps in-face coordinates and rejects a match the (-1, -1) epipole lets through
    p = triangulation_pairs(oracle)[-1]
    c2 = transform(p["T2"], p["Ow"])
    assert oracle.ray_to_cubemap(c2, 450, 450)[1][0] == -1 and oracle.ray_to_cubemap(c2, 450, 450)[0][0, 0] == 450
    n_seam, m_seam = oracle_triangulation(oracle, p, 450, False)
    n_none, m_none = oracle_triangulation(oracle, dict(p, Ow=np.zeros(3, F32)), 450, False)
    assert n_none > n_seam and n_seam > 50


# ----------------------------------------------------------------------------------------------------------------- GPU parity
@pytest.mark.gpu
def test_fuse_ties_and_complements(oracle, mapper, scenes):
    check_fuse(oracle, mapper, scenes["ties"])


@pytest.mark.gpu
@pytest.mark.parametrize("th", ["edge1", "edge2"])
def test_fuse_window_edge(oracle, mapper, scenes, th):
    check_fuse(oracle, mapper, scenes[th])


@pytest.mark.gpu
@pytest.mark.parametrize("nlevels", [1, 4, 8])
def test_fuse_levels(oracle, mapper, scenes, nlevels):
    check_fuse(oracle, mapper, scenes["levels"][nlevels])


@pytest.mark.gpu
def test_fuse_seams_behind_origin(oracle, mapper, scenes):
    a = scenes["seam"]
    bi, bd = check_fuse(oracle, mapper, a)
    assert (bd[(a["face"] < 0) & (a["valid"] == 1)] <= 50).sum() > 60


@pytest.mark.gpu
def test_fuse_sizes(oracle, mapper):
    S = crowded_scene(oracle)
    assert len(S.kps) == 4096
    check_fuse(oracle, mapper, S)
    # 50 001 MapPoints (the last CTA holds one warp), on every face, at random depths and levels
    rng = np.random.default_rng(8)
    s = synth.mapping_pair(6, n=1500, faceW=650)
    n = 50001
    T = s["TcwCur"].astype(np.float64)
    pick = rng.integers(0, len(s["kCur"]), n)
    px = s["kCur"]["x"][pick] + rng.normal(0, 2, n); py = s["kCur"]["y"][pick] + rng.normal(0, 2, n)
    Xw = np.zeros((n, 3), F32)
    for i in range(n):
        ray = synth._pixel_to_ray(float(px[i]), float(py[i]), 650)
        ray = np.array([0.0, 0.0, 1.0]) if ray is None else ray
        Xw[i] = T[:3, :3].T @ (ray * rng.uniform(2, 12) - T[:3, 3])
    dMP = s["dCur"][pick] ^ np.packbits(rng.random((n, 256)) < 0.08, axis=1, bitorder="little")
    a = dict(kKF=s["kCur"], dKF=s["dCur"], Tcw=s["TcwCur"], valid=(rng.random(n) < 0.9).astype(np.uint8), Xw=Xw,
             level=np.clip(s["kCur"]["octave"][pick] + rng.integers(-1, 2, n), 0, 7).astype(np.int32), dMP=dMP, th=3.0, scale=s["scale"],
             isg=s["inv_level_sigma2"], W=650)
    bi, bd = check_fuse(oracle, mapper, a)
    assert (bd <= 50).sum() > 20000
    # no key points at all
    from oracle import KP_DTYPE
    a = dict(a, kKF=np.zeros(0, KP_DTYPE), dKF=np.zeros((0, 32), np.uint8))
    gi, gd = gpu_fuse(mapper, a)
    assert (gi == -1).all() and (gd == 256).all()
    bi, bd = oracle_fuse(oracle, a)
    assert (bi == -1).all() and (bd == 256).all()


@pytest.mark.gpu
@pytest.mark.parametrize("seed,th", [(0, 3.0), (2, 12.0)])
def test_fuse_450(oracle, mapper, seed, th):
    s = synth.mapping_pair(seed, n=1500, faceW=450)
    rng = np.random.default_rng(seed)
    n = len(s["Xw"])
    a = dict(kKF=s["kCur"], dKF=s["dCur"], Tcw=s["TcwCur"], valid=(rng.random(n) < 0.9).astype(np.uint8), Xw=s["Xw"],
             level=np.clip(s["kLast"]["octave"] + rng.integers(-1, 2, n), 0, 7).astype(np.int32), dMP=s["dLast"], th=th, scale=s["scale"],
             isg=s["inv_level_sigma2"], W=450)
    bi, bd = check_fuse(oracle, mapper, a)
    assert (bd <= 50).sum() > 150


@pytest.mark.gpu
def test_distinctive_ties_and_sizes(oracle, mapper):
    rng = np.random.default_rng(1)
    sets = distinctive_sets()
    desc, off, where = pack(sets, rng, lead=5)
    want = oracle.distinctive_descriptors(desc, off)
    got = mapper.ComputeDistinctiveDescriptors(desc, off)
    assert np.array_equal(got, want)
    for (N, rows), p in zip(TIE_SETS, where):
        assert want[p] == rows[0], (N, rows)
    assert (want[[p for p in range(len(off) - 1) if off[p] == off[p + 1]]] == -1).all()


@pytest.mark.gpu
def test_distinctive_100k_points(oracle, mapper):
    rng = np.random.default_rng(2)
    sets = []
    for _ in range(75000):
        N = int(rng.choice([1, 2, 3, 4, 5, 6, 9, 17]))
        base = rng.integers(0, 256, 32, dtype=np.uint8)
        sets.append(base ^ np.packbits(rng.random((N, 256)) < rng.uniform(0, 0.3), axis=1, bitorder="little"))
    desc, off, _ = pack(sets, rng, lead=3, empty_every=3)
    assert len(off) - 1 == 100000
    want = oracle.distinctive_descriptors(desc, off)
    assert np.array_equal(mapper.ComputeDistinctiveDescriptors(desc, off), want)


@pytest.mark.gpu
@pytest.mark.parametrize("ori", [False, True])
def test_search_for_triangulation_450(oracle, mapper, ori):
    W = 450
    ps = triangulation_pairs(oracle, W)
    P = len(ps)
    s1 = max(len(p["s"]["kCur"]) for p in ps); s2 = max(len(p["s"]["kLast"]) for p in ps)
    KP = ps[0]["s"]["kCur"].dtype
    k1 = np.zeros((P, s1), KP); d1 = np.zeros((P, s1, 32), np.uint8); r1 = np.zeros((P, s1, 3), F32); h1 = np.zeros((P, s1), np.uint8); nd1 = np.zeros((P, s1), np.int32)
    k2 = np.zeros((P, s2), KP); d2 = np.zeros((P, s2, 32), np.uint8); r2 = np.zeros((P, s2, 3), F32); h2 = np.zeros((P, s2), np.uint8); nd2 = np.zeros((P, s2), np.int32)
    n1 = np.zeros(P, np.int32); n2 = np.zeros(P, np.int32)
    want = []
    for i, p in enumerate(ps):
        s = p["s"]; a, b = len(s["kCur"]), len(s["kLast"]); n1[i] = a; n2[i] = b
        k1[i, :a] = s["kCur"]; d1[i, :a] = s["dCur"]; r1[i, :a] = oracle.key_point_rays(s["kCur"], W, W)[0]; h1[i, :a] = s["hasMPCur"]; nd1[i, :a] = s["nodeCur"]
        k2[i, :b] = s["kLast"]; d2[i, :b] = s["dLast"]; r2[i, :b] = oracle.key_point_rays(s["kLast"], W, W)[0]; h2[i, :b] = s["hasMPObs"]; nd2[i, :b] = s["nodeObs"]
        want.append(oracle_triangulation(oracle, p, W, ori))
    Ow = np.stack([p["Ow"] for p in ps]); T2 = np.stack([np.asarray(p["T2"], F32).reshape(16) for p in ps]); E = np.stack([np.asarray(p["E"], F32).reshape(9) for p in ps])
    nm, m = mapper.SearchForTriangulation(k1, d1, r1, h1, nd1, n1, k2, d2, r2, h2, nd2, n2, Ow, T2, E, ps[0]["s"]["scale"], ps[0]["s"]["level_sigma2"], W, W, ori)
    for i in range(P):
        assert nm[i] == want[i][0], (i, nm[i], want[i][0])
        assert np.array_equal(m[i, :n1[i]], want[i][1]), i
    assert want[3][0] == 0 and min(w[0] for i, w in enumerate(want) if i != 3) > 50

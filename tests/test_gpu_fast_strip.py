"""k_fast walks a strip of consecutive cell rows per CTA, double-buffering the tiles; these tests compare it with the CPU oracle, bit for bit
(tests marked gpu).

Each tile of a strip must behave exactly like a tile scored on its own. The caller canvases below place, in consecutive cell rows of one tile
column: a cell whose only corner passes the initial threshold above or below a cell whose corners only pass the minimum one (the 20 -> 7
fallback is decided per cell, so a count left over from the previous tile would drop them); a densely textured cell row directly above a
flat one (scores left over from the previous tile would show up as candidates); and textured tiles between all-zero tiles, which the kernel
skips, at the start, middle and end of strips, with whole strips of zero tiles. Candidates of every level, key points and descriptors are
compared. On the warp path, strips start and end in the black canvas corners, whose tiles are skipped, and at the face sizes used here some
levels have an odd number of cell rows, so their last strip is shorter than the others."""
import os

import numpy as np
import pytest

from cubemapslam_b200 import _capi, config, synth

pytestmark = pytest.mark.gpu
NTHREADS = max(1, min(32, os.cpu_count() or 1))
FACE = 450
BG = 100


def _cells(side):
    """Level geometry of a side x side level: (minB, wCell = hCell, nColsEff = nRowsEff), as the front end computes it."""
    minB, maxB = 16, side - 16
    width = np.float32(maxB - minB)
    n = int(width / np.float32(30))
    cell = int(np.ceil(width / np.float32(n)))
    neff = max(j + 1 for j in range(n) if not minB + j * cell >= maxB - 6)
    return minB, cell, neff


def _level_sides(face, nlevels=8):
    return [int(np.rint(np.float32(3 * face) * (np.float32(1.0) / np.float32(np.float32(1.2) ** l)))) for l in range(nlevels)]


def _origin(i, j):
    """Canvas position of the first detection pixel of level-0 cell (row i, column j)."""
    minB, cell, _ = _cells(3 * FACE)
    return minB + 3 + i * cell, minB + 3 + j * cell


def _spike(c, i, j, dy, dx, d):
    """One pixel d above a flat field: arc score |d| at that pixel and 0 around it."""
    y, x = _origin(i, j)
    c[y + dy, x + dx] = BG + d


def _fallback_canvas():
    c = np.full((3 * FACE, 3 * FACE), BG, np.uint8)
    for j in (1, 6, 13, 22):
        # a strong corner (s = 60 > iniTh) above a cell with weak corners only (minTh < s <= iniTh), in every pair of consecutive rows
        for i0 in range(0, 12, 3):
            _spike(c, i0, j, 9, 11, 60)
            _spike(c, i0 + 1, j, 5, 7, 12); _spike(c, i0 + 1, j, 18, 20, -15)
        # and the reverse order
        for i0 in range(14, 26, 3):
            _spike(c, i0, j, 12, 4, 13); _spike(c, i0, j, 20, 15, -9)
            _spike(c, i0 + 1, j, 8, 8, -70)
    return c


def _texture_canvas(seed):
    """Noise over whole cell rows directly above flat ones, in several tile columns and rows."""
    rng = np.random.default_rng(seed)
    c = np.full((3 * FACE, 3 * FACE), BG, np.uint8)
    _, cell, _ = _cells(3 * FACE)
    for i in (2, 5, 8, 17, 30):
        y, x = _origin(i, 4 * (i % 5))
        c[y:y + cell, x:x + 8 * cell] = rng.integers(0, 256, (cell, 8 * cell))
    return c


def _dead_canvas(seed):
    """A zero canvas with textured tiles only in some cell rows of a few tile columns (texture kept 5 px inside its cells, so the tiles
    around it stay all-zero up to their halo)."""
    rng = np.random.default_rng(seed)
    c = np.zeros((3 * FACE, 3 * FACE), np.uint8)
    _, cell, n = _cells(3 * FACE)
    for tc, rows in ((1, (1, 2, 5)), (3, (0, 3, 9, 10)), (6, (7, 8, 15)), (9, (n - 1,))):
        for i in rows:
            y, x = _origin(i, 4 * tc + 1)
            c[y + 5:y + cell - 5, x + 5:x + 2 * cell - 5] = rng.integers(0, 256, (cell - 10, 2 * cell - 10))
    return c


def _key(a):
    return a[np.lexsort((a[:, 0], a[:, 1]))]


@pytest.fixture(scope="module")
def geom(oracle):
    cfg = config.camera("lafida_cam0_params", CubeFace_w=FACE, CubeFace_h=FACE)
    cp = oracle.cam_params(cfg)
    return cfg, cp, oracle.build_maps(cp), np.full((3 * FACE, 3 * FACE), 255, np.uint8)


def _check_canvases(oracle, fe, canv, mask, what):
    o = fe.orb
    got = fe.extract(canv)
    for f in range(len(canv)):
        ex = oracle.ORBextractor(o.nfeatures, o.scale_factor, o.nlevels, o.ini_th_fast, o.min_th_fast, FACE, FACE)
        kps, desc = ex(canv[f], mask)
        for l in range(o.nlevels):
            c = ex.stage(l, 0)
            ref = np.stack([c["x"], c["y"], c["response"]], 1).astype(np.int32)
            g = fe.candidates(f, l)
            assert len(g) == len(ref), "%s canvas %d level %d: %d candidates vs %d" % (what, f, l, len(g), len(ref))
            assert np.array_equal(_key(g), _key(ref)), "%s canvas %d level %d candidates" % (what, f, l)
        gk, gd = got[f]
        assert len(gk) == len(kps), "%s canvas %d: %d key points vs %d" % (what, f, len(gk), len(kps))
        assert np.array_equal(gk.view(np.uint8), kps.view(np.uint8)) and np.array_equal(gd, desc), "%s canvas %d" % (what, f)


def test_fallback_does_not_leak_between_tiles(oracle, geom):
    from cubemapslam_b200.frontend import FrontEnd
    cfg, _, _, mask = geom
    canv = _fallback_canvas()[None]
    fe = FrontEnd(cfg, mask, max_batch=1)
    try:
        _check_canvases(oracle, fe, canv, mask, "fallback")
        # the weak corners are kept: every level-0 spike of the canvas is a candidate
        assert len(fe.candidates(0, 0)) == int((canv[0] != BG).sum())
    finally:
        fe.close()


def test_scores_do_not_leak_between_tiles(oracle, geom):
    from cubemapslam_b200.frontend import FrontEnd
    cfg, _, _, mask = geom
    canv = np.stack([_texture_canvas(s) for s in (1, 2)])
    fe = FrontEnd(cfg, mask, max_batch=2)
    try:
        _check_canvases(oracle, fe, canv, mask, "texture")
    finally:
        fe.close()


def test_dead_tiles_in_strips(oracle, geom):
    from cubemapslam_b200.frontend import FrontEnd
    cfg, _, _, mask = geom
    canv = np.stack([_dead_canvas(s) for s in (3, 4, 5)])
    fe = FrontEnd(cfg, mask, max_batch=3)
    try:
        _check_canvases(oracle, fe, canv, mask, "dead tiles")
    finally:
        fe.close()


@pytest.mark.parametrize("face", [333, 450, 560, 650])
def test_short_strips_warp_path(oracle, face):
    from cubemapslam_b200.frontend import FrontEnd
    assert any(_cells(s)[2] % 2 for s in _level_sides(face)), "no level with an odd number of cell rows"
    cfg = config.camera("front_cam_params", Camera_Ih=1024, Camera_v0=512.0, CubeFace_w=face, CubeFace_h=face)
    mask = np.full((3 * face, 3 * face), 255, np.uint8)
    frames = np.stack([synth.fisheye_frame(cfg, i) for i in range(13)])
    frames[5, 0, 0] = 90   # the out-of-view class differs from the black corners
    fe = FrontEnd(cfg, mask, max_batch=13)
    try:
        cp = oracle.cam_params(cfg)
        m1, m2 = oracle.build_maps(cp)
        o = fe.orb
        rk, rd, rn = oracle.warp_extract_batch_out(cp, frames, m1, m2, mask, o.nfeatures, o.scale_factor, o.nlevels, o.ini_th_fast,
                                                   o.min_th_fast, NTHREADS, fe.kp_cap)
        for b in (1, 3, 13):
            got = fe.run(frames[:b])
            for i in range(b):
                gk, gd = got[i]
                assert len(gk) == rn[i], "face %d batch %d frame %d: %d key points vs %d" % (face, b, i, len(gk), rn[i])
                assert np.array_equal(gk.view(np.uint8), rk[i, :rn[i]].view(np.uint8)), "face %d batch %d frame %d" % (face, b, i)
                assert np.array_equal(gd, rd[i, :rn[i]]), "face %d batch %d frame %d descriptors" % (face, b, i)
    finally:
        fe.close()


def test_caller_canvas_then_warp_path(oracle, geom):
    """Strip canvases through cslam_orb_extract, then the warp path on the same front end: equal to a fresh front end and the oracle."""
    from cubemapslam_b200.frontend import FrontEnd
    cfg, cp, maps, mask = geom
    canv = np.stack([_fallback_canvas(), _texture_canvas(7), _dead_canvas(8)])
    frames = np.stack([synth.fisheye_frame(cfg, i) for i in range(3)])
    fe = FrontEnd(cfg, mask, max_batch=3); fresh = FrontEnd(cfg, mask, max_batch=3)
    try:
        _check_canvases(oracle, fe, canv, mask, "before the warp path")
        got = fe.run(frames)
        want = fresh.run(frames)
        o = fe.orb
        rk, rd, rn = oracle.warp_extract_batch_out(cp, frames, maps[0], maps[1], mask, o.nfeatures, o.scale_factor, o.nlevels, o.ini_th_fast,
                                                   o.min_th_fast, NTHREADS, fe.kp_cap)
        for f in range(3):
            assert np.array_equal(got[f][0].view(np.uint8), want[f][0].view(np.uint8)) and np.array_equal(got[f][1], want[f][1]), "frame %d" % f
            assert len(got[f][0]) == rn[f] and np.array_equal(got[f][0].view(np.uint8), rk[f, :rn[f]].view(np.uint8)), "frame %d" % f
            assert np.array_equal(got[f][1], rd[f, :rn[f]]), "frame %d descriptors" % f
    finally:
        fe.close(); fresh.close()

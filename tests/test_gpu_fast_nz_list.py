"""k_fast's phase B (NMS) walks only the items phase A scored non-zero (the tile's nz list); these tests compare the candidates with the CPU
oracle, bit for bit (tests marked gpu), where that list is empty, full, or filled only in the last round of phase A's loop, on caller
canvases (cslam_orb_extract: every item of a tile is scored) and on the warp path (only the live items are)."""
import numpy as np
import pytest

from tests.test_gpu_fast_output import FACE, _cells, _check_canvases, _key, geom  # noqa: F401 (geom: fixture)

pytestmark = pytest.mark.gpu
BG, SPIKE = 20, 220


def _full(c, y0, y1, x0, x1):
    """Spikes at x = 0 mod 4 on even rows and x = 2 mod 4 on odd rows: one in every 4 adjacent pixels of a row, none on another's FAST
    ring or in its 3x3 neighbourhood, so every 4-pixel work item holds a corner that survives NMS."""
    for y in range(y0, y1):
        c[y, x0 + (-(x0 - 2 * (y & 1)) % 4):x1:4] = SPIKE


def _canvas():
    return np.full((3 * FACE, 3 * FACE), BG, np.uint8)


def _full_tile_canvas():
    """Level-0 tile (cell row 9, tile column 1) covered with _full over its whole ROI (the detection area plus the 3-pixel halo):
    every item of the tile scores, so the nz list holds all nw x ny items."""
    minB, cell, _ = _cells(3 * FACE)
    c = _canvas()
    y0, x0 = minB + 9 * cell, minB + 4 * cell
    _full(c, y0, y0 + cell + 6, x0, x0 + 4 * cell + 6)
    return c


def _last_round_canvas():
    """Corners only in the last detection row of level-0 tiles (cell row 5, tile columns 0 and 2): row-major item order puts them in
    the last round of phase A's loop (items 256 * k.. of a tile with nw x ny > 256 items), in its last warp."""
    minB, cell, _ = _cells(3 * FACE)
    c = _canvas()
    y = minB + 5 * cell + 3 + cell - 1
    for tc in (0, 2):
        x0 = minB + 4 * tc * cell + 3
        _full(c, y, y + 1, x0 + 2 * cell, x0 + 4 * cell)
    return c


def test_caller_canvases_empty_full_and_last_round(oracle, geom):
    from cubemapslam_b200.frontend import FrontEnd
    cfg, mask = geom
    # a flat canvas: every tile is scored (it is not all zero) and every tile's nz list is empty
    canv = np.stack([_canvas(), _full_tile_canvas(), _last_round_canvas()])
    fe = FrontEnd(cfg, mask, max_batch=len(canv))
    try:
        _check_canvases(oracle, fe, canv, mask, "nz list")
        assert len(fe.candidates(0, 0)) == 0
        # every spike is a level-0 candidate (the ones in the full tile's halo in the neighbouring tiles')
        assert len(fe.candidates(1, 0)) == int((canv[1] == SPIKE).sum())
        assert len(fe.candidates(2, 0)) == int((canv[2] == SPIKE).sum()) > 0
    finally:
        fe.close()


def _check_warp(oracle, fe, frames, mask, what):
    """fe.run (warp path: live lists) against the oracle's warp + extract, candidates of every level and the key points."""
    cfg, o = fe.cfg, fe.orb
    cp = oracle.cam_params(cfg)
    m1, m2 = oracle.build_maps(cp)
    got = fe.run(frames)
    for f in range(len(frames)):
        ex = oracle.ORBextractor(o.nfeatures, o.scale_factor, o.nlevels, o.ini_th_fast, o.min_th_fast, FACE, FACE)
        kps, desc = ex(oracle.warp(cp, frames[f], m1, m2), mask)
        for l in range(o.nlevels):
            c = ex.stage(l, 0)
            ref = np.stack([c["x"], c["y"], c["response"]], 1).astype(np.int32)
            g = fe.candidates(f, l)
            assert len(g) == len(ref), "%s frame %d level %d: %d candidates vs %d" % (what, f, l, len(g), len(ref))
            assert np.array_equal(_key(g), _key(ref)), "%s frame %d level %d candidates" % (what, f, l)
        gk, gd = got[f]
        assert len(gk) == len(kps) and np.array_equal(gk.view(np.uint8), kps.view(np.uint8)) and np.array_equal(gd, desc), "%s frame %d" % (what, f)


def test_warp_path_sparse_and_dense_lists(oracle, geom):
    """A constant fisheye frame leaves corners only where the faces meet the black canvas corners (nearly every live item scores 0);
    the synthetic textured frame gives lists of about half the live items."""
    from cubemapslam_b200 import synth
    from cubemapslam_b200.frontend import FrontEnd
    cfg, mask = geom
    Ih, Iw = int(cfg["Camera.Ih"]), int(cfg["Camera.Iw"])
    frames = np.stack([np.full((Ih, Iw), 128, np.uint8), synth.fisheye_frame(cfg, 3)])
    fe = FrontEnd(cfg, mask, max_batch=len(frames))
    try:
        _check_warp(oracle, fe, frames, mask, "warp path")
    finally:
        fe.close()

"""k_fast collects a strip's candidates in a shared-memory buffer and copies them to the frame's list when the buffer could not hold another
tile's survivors and at the end of the strip; these tests compare it with the CPU oracle, bit for bit (tests marked gpu).

The caller canvases below hold isolated spikes (one pixel above a flat field, no other spike on its ring, so every spike is a corner that
survives NMS) at one spike per 8 pixels: about 480 candidates per level-0 tile, several times the buffer's room per strip. One canvas fills
whole strips of one tile column; one fills the middle of a strip whose first and last tiles are all zero, which the kernel skips (the last
one ends the strip without scoring); one covers the whole level, more candidates than the level's list holds, which must be reported as
CSLAM_E_CAPACITY and leave the front end correct for the next call. Candidate lists are compared sorted: their order depends on the order
in which CTAs reach the frame's count."""
import numpy as np
import pytest

from cubemapslam_b200 import config

pytestmark = pytest.mark.gpu
FACE = 450
SPIKE = 60


def _cells(side):
    """Level geometry of a side x side level: (minB, wCell = hCell, nColsEff = nRowsEff), as the front end computes it."""
    minB, maxB = 16, side - 16
    width = np.float32(maxB - minB)
    n = int(width / np.float32(30))
    cell = int(np.ceil(width / np.float32(n)))
    neff = max(j + 1 for j in range(n) if not minB + j * cell >= maxB - 6)
    return minB, cell, neff


def _spikes(c, y0, y1, x0, x1, bg):
    """Spikes over rows [y0, y1) and columns [x0, x1): every 2nd column and every 4th row, so no spike lies on another's FAST ring."""
    c[y0:y1:4, x0:x1:2] = bg + SPIKE


def _strip_canvas():
    """Spikes over cell rows 8..23 (level-0 strips 1 and 2) of tile column 2 (cells 8..11) on a flat field."""
    bg = 100
    minB, cell, _ = _cells(3 * FACE)
    c = np.full((3 * FACE, 3 * FACE), bg, np.uint8)
    _spikes(c, minB + 3 + 8 * cell, minB + 3 + 24 * cell, minB + 3 + 8 * cell, minB + 3 + 12 * cell, bg)
    return c


def _dead_ends_canvas():
    """A zero canvas with spikes in cell rows 9..14 of level-0 strip 1 (rows 8..15), kept out of the 6 halo rows that tile row 8 loads
    below its cell row, so the strip's first and last tiles (rows 8 and 15) stay all-zero, in two tile columns."""
    minB, cell, _ = _cells(3 * FACE)
    c = np.zeros((3 * FACE, 3 * FACE), np.uint8)
    for tc in (1, 5):
        _spikes(c, minB + 9 * cell + 8, minB + 15 * cell - 4, minB + 3 + 4 * tc * cell, minB + 3 + 4 * (tc + 1) * cell, 0)
    return c


def _key(a):
    return a[np.lexsort((a[:, 0], a[:, 1]))]


@pytest.fixture(scope="module")
def geom():
    cfg = config.camera("lafida_cam0_params", CubeFace_w=FACE, CubeFace_h=FACE)
    return cfg, np.full((3 * FACE, 3 * FACE), 255, np.uint8)


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


def test_strip_overflows_buffer(oracle, geom):
    from cubemapslam_b200.frontend import FrontEnd
    cfg, mask = geom
    canv = _strip_canvas()[None]
    fe = FrontEnd(cfg, mask, max_batch=1)
    try:
        _check_canvases(oracle, fe, canv, mask, "dense strips")
        # every level-0 spike is a candidate: 3 844 in each of the two strips, more than the strip buffer's 2 304 entries
        assert len(fe.candidates(0, 0)) == int((canv[0] != 100).sum()) > 3 * 2304
    finally:
        fe.close()


def test_strip_with_dead_first_and_last_tiles(oracle, geom):
    from cubemapslam_b200.frontend import FrontEnd
    cfg, mask = geom
    canv = np.stack([_dead_ends_canvas(), _strip_canvas()])
    fe = FrontEnd(cfg, mask, max_batch=2)
    try:
        _check_canvases(oracle, fe, canv, mask, "dead ends")
        g = fe.candidates(0, 0)
        assert len(np.unique(g[:, :2], axis=0)) == len(g) == int((canv[0] != 0).sum())
    finally:
        fe.close()


def test_candidate_list_overflow_is_reported(oracle, geom):
    from cubemapslam_b200 import _capi
    from cubemapslam_b200.frontend import FrontEnd
    cfg, mask = geom
    full = np.full((3 * FACE, 3 * FACE), 100, np.uint8)
    _spikes(full, 0, 3 * FACE, 0, 3 * FACE, 100)
    fe = FrontEnd(cfg, mask, max_batch=1)
    try:
        with pytest.raises(_capi.CslamError, match="error -4"):
            fe.extract(full)
        _check_canvases(oracle, fe, _strip_canvas()[None], mask, "after an overflow")
    finally:
        fe.close()

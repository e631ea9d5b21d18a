"""k_fast's compass pretest (phase A0) drops a work item only when the compass bound proves all 4 of its arc scores <= minThFAST; these tests
compare the candidates and key points with the CPU oracle, bit for bit (tests marked gpu), on canvases where many pixels sit exactly on
that bound, through cslam_orb_extract (every item of a tile is tested) and through the warp path (only the live items are).

Each stamp is a centre c on a flat field of c with its 16-pixel ring set: compass pairs (ring 0 and 4, or 8 and 12) at c +- mt or
c +- (mt + 1), the 9-run from the first of them filled at the same value or broken by one pixel at c, so the exact scores are mt, mt + 1
or 0 while the bound is mt or mt + 1; and saturated 0 / 255 stamps, scores of 255. One tile holds low-contrast noise whose every
difference is <= 7 (each of its items is rejected at minThFAST 7 and above), one holds a corner in every item (none is rejected)."""
import numpy as np
import pytest

from tests.test_gpu_fast_nz_list import _check_warp, _full
from tests.test_gpu_fast_output import FACE, _cells, _check_canvases, geom  # noqa: F401 (geom: fixture)
from tests.test_gpu_fast_score import _orb

pytestmark = pytest.mark.gpu
RING = [(0, -3), (1, -3), (2, -2), (3, -1), (3, 0), (3, 1), (2, 2), (1, 3), (0, 3), (-1, 3), (-2, 2), (-3, 1), (-3, 0), (-3, -1), (-2, -2), (-1, -3)]
THRESHOLDS = [(20, 0), (12, 1), (20, 7), (255, 255)]
PITCH = 11   # stamp spacing: no stamp's 7x7 window reaches another's ring


def _stamps(mt, rng):
    """7x7 stamps (value arrays, centre at [3, 3]) that put their centre on the compass bound at margin mt."""
    out = []
    for c in (40, 128, 215):
        for sign in (1, -1):
            for d in (mt, mt + 1):
                v = int(np.clip(c + sign * d, 0, 255))
                for start in (0, 8, 4, 12):          # the run begins at a compass point and holds the next one
                    for gap in (None, 2, 6):         # a pixel at c inside the run: the bound still passes, the score is 0
                        s = np.full((7, 7), c, np.int32)
                        for k in range(9):
                            dx, dy = RING[(start + k) % 16]
                            s[3 + dy, 3 + dx] = c if gap is not None and k == gap else v
                        out.append(s)
    for c, v in ((0, 255), (255, 0)):                # score 255
        s = np.full((7, 7), c, np.int32)
        for k in range(int(rng.integers(0, 16)), 16 + 9):
            dx, dy = RING[k % 16]
            s[3 + dy, 3 + dx] = v
        out.append(s)
    return out


def _bound_canvas(mn, seed, bg=100):
    """The stamps of minThFAST mn on a grid over a FACE x FACE square of the level-0 canvas, on a field of bg (about 1 700 stamps: the
    candidates stay well inside the level's list)."""
    mt = min(max(mn, 1), 255)
    rng = np.random.default_rng(seed)
    c = np.full((3 * FACE, 3 * FACE), bg, np.uint8)
    st = _stamps(mt, rng)
    k = 0
    for y in range(FACE // 2, 3 * FACE // 2 - 7, PITCH):
        for x in range(FACE // 2 + (y % 4), 3 * FACE // 2 - 7, PITCH):
            c[y:y + 7, x:x + 7] = st[k % len(st)]
            k += 1
    return c


def _reject_all_and_none_canvas():
    """Level-0 tile (cell row 4, tile column 0): noise in 100..107, every item rejected at mt >= 7; tile (cell row 4, tile column 2):
    _full's spikes, every item holds a corner."""
    minB, cell, _ = _cells(3 * FACE)
    rng = np.random.default_rng(7)
    c = np.full((3 * FACE, 3 * FACE), 100, np.uint8)
    y0 = minB + 4 * cell
    c[y0:y0 + cell + 6, minB:minB + 4 * cell + 6] = rng.integers(100, 108, (cell + 6, 4 * cell + 6))
    x0 = minB + 8 * cell
    _full(c, y0, y0 + cell + 6, x0, x0 + 4 * cell + 6)
    return c


@pytest.mark.parametrize("ini,mn", THRESHOLDS)
def test_caller_canvases_on_the_bound(oracle, geom, ini, mn):
    from cubemapslam_b200.frontend import FrontEnd
    cfg, mask = geom
    canv = np.stack([_bound_canvas(mn, 1), _bound_canvas(mn, 2, bg=30), _reject_all_and_none_canvas()])
    fe = FrontEnd(cfg, mask, max_batch=len(canv), orb=_orb(cfg, ini, mn))
    try:
        _check_canvases(oracle, fe, canv, mask, "pretest (%d,%d)" % (ini, mn))
        if mn <= 7:   # every spike of the fully passing tile is a corner at these thresholds (the noise tile has none at 7)
            assert len(fe.candidates(2, 0)) >= int((canv[2] == 220).sum())
    finally:
        fe.close()


@pytest.mark.parametrize("ini,mn", THRESHOLDS)
def test_warp_path_on_the_bound(oracle, geom, ini, mn):
    """The stamps pasted into fisheye frames: the warp resamples them, so the frames hold bound-edge pixels beside scene texture."""
    from cubemapslam_b200 import synth
    from cubemapslam_b200.frontend import FrontEnd
    cfg, mask = geom
    Ih, Iw = int(cfg["Camera.Ih"]), int(cfg["Camera.Iw"])
    frames = []
    for i in range(2):
        f = synth.fisheye_frame(cfg, i).copy()
        b = _bound_canvas(mn, 10 + i)[FACE // 2:FACE // 2 + min(FACE, Ih // 2), FACE // 2:FACE // 2 + min(FACE, Iw // 2)]
        y0, x0 = Ih // 4 + 3 * i, Iw // 4 + 5 * i
        f[y0:y0 + b.shape[0], x0:x0 + b.shape[1]] = b
        frames.append(f)
    frames = np.stack(frames).astype(np.uint8)
    fe = FrontEnd(cfg, mask, max_batch=len(frames), orb=_orb(cfg, ini, mn))
    try:
        _check_warp(oracle, fe, frames, mask, "pretest warp (%d,%d)" % (ini, mn))
    finally:
        fe.close()

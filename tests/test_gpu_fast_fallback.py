"""k_fast selects key points in two rounds: the NMS at minThFAST keeps the survivors above iniThFAST, and only the cells where none survives
score their deferred items (compass bound <= iniThFAST) and run the NMS again, keeping every survivor there. These tests compare the
candidates and key points with the CPU oracle, bit for bit (tests marked gpu), through cslam_orb_extract and through the warp path, on
canvases with: a cell whose only scores above iniThFAST are a tie plateau, cells whose only corners lie in deferred items, fallback and
non-fallback cells that share a 4-pixel item, whole tiles without fallback and whole tiles of fallback. An iniThFAST below minThFAST acts
as minThFAST, so those front ends are compared with the oracle at (minThFAST, minThFAST)."""
import numpy as np
import pytest

from tests.test_gpu_fast_nz_list import _check_warp
from tests.test_gpu_fast_output import FACE, _cells, _check_canvases, geom  # noqa: F401 (geom: fixture)
from tests.test_gpu_fast_score import _orb

pytestmark = pytest.mark.gpu
THRESHOLDS = [(20, 7), (20, 0), (12, 1), (7, 7), (5, 7), (0, 0), (255, 7), (255, 255)]
BG, STRONG, WEAK = 100, 60, 12   # spike contrasts: an isolated spike scores its contrast (above 20, and between 7 and 20)


def _spikes(c, y0, y1, x0, x1, d):
    """Spikes of contrast d on every 2nd column and every 4th row of [y0, y1) x [x0, x1): none lies on another's FAST ring."""
    c[y0:y1:4, x0:x1:2] = BG + d


def _plateaus(c, y0, y1, x0, x1):
    """Horizontal pairs of equal strong spikes, 8 pixels apart: both pixels score STRONG, so neither survives the NMS at any threshold."""
    for y in range(y0, y1, 8):
        for x in range(x0, x1 - 1, 8):
            c[y, x:x + 2] = BG + STRONG


def _fallback_canvas(r=4):
    """Level-0 cell row r. Tile column 0: strong spikes in all 4 cells (no fallback). Tile column 1: weak spikes in all 4 cells (the whole
    tile falls back; its corners lie in deferred items at iniThFAST 20). Tile column 2: cell 0 strong spikes up to its last column and
    cell 1 weak spikes from its first (the items across their border hold both), cell 2 plateaus beside weak spikes, cell 3 plateaus
    only. Tile column 3: strong spikes in cells 0 and 2, nothing in cells 1 and 3."""
    minB, cell, _ = _cells(3 * FACE)
    c = np.full((3 * FACE, 3 * FACE), BG, np.uint8)
    y0, y1 = minB + 3 + r * cell, minB + 3 + (r + 1) * cell
    cx = lambda j: minB + 3 + j * cell   # noqa: E731   first detection column of level-0 cell j
    _spikes(c, y0, y1, cx(0), cx(4), STRONG)
    _spikes(c, y0, y1, cx(4), cx(8), WEAK)
    _spikes(c, y0, y1, cx(8), cx(9), STRONG)
    _spikes(c, y0, y1, cx(9) + (cx(9) - cx(8)) % 2, cx(10), WEAK)   # the spike columns continue across the border
    _plateaus(c, y0, y1, cx(10), cx(11))
    _spikes(c, y0 + 2, y1, cx(10) + 4, cx(11), WEAK)
    _plateaus(c, y0, y1, cx(11), cx(12))
    _spikes(c, y0, y1, cx(12), cx(13), STRONG)
    _spikes(c, y0, y1, cx(14), cx(15), STRONG)
    return c


def _orbs(cfg, ini, mn):
    """The front end's thresholds, and the oracle's: an iniThFAST below minThFAST acts as minThFAST."""
    return _orb(cfg, ini, mn), max(ini, mn)


@pytest.mark.parametrize("ini,mn", THRESHOLDS)
def test_caller_canvases_fall_back_per_cell(oracle, geom, ini, mn):
    from cubemapslam_b200.frontend import FrontEnd
    cfg, mask = geom
    canv = np.stack([_fallback_canvas(4), _fallback_canvas(9)[:, ::-1].copy()])
    orb, ref_ini = _orbs(cfg, ini, mn)
    fe = FrontEnd(cfg, mask, max_batch=len(canv), orb=orb)
    try:
        fe.orb.ini_th_fast = ref_ini   # the oracle's; the front end copied its own at create
        _check_canvases(oracle, fe, canv, mask, "fallback (%d,%d)" % (ini, mn))
    finally:
        fe.close()


@pytest.mark.parametrize("ini,mn", THRESHOLDS)
def test_warp_path_falls_back_per_cell(oracle, geom, ini, mn):
    """The canvases pasted into a flat and a textured fisheye frame: the warp resamples them into weak and strong corners and plateaus."""
    from cubemapslam_b200 import synth
    from cubemapslam_b200.frontend import FrontEnd
    cfg, mask = geom
    Ih, Iw = int(cfg["Camera.Ih"]), int(cfg["Camera.Iw"])
    frames = []
    for i, f in enumerate((np.full((Ih, Iw), BG, np.uint8), synth.fisheye_frame(cfg, 5).copy())):
        b = _fallback_canvas(4 + i)[FACE // 2:FACE // 2 + min(FACE, Ih // 2), FACE // 2:FACE // 2 + min(FACE, Iw // 2)]
        y0, x0 = Ih // 4 + 2 * i, Iw // 4 + 3 * i
        f[y0:y0 + b.shape[0], x0:x0 + b.shape[1]] = b
        frames.append(f)
    frames = np.stack(frames).astype(np.uint8)
    orb, ref_ini = _orbs(cfg, ini, mn)
    fe = FrontEnd(cfg, mask, max_batch=len(frames), orb=orb)
    try:
        fe.orb.ini_th_fast = ref_ini
        _check_warp(oracle, fe, frames, mask, "fallback warp (%d,%d)" % (ini, mn))
    finally:
        fe.close()

"""k_fast selects FAST key points in two rounds (frontend.cu): round 1 runs the NMS at minThFAST over the items that scored above iniThFAST
and keeps the survivors above iniThFAST; round 2 scores the deferred items (compass bound <= iniThFAST) of the cells round 1 left empty and
runs the NMS at minThFAST there. A numpy model of those rounds, on random tiles, must select exactly what one NMS at minThFAST plus the
per-cell iniThFAST filter selects, and what the reference's per-cell cv::FAST at iniThFAST with the fallback to minThFAST selects (an
iniThFAST below minThFAST acting as minThFAST). Ties and plateaus above iniThFAST, cells that fall back beside cells that do not, and items
that straddle two cells are all common on these tiles. CPU only."""
import numpy as np
import pytest

CG = 4   # cells per tile, as in frontend.cu
PAIRS = [(20, 7), (20, 0), (12, 1), (7, 7), (5, 7), (0, 0), (255, 7), (255, 255), (300, 7), (-3, -5), (9, 8), (30, 12)]


def _nms(r, cells, thr_keep):
    """Per-cell 3x3 NMS of the response map r (0 = not a corner): a pixel is kept iff r > thr_keep and r > every same-cell neighbour."""
    h, w = r.shape
    keep = np.zeros((h, w), bool)
    for c in range(cells.max() + 1):
        cols = np.flatnonzero(cells == c)
        if not len(cols):
            continue
        sub = np.pad(r[:, cols[0]:cols[-1] + 1], 1)
        nb = np.max([sub[1 + dy:h + 1 + dy, 1 + dx:len(cols) + 1 + dx] for dy in (-1, 0, 1) for dx in (-1, 0, 1) if dy or dx], 0)
        keep[:, cols] = (sub[1:-1, 1:-1] > nb) & (sub[1:-1, 1:-1] > thr_keep)
    return keep


def _reference(s, cells, ini, mn):
    """cv::FAST per cell at iniTh, and at minTh in the cells that found nothing: the response of a corner is s - 1, 0 otherwise."""
    def fast(t):
        t = min(max(t, 0), 255)
        return _nms(np.where(s > t, s - 1, 0), cells, 0) & (s > t)
    hi, lo = fast(ini), fast(mn)
    out = hi.copy()
    for c in range(cells.max() + 1):
        if not hi[:, cells == c].any():
            out[:, cells == c] = lo[:, cells == c]
    return out


def _one_round(s, cells, ini, mn):
    """NMS at mt = clamp(minTh, 1, 255) and the per-cell filter s > iniTh unless the cell has no such survivor."""
    mt = min(max(mn, 1), 255)
    surv = _nms(np.where(s > mt, s, 0), cells, 0)
    out = surv.copy()
    for c in range(cells.max() + 1):
        m = cells == c
        if (surv[:, m] & (s[:, m] > ini)).any():
            out[:, m] = surv[:, m] & (s[:, m] > ini)
    return out


def _two_rounds(s, bound, cells, valid, ini, mn):
    """k_fast's rounds over 4-pixel items (columns 4k..4k+3 of the padded tile; `valid` marks the detection area)."""
    mt = min(max(mn, 1), 255)
    ti = max(min(max(ini, 1), 255), mt)
    h, w = s.shape
    items = [(y, k) for y in range(h) for k in range(w // 4)]
    lanes = lambda y, k: (y, slice(4 * k, 4 * k + 4))   # noqa: E731
    passed = [it for it in items if (bound[lanes(*it)] > ti).any()]
    deferred = [it for it in items if it not in passed and (bound[lanes(*it)] > mt).any()]
    S = np.zeros_like(s)
    for it in passed:
        S[lanes(*it)] = np.where(s[lanes(*it)] > mt, s[lanes(*it)], 0)
    nz_hi = [it for it in passed if (S[lanes(*it)] > ti).any()]
    nz_lo = [it for it in passed if it not in nz_hi and S[lanes(*it)].any()]
    vc = np.where(valid, cells, -1)
    out = np.zeros((h, w), bool)
    # round 1: survivors above ti of the nzHi items (the other scores cannot matter to them)
    r1 = _nms(np.where(valid, S, 0), vc_cells(vc), ti)
    for it in nz_hi:
        out[lanes(*it)] |= r1[lanes(*it)] & valid[lanes(*it)]
    hit = {int(c) for c in vc[out]}
    F = set(range(CG)) - hit
    if not F:
        return out
    touches = lambda it: bool(set(vc[lanes(*it)].tolist()) & F)   # noqa: E731
    for it in deferred:
        if touches(it):
            S[lanes(*it)] = np.where(s[lanes(*it)] > mt, s[lanes(*it)], 0)
            if S[lanes(*it)].any():
                nz_lo.append(it)
    r2 = _nms(np.where(valid, S, 0), vc_cells(vc), 0)
    inF = np.isin(vc, sorted(F))
    for it in nz_hi + nz_lo:
        if touches(it):
            out[lanes(*it)] |= r2[lanes(*it)] & inF[lanes(*it)]
    return out


def vc_cells(vc):
    """Cell index per column for _nms, with the padding columns (-1) as cells of their own so they neighbour nothing."""
    row = vc[0].copy()
    pad = row < 0
    row[pad] = CG + np.cumsum(pad)[pad]
    return row


def _tile(rng, kind):
    """A random tile: CG cells of wc columns after xoff padding columns (items straddle cell borders when wc % 4 != 0), its scores and
    compass bounds (>= the scores, often equal)."""
    wc, h, xoff = int(rng.integers(3, 10)), int(rng.integers(3, 9)), int(rng.integers(0, 4))
    w = 4 * -(-(xoff + CG * wc) // 4)
    cells_row = np.full(w, -1)
    cells_row[xoff:xoff + CG * wc] = np.repeat(np.arange(CG), wc)
    valid = np.broadcast_to(cells_row >= 0, (h, w)).copy()
    if kind == "plateau":          # few distinct values: ties above and below iniTh
        s = rng.choice([0, 0, 0, 3, 8, 12, 21, 21, 40, 255], (h, w))
    elif kind == "sparse":         # mostly weak corners: cells fall back
        s = np.where(rng.random((h, w)) < 0.15, rng.integers(0, 25, (h, w)), 0)
    else:
        s = rng.integers(0, 256, (h, w)) * (rng.random((h, w)) < 0.5)
    bound = np.minimum(s + rng.integers(0, 30, (h, w)) * (rng.random((h, w)) < 0.5), 255)
    bound = np.where(rng.random((h, w)) < 0.1, np.maximum(bound, rng.integers(0, 60, (h, w))), bound)   # bounds above zero scores
    return s.astype(np.int32), bound.astype(np.int32), np.broadcast_to(np.where(cells_row >= 0, cells_row, 0), (h, w)), valid


@pytest.mark.parametrize("ini,mn", PAIRS)
@pytest.mark.parametrize("kind", ["plateau", "sparse", "dense"])
def test_two_rounds_select_what_one_nms_and_the_filter_select(ini, mn, kind):
    rng = np.random.default_rng(1000 * (ini % 997) + 10 * (mn % 97) + len(kind))
    for _ in range(25):
        s, bound, cells, valid = _tile(rng, kind)
        cols = np.flatnonzero(valid[0])
        sd, cd = s[:, cols], cells[:, cols][0]
        want = _one_round(sd, cd, ini, mn)
        # an iniThFAST below minThFAST acts as minThFAST (every survivor at minThFAST is kept)
        assert np.array_equal(want, _reference(sd, cd, max(ini, mn), mn))
        got = _two_rounds(s, bound, cells, valid, ini, mn)
        assert np.array_equal(got[:, cols], want) and not got[:, ~valid[0]].any()

#!/usr/bin/env python
"""How much of k_fast's phase-B work (3x3 NMS) the nz list removes, at bench.py's headline shape; CPU only (the oracle, numpy, no GPU).

The bench's fisheye frames go through the oracle's warp and pyramid (oracle.ORBextractor.level_image). Per level, FAST-9 arc scores are
computed in numpy from the definition, without NMS, and the detection area is cut into k_fast's tiles and 4-pixel work items (the geometry
of fast_tile_x in frontend.cu). Per level, summed over --frames frames, one JSON line on stdout:

  live_items       items with a pixel of the detection area whose 7x7 window is not all one value: what phase A scores, and phase B scored
                   before the nz list (within 1 % of the real live lists, DESIGN.md section 4)
  nz_items         live items with a pixel of the detection area whose score is above minThFAST: what phase B scores now
  nz_fraction      nz_items / live_items
  compass_items    live items with a pixel of the detection area that the compass bound cannot prove corner-free (compass_x2 in
                   frontend.cu): what phase A0 passes on to phase A (it also tests the item's pixels outside the detection area, so
                   the kernel's pass lists can be slightly longer)
  compass_fraction compass_items / live_items
  zero_warp_groups share of 32-item groups of a tile's live items (one warp's items in one pass) that hold no nz item: what phase B's
                   early return for an all-zero item already skipped as a whole warp

With --ini the line also holds, per level and in total, what k_fast's two rounds see (iniThFAST, the fallback to minThFAST):

  compass_ini_items  live items the compass bound cannot prove <= iniThFAST: phase A's pass list (the rest of compass_items is deferred)
  nz_ini_items       live items with a pixel of the detection area whose score is above iniThFAST: round 1's work list (nzHi)
  cells              cells with a live pixel; fallback_cells of them have no keypoint at iniThFAST (per-cell NMS, the reference's rule)
  fallback_live_px   live pixels (detection area, 7x7 window not all one value) in fallback cells, and live_px in all cells
  fallback_compass_px  of those, the pixels the compass bound cannot prove <= minThFAST
  tiles, round2_tiles  tiles with a live pixel, and those of them with a cell without a keypoint at iniThFAST, live or not (the tiles
                     that run round 2)

  python tools/fast_nz_items.py [--frames 2] [--ini]
"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

CG = 4                      # k_fast cells per tile, as in frontend.cu
RING = [(0, -3), (1, -3), (2, -2), (3, -1), (3, 0), (3, 1), (2, 2), (1, 3), (0, 3), (-1, 3), (-2, 2), (-3, 1), (-3, 0), (-3, -1), (-2, -2), (-1, -3)]


def fast_scores(img):
    """Arc score s of every pixel at least 3 from the border (0 elsewhere): the largest t such that 9 contiguous ring pixels are all
    brighter than centre + t or all darker than centre - t, at least 0. corner(thr) <=> s > thr."""
    h, w = img.shape
    c = img[3:h - 3, 3:w - 3].astype(np.int16)
    d = np.stack([c - img[3 + dy:h - 3 + dy, 3 + dx:w - 3 + dx].astype(np.int16) for dx, dy in RING])   # centre minus ring
    d = np.concatenate([d, d[:8]])
    s = np.zeros(c.shape, np.int16)
    for k in range(16):
        lo, hi = d[k:k + 9].min(0), d[k:k + 9].max(0)
        s = np.maximum(s, np.maximum(lo, -hi))
    out = np.zeros((h, w), np.int16)
    out[3:h - 3, 3:w - 3] = s
    return out


def compass_pass(img, minth):
    """True where the compass bound of the arc score exceeds mt = minth clamped to 1..255: min(max(R0, R8), max(R4, R12)) > c + mt or
    max(min(R0, R8), min(R4, R12)) < c - mt (0 within 3 of the border)."""
    h, w = img.shape
    mt = min(max(minth, 1), 255)
    c = img[3:h - 3, 3:w - 3].astype(np.int16)
    r0, r4, r8, r12 = (img[3 + dy:h - 3 + dy, 3 + dx:w - 3 + dx].astype(np.int16) for dx, dy in (RING[0], RING[4], RING[8], RING[12]))
    ua = np.minimum(np.maximum(r0, r8), np.maximum(r4, r12))
    lb = np.maximum(np.minimum(r0, r8), np.minimum(r4, r12))
    out = np.zeros((h, w), bool)
    out[3:h - 3, 3:w - 3] = (ua - c > mt) | (c - lb > mt)
    return out


def single_valued(img):
    """True where the 7x7 window centred on the pixel holds one value."""
    from scipy.ndimage import maximum_filter, minimum_filter
    return maximum_filter(img, size=7, mode="nearest") == minimum_filter(img, size=7, mode="nearest")


def tile_items(score, flat, cpass, minth, minB, maxBX, maxBY, wCell, hCell, nColsEff, nRowsEff):
    """Per k_fast tile, its items in list order (detection row, then item): (live, nz, compass) boolean vectors."""
    for cy in range(nRowsEff):
        iniY = minB + cy * hCell
        ny = min(iniY + hCell + 6, maxBY) - iniY - 6
        for cx in range(-(-nColsEff // CG)):
            ncell = min(CG, nColsEff - cx * CG)
            tx0 = minB + cx * CG * wCell
            tx1 = min(tx0 + ncell * wCell + 6, maxBX)
            nx = tx1 - tx0 - 6
            if nx <= 0 or ny <= 0:
                continue
            a0 = tx0 & ~15
            xoff = tx0 - a0 + 3
            w0, w1 = xoff >> 2, (xoff + nx + 3) >> 2
            cols = np.arange(4 * w0, 4 * w1) + a0                    # level x of the items' pixels
            valid = (cols >= tx0 + 3) & (cols < tx0 + 3 + nx)
            ys = iniY + 3 + np.arange(ny)
            cc = np.clip(cols, 0, score.shape[1] - 1)
            lv = ~flat[ys][:, cc] & valid
            nz = (score[ys][:, cc] > minth) & valid
            cp = cpass[ys][:, cc] & valid
            yield tuple(m.reshape(ny, -1, 4).any(2).ravel() for m in (lv, nz, cp))


def cell_keypoints(score, thr, y0, y1, x0, x1):
    """True if the cell's detection area [y0, y1) x [x0, x1) has a keypoint of cv::FAST at thr: a score above thr that is above every
    neighbour's in the cell (scores at or below thr count as 0)"""
    s = np.pad(np.where(score[y0:y1, x0:x1] > thr, score[y0:y1, x0:x1], 0), 1)
    h, w = y1 - y0, x1 - x0
    nb = np.max([s[1 + dy:h + 1 + dy, 1 + dx:w + 1 + dx] for dy in (-1, 0, 1) for dx in (-1, 0, 1) if dy or dx], 0)
    return bool(((s[1:-1, 1:-1] > nb) & (s[1:-1, 1:-1] > 0)).any())


def fallback_stats(score, flat, cpass_min, ini, minB, maxBX, maxBY, wCell, hCell, nColsEff, nRowsEff):
    """Per level: cells with a live pixel, those without a keypoint at ini, live and compass-passing pixels in them, and tiles with a live
    pixel / with a live pixel and a cell without a keypoint at ini."""
    out = dict(cells=0, fallback_cells=0, live_px=0, fallback_live_px=0, fallback_compass_px=0, tiles=0, round2_tiles=0)
    live = ~flat
    for cy in range(nRowsEff):
        iniY = minB + cy * hCell
        y1 = min(iniY + hCell + 6, maxBY) - 3
        if y1 <= iniY + 3:
            continue
        for tx in range(-(-nColsEff // CG)):
            tile_live, tile_fb = False, False
            for cx in range(tx * CG, min(nColsEff, tx * CG + CG)):
                iniX = minB + cx * wCell
                x1 = min(iniX + wCell + 6, maxBX) - 3
                if x1 <= iniX + 3:
                    continue
                ys, xs = slice(iniY + 3, y1), slice(iniX + 3, x1)
                lv = int(live[ys, xs].sum())
                fb = not cell_keypoints(score, ini, iniY + 3, y1, iniX + 3, x1)
                tile_fb |= fb
                if lv == 0:
                    continue
                out["cells"] += 1
                out["live_px"] += lv
                tile_live = True
                if fb:
                    out["fallback_cells"] += 1
                    out["fallback_live_px"] += lv
                    out["fallback_compass_px"] += int((cpass_min[ys, xs] & live[ys, xs]).sum())
            out["tiles"] += tile_live
            out["round2_tiles"] += tile_live and tile_fb
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=2)
    ap.add_argument("--ini", action="store_true", help="also count what the two rounds at iniThFAST see")
    args = ap.parse_args()
    import oracle as orc
    from cubemapslam_b200 import _capi, config, synth
    import bench
    from fast_live_roofline import _grid
    cfg = config.front_1024()
    o = _capi.orb_params(cfg)
    cp = orc.cam_params(cfg)
    m1, m2 = orc.build_maps(cp)
    mask = bench.load_mask()
    INI = ("compass_ini_items", "nz_ini_items", "cells", "fallback_cells", "live_px", "fallback_live_px", "fallback_compass_px", "tiles",
           "round2_tiles")
    levels = [dict(live_items=0, nz_items=0, compass_items=0, groups=0, zero_groups=0, **{k: 0 for k in INI}) for _ in range(o.nlevels)]
    for f in range(args.frames):
        ex = orc.ORBextractor(o.nfeatures, o.scale_factor, o.nlevels, o.ini_th_fast, o.min_th_fast, cp.faceW, cp.faceH)
        ex(orc.warp(cp, synth.fisheye_frame(cfg, f), m1, m2), mask)
        for l in range(o.nlevels):
            img = ex.level_image(l)
            h, w = img.shape
            score, flat, cpass = fast_scores(img), single_valued(img), compass_pass(img, o.min_th_fast)
            L = levels[l]
            L["side"] = w
            for live, nz, comp in tile_items(score, flat, cpass, o.min_th_fast, *_grid(w, h)):
                nzl = nz[live]                                       # the live list, in k_fast's order
                L["live_items"] += int(live.sum())
                L["nz_items"] += int(nzl.sum())
                L["compass_items"] += int(comp[live].sum())
                for g in range(0, len(nzl), 32):
                    L["groups"] += 1
                    L["zero_groups"] += int(not nzl[g:g + 32].any())
            if args.ini:
                ci = compass_pass(img, o.ini_th_fast)
                for live, nz, comp in tile_items(score, flat, ci, o.ini_th_fast, *_grid(w, h)):
                    L["nz_ini_items"] += int(nz[live].sum())
                    L["compass_ini_items"] += int(comp[live].sum())
                for k, v in fallback_stats(score, flat, cpass, o.ini_th_fast, *_grid(w, h)).items():
                    L[k] += v
    out = []
    for L in levels:
        out.append({"side": L["side"], "live_items": L["live_items"] // args.frames, "nz_items": L["nz_items"] // args.frames,
                    "nz_fraction": round(L["nz_items"] / max(L["live_items"], 1), 4),
                    "compass_items": L["compass_items"] // args.frames,
                    "compass_fraction": round(L["compass_items"] / max(L["live_items"], 1), 4),
                    "zero_warp_groups": round(L["zero_groups"] / max(L["groups"], 1), 4)})
        if args.ini:
            out[-1].update({k: L[k] // args.frames for k in INI})
    tl, tn, tc = (sum(L[k] for L in levels) for k in ("live_items", "nz_items", "compass_items"))
    total = {"live_items": tl // args.frames, "nz_items": tn // args.frames, "nz_fraction": round(tn / max(tl, 1), 4),
             "compass_items": tc // args.frames, "compass_fraction": round(tc / max(tl, 1), 4)}
    if args.ini:
        T = {k: sum(L[k] for L in levels) for k in INI}
        total.update({k: T[k] // args.frames for k in INI})
        total.update({"compass_ini_fraction": round(T["compass_ini_items"] / max(tl, 1), 4), "nz_ini_fraction": round(T["nz_ini_items"] / max(tl, 1), 4),
                      "fallback_cell_fraction": round(T["fallback_cells"] / max(T["cells"], 1), 4),
                      "fallback_live_px_fraction": round(T["fallback_live_px"] / max(T["live_px"], 1), 4),
                      "fallback_compass_px_fraction": round(T["fallback_compass_px"] / max(T["live_px"], 1), 4),
                      "round2_tile_fraction": round(T["round2_tiles"] / max(T["tiles"], 1), 4)})
    print(json.dumps({"frames": args.frames, "min_th_fast": o.min_th_fast, "ini_th_fast": o.ini_th_fast, "per_frame": out, "total": total}))


if __name__ == "__main__":
    main()

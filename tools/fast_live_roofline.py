#!/usr/bin/env python
"""k_fast's work against its instruction bound, at bench.py's headline shape (front camera, 1280x1024 frames, 650-px faces, batches of 128
on one stream). One JSON line on stdout:

  levels            per pyramid level, pixels per frame:
                      detection_px    the FAST detection area of the cell grid, what bench.py's k_fast figures count
                      corner_skip_px  detection pixels of CTA tiles that are not entirely in the black canvas corners (the tiles scored before
                                      the live-item lists)
                      live_window_px  detection pixels whose 7x7 window is not all one static class (frontend.cu, build_static_classes)
                      live_item_px    detection pixels of the live work items (4-pixel words holding a live_window pixel): what k_fast scores
  k_fast            ms_per_batch from the front end's own CUDA events (cslam_frontend_set_timing) over --batches batches after a warm-up;
                    frac_of_minmax3_peak_live: 40 VIMNMX3.U16x2 per scored pixel (80 per pixel pair, DESIGN.md section 4) over the live item
                    pixels, against cslam_ubench_minmax3 measured in the same run; frac_of_minmax3_peak_bench: the same over detection_px
  card              name, power limit and maximum SM clock of the GPU the times come from

  python tools/fast_live_roofline.py [--batches 16]
"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

CG, EDGE = 4, 19            # k_fast cells per CTA and the ORB edge threshold, as in frontend.cu
K_LIVE, K_Z, K_C = 0, 1, 2


def _resize_tables(sn, dn):
    """build_resize_tables (frontend.cu): source index and the two 11-bit weights per destination index."""
    f = ((np.arange(dn) + 0.5) * (sn / dn) - 0.5).astype(np.float32)
    s = np.floor(f).astype(np.int64)
    f = (f - s.astype(np.float32)).astype(np.float32)
    f[s < 0] = 0; s[s < 0] = 0
    hi = s >= sn - 1
    f[hi] = 0; s[hi] = sn - 1
    a0 = np.rint((np.float32(1) - f) * np.float32(2048)).astype(np.int64); a1 = np.rint(f * np.float32(2048)).astype(np.int64)
    return s, a0 + a1


def _grid(w, h):
    """LevelGeom's FAST cell grid: (minB, maxBX, maxBY, wCell, hCell, nColsEff, nRowsEff)."""
    minB, maxBX, maxBY = EDGE - 3, w - EDGE + 3, h - EDGE + 3
    width, height = np.float32(maxBX - minB), np.float32(maxBY - minB)
    nCols, nRows = int(width / np.float32(30)), int(height / np.float32(30))
    wCell, hCell = int(np.ceil(width / np.float32(nCols))), int(np.ceil(height / np.float32(nRows)))
    nColsEff = max([j + 1 for j in range(nCols) if not minB + j * wCell >= maxBX - 6] + [0])
    nRowsEff = max([i + 1 for i in range(nRows) if not minB + i * hCell >= maxBY - 3] + [0])
    return minB, maxBX, maxBY, wCell, hCell, nColsEff, nRowsEff


def _uniform(K):
    """U[y, x] = True where the 7x7 window centred on (x, y) is all Z or all C."""
    h, w = K.shape
    U = np.zeros((h, w), bool)
    for k in (K_Z, K_C):
        S = np.zeros((h + 1, w + 1), np.int64)
        S[1:, 1:] = (K == k).cumsum(0).cumsum(1)
        U[3:h - 3, 3:w - 3] |= (S[7:, 7:] - S[:-7, 7:] - S[7:, :-7] + S[:-7, :-7]) == 49
    return U


def live_counts(cfg, nlevels=8, scale=1.2):
    """Per level, the pixel counts described in the module doc, from the front camera's geometry alone (no GPU)."""
    import oracle as orc
    cp = orc.cam_params(cfg)
    m1, m2 = orc.build_maps(cp)
    W = cp.faceW
    CW = 3 * W
    face = np.zeros((CW, CW), bool)
    face[W:2 * W, :] = True; face[:, W:2 * W] = True
    origin = (np.rint(m1 * np.float32(32)) == 0) & (np.rint(m2 * np.float32(32)) == 0)
    K = np.where(face, np.where(origin, K_C, K_LIVE), K_Z).astype(np.uint8)
    out = []
    s = np.float32(1.0)
    for l in range(nlevels):
        side = int(np.rint(np.float32(CW) * (np.float32(1.0) / s)))
        s = np.float32(s * np.float32(scale))
        if l > 0:
            sh, sw = K.shape
            yo, ys = _resize_tables(sh, side); xo, xs = _resize_tables(sw, side)
            y1, x1 = np.minimum(yo + 1, sh - 1), np.minimum(xo + 1, sw - 1)
            k00, k01, k10, k11 = K[yo][:, xo], K[yo][:, x1], K[y1][:, xo], K[y1][:, x1]
            same = (k00 == k01) & (k00 == k10) & (k00 == k11)
            unit = (ys[:, None] == 2048) & (xs[None, :] == 2048)
            K = np.where(same & ((k00 == K_Z) | ((k00 == K_C) & unit)), k00, K_LIVE).astype(np.uint8)
        U = _uniform(K)
        minB, maxBX, maxBY, wCell, hCell, nColsEff, nRowsEff = _grid(side, side)
        det = corner = live_win = live_item = 0
        for cy in range(nRowsEff):
            for cxg in range(-(-nColsEff // CG)):
                iniY = minB + cy * hCell; maxY = min(iniY + hCell + 6, maxBY)
                ncell = min(CG, nColsEff - cxg * CG)
                tx0 = minB + cxg * CG * wCell; tx1 = min(tx0 + ncell * wCell + 6, maxBX)
                nx, ny = tx1 - tx0 - 6, maxY - iniY - 6
                if nx <= 0 or ny <= 0:
                    continue
                det += nx * ny
                if (K[iniY:maxY, tx0:tx1] != K_Z).any():
                    corner += nx * ny
                lv = ~U[iniY + 3:iniY + 3 + ny, tx0 + 3:tx0 + 3 + nx]
                live_win += int(lv.sum())
                pad = (tx0 - (tx0 & ~3) + 3) & 3          # detection x = 0 sits at this lane of its 4-pixel word
                n4 = -(-(pad + nx) // 4) * 4
                L = np.zeros((ny, n4), bool); V = np.zeros((ny, n4), bool)
                L[:, pad:pad + nx] = lv; V[:, pad:pad + nx] = True
                item = L.reshape(ny, -1, 4).any(2)
                live_item += int((V.reshape(ny, -1, 4).sum(2) * item).sum())
        out.append({"side": side, "detection_px": det, "corner_skip_px": corner, "live_window_px": live_win, "live_item_px": live_item})
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", type=int, default=16)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("fast_live_roofline.py: no CUDA device")
    import bench
    from match_roofline import card
    from cubemapslam_b200 import config
    from cubemapslam_b200.frontend import FrontEnd
    from cubemapslam_b200.matcher import ORBMatcher
    dev = torch.device("cuda", 0)
    cfg = config.front_1024()
    B = 128
    levels = live_counts(cfg)
    tot = {k: sum(lv[k] for lv in levels) for k in ("detection_px", "corner_skip_px", "live_window_px", "live_item_px")}
    fish, _ = bench.make_frames_device(torch, cfg, B, dev)
    fe = FrontEnd(cfg, bench.load_mask(), max_batch=B)
    cap = fe.kp_cap
    kps = torch.empty((B, cap, 28), dtype=torch.uint8, device=dev); desc = torch.empty((B, cap, 32), dtype=torch.uint8, device=dev)
    n = torch.zeros(B, dtype=torch.int32, device=dev)
    torch.cuda.synchronize()
    run = lambda: fe.run_dev(fish.data_ptr(), B, kps.data_ptr(), desc.data_ptr(), n.data_ptr())
    for _ in range(3):
        run()
    fe.sync()
    fe.set_timing(True)
    for _ in range(args.batches):
        run(); fe.sync()
    tm = fe.timing(); fe.set_timing(False)
    fe.close()
    mt = ORBMatcher(0.6, True, max_pairs=1, max_features=256)
    peak = mt.ubench_minmax3()
    mt.close()
    sec = tm["k_fast"][0] / args.batches / 1e3
    fast = {"ms_per_batch": round(sec * 1e3, 4), "measured_peak_minmax3_per_s": round(peak, 1),
            "frac_of_minmax3_peak_live": round(40.0 * tot["live_item_px"] * B / sec / peak, 4),
            "frac_of_minmax3_peak_bench": round(40.0 * tot["detection_px"] * B / sec / peak, 4)}
    print(json.dumps({"card": card(), "batch": B, "levels": levels, "total": tot, "k_fast": fast,
                      "all_kernels_ms_per_batch": {k: round(v[0] / args.batches, 4) for k, v in tm.items()}}))


if __name__ == "__main__":
    main()

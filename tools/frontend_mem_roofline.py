#!/usr/bin/env python
"""Memory roofline of the front end's byte kernels, k_warp and k_pyramid, at bench.py's headline shape (front camera, 1280x1024 frames,
650-px faces, batches of 128 on one stream). One JSON line on stdout:

  run                 the one timed run: per kernel ms_per_batch, the time from the front end's own CUDA events between launches
                      (cslam_frontend_set_timing) over --batches batches after a warm-up, and the frac_* below
  bytes_live          bytes the algorithm needs per frame: k_warp reads every fisheye pixel some face pixel taps once and writes the five
                      faces; k_pyramid reads and writes only the pixels outside the provably black cubemap corners (Z_l, frontend.cu)
  bytes_full          bench.py's accounting: the whole fisheye frame + 5 faces, and every level of the pyramid in full
  frac_*              those bytes per second over 3.35 TB/s (H100 SXM HBM3 data sheet)

  python tools/frontend_mem_roofline.py [--batches 16]
"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

HBM = 3.35e12


def resize_ofs(sn, dn):
    """build_resize_tables' source index per destination index (frontend.cu)."""
    scale = sn / dn
    f = ((np.arange(dn) + 0.5) * scale - 0.5).astype(np.float32)
    s = np.floor(f).astype(np.int64)
    return np.clip(s, 0, sn - 1)


def live_bytes(cfg, sizes):
    """(warp, pyramid) bytes per frame the algorithm needs on the live region (see module doc)."""
    import oracle as orc
    cp = orc.cam_params(cfg)
    m1, m2 = orc.build_maps(cp)
    W = cp.faceW
    face = np.zeros((3 * W, 3 * W), bool)
    face[W:2 * W, :] = True; face[:, W:2 * W] = True
    sx = np.rint(m1 * 32).astype(np.int64)[face]; sy = np.rint(m2 * 32).astype(np.int64)[face]
    taps = np.zeros((cp.Ih + 2, cp.Iw + 2), bool)
    ix, iy = sx >> 5, sy >> 5
    for dy in (0, 1):
        for dx in (0, 1):
            taps[iy + dy, ix + dx] = True
    warp = int(taps[:cp.Ih, :cp.Iw].sum()) + 5 * W * W
    Z = ~face
    pyr = 0
    for l in range(1, len(sizes)):
        sh, sw = Z.shape
        dn = sizes[l]
        yo, xo = resize_ofs(sh, dn), resize_ofs(sw, dn)
        y1, x1 = np.minimum(yo + 1, sh - 1), np.minimum(xo + 1, sw - 1)
        Zn = Z[yo][:, xo] & Z[yo][:, x1] & Z[y1][:, xo] & Z[y1][:, x1]
        pyr += int((~Z).sum()) + int((~Zn).sum())
        Z = Zn
    return warp, pyr


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", type=int, default=16)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("frontend_mem_roofline.py: no CUDA device")
    import bench
    from match_roofline import card
    from cubemapslam_b200 import config
    from cubemapslam_b200.frontend import FrontEnd
    dev = torch.device("cuda", 0)
    cfg = config.front_1024()
    B = 128
    gb = bench.geometry_bytes(cfg)
    side = [int(round(s ** 0.5)) for s in gb["levels_px"]]
    warp_live, pyr_live = live_bytes(cfg, side)
    out = {"card": card(), "batch": B, "bytes_full": {"k_warp": gb["k_warp"], "k_pyramid": gb["k_pyramid"]},
           "bytes_live": {"k_warp": warp_live, "k_pyramid": pyr_live}}
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
    r = {}
    for k in ("k_warp", "k_pyramid"):
        sec = tm[k][0] / args.batches / 1e3
        r[k] = {"ms_per_batch": round(sec * 1e3, 4),
                "frac_of_hbm_live": round(out["bytes_live"][k] * B / sec / HBM, 4),
                "frac_of_hbm_full": round(out["bytes_full"][k] * B / sec / HBM, 4)}
    r["all_kernels_ms_per_batch"] = {k: round(v[0] / args.batches, 4) for k, v in tm.items()}
    out["run"] = r
    fe.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()

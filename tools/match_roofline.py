#!/usr/bin/env python
"""Roofline of the all-pairs matcher (k_match_bruteforce) on this GPU, one JSON line on stdout:

  peaks     register-only tensor-core chains (cslam_ubench_bmma): BMMA m16n8k256 AND.POPC, the unit the kernel runs on, and m16n8k32 s8 IMMA
            on +-1 int8 expansions for comparison, both in 256-bit products (= Hamming distances) per second; the POPC issue rate
            (cslam_ubench_popc, 8 POPC per distance) of the previous kernel for reference
  headline  bench.py's shape: 128 consecutive-frame pairs of the front end's key points (~2 100 per frame, kp_stride 3024) through
            cslam_match_frames_dev
  config3   2000 x 2000 descriptors, 4096 pairs through cslam_match_bruteforce_dev (bench.py's extra.match.bruteforce)
Achieved = sum over pairs of nA * nB distances / kernel time (CUDA events over --reps launches after a warm-up).

  python tools/match_roofline.py [--reps 20]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip()
        name, power, clk = [s.strip() for s in out.split(",")]
        return {"name": name, "power_limit": power, "sm_clock_max": clk}
    except Exception as e:   # the timing itself does not depend on it
        return {"error": str(e)}


def time_launches(torch, stream, fn, reps):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    e0 = torch.cuda.Event(enable_timing=True); e1 = torch.cuda.Event(enable_timing=True)
    e0.record(stream)
    for _ in range(reps):
        fn()
    e1.record(stream)
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps / 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("match_roofline.py: no CUDA device")
    import bench
    from cubemapslam_b200 import config, synth
    from cubemapslam_b200.frontend import FrontEnd
    from cubemapslam_b200.matcher import ORBMatcher
    dev = torch.device("cuda", 0)
    out = {"card": card()}

    # headline shape: one front-end batch of 129 frames -> 128 pairs
    cfg = config.front_1024()
    B = 129
    fe = FrontEnd(cfg, bench.load_mask(), max_batch=B)
    cap = fe.kp_cap
    fish, _ = bench.make_frames_device(torch, cfg, B, dev)
    kps = torch.empty((B, cap, 28), dtype=torch.uint8, device=dev); desc = torch.empty((B, cap, 32), dtype=torch.uint8, device=dev)
    n = torch.zeros(B, dtype=torch.int32, device=dev)
    fe.run_dev(fish.data_ptr(), B, kps.data_ptr(), desc.data_ptr(), n.data_ptr()); fe.sync()
    mt = ORBMatcher(0.6, True, max_pairs=B, max_features=cap)
    match = torch.empty((B, cap), dtype=torch.int32, device=dev); nm = torch.empty(B, dtype=torch.int32, device=dev)
    ms = torch.cuda.ExternalStream(mt.stream, device=dev)
    sec = time_launches(torch, ms, lambda: mt.match_frames_dev(kps.data_ptr(), desc.data_ptr(), n.data_ptr(), cap, B, match.data_ptr(), nm.data_ptr()), args.reps)
    hn = n.cpu().numpy().astype(np.int64)
    dist = float((hn[:-1] * hn[1:]).sum())
    out["headline"] = {"pairs": B - 1, "mean_keypoints": round(float(hn.mean()), 1), "distances": dist, "ms_per_launch": round(sec * 1e3, 4),
                       "distances_per_s": dist / sec}
    bmma, imma = mt.ubench_bmma()
    popc = mt.ubench_popc()
    fe.close(); mt.close()
    del fish, kps, desc, match
    torch.cuda.empty_cache()

    # config 3: 2000 x 2000, 4096 pairs (tiles of 16 generated pairs, B rolled per tile as in bench_extra)
    P, nd = 4096, 2000
    base = [synth.descriptor_pair(p, n=nd) for p in range(16)]
    reps = P // 16
    dA = torch.from_numpy(np.stack([b[0] for b in base])).to(dev).repeat(reps, 1, 1).contiguous()
    daA = torch.from_numpy(np.stack([b[1] for b in base])).to(dev).repeat(reps, 1).contiguous()
    Bd = torch.from_numpy(np.stack([b[2] for b in base])).to(dev); aB = torch.from_numpy(np.stack([b[3] for b in base])).to(dev)
    dB = torch.cat([torch.roll(Bd, shifts=r, dims=1) for r in range(reps)]).contiguous()
    daB = torch.cat([torch.roll(aB, shifts=r, dims=1) for r in range(reps)]).contiguous()
    m3 = ORBMatcher(0.6, True, max_pairs=P, max_features=2048)
    match = torch.empty((P, nd), dtype=torch.int32, device=dev); nm = torch.empty(P, dtype=torch.int32, device=dev)
    s3 = torch.cuda.ExternalStream(m3.stream, device=dev)
    sec = time_launches(torch, s3, lambda: m3.match_bruteforce_dev(dA.data_ptr(), daA.data_ptr(), nd, dB.data_ptr(), daB.data_ptr(), nd, P, match.data_ptr(),
                                                                    nm.data_ptr()), max(2, args.reps // 4))
    dist = float(P) * nd * nd
    out["config3"] = {"pairs": P, "distances": dist, "ms_per_launch": round(sec * 1e3, 3), "pairs_per_s": round(P / sec, 1), "distances_per_s": dist / sec}
    m3.close()

    out["peaks"] = {"bmma_products_per_s": bmma, "imma_s8_products_per_s": imma, "popc32_per_s": popc, "popc_distances_per_s": popc / 8.0,
                    "bmma_over_popc": round(bmma / (popc / 8.0), 2), "imma_over_popc": round(imma / (popc / 8.0), 2),
                    "source": "cslam_ubench_bmma / cslam_ubench_popc on this GPU (register-only chains)"}
    for k in ("headline", "config3"):
        out[k]["frac_of_bmma_peak"] = round(out[k]["distances_per_s"] / bmma, 4)
        out[k]["vs_popc_peak"] = round(out[k]["distances_per_s"] / (popc / 8.0), 3)
    print(json.dumps(out))


if __name__ == "__main__":
    main()

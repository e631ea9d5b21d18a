"""Front-end throughput of the three ways to feed it, in one process (BASELINE config 2: front_cam_params with a 1280x1024 sensor, 650-px
faces, nFeatures 3000, bench.py's synthetic frames):

  run_dev      frames and outputs on the device, cslam_frontend_run_dev per batch: the ceiling
  run          the synchronous host entry, cslam_frontend_run per batch
  submit_wait  the asynchronous host entry: submit batch i+1, then wait for batch i

Outputs are page-locked in every mode; `run` and `submit_wait` are run with page-locked and with pageable input. Modes alternate, each timed
--runs times. Prints one JSON line: frames/s of every mode and run, the card (name, power limit, max SM clock), page-locked copy rates measured
like tools/pcie_bw.py, and whether `run` and `submit_wait` wrote identical bytes for every frame.

  python tools/frontend_async.py [--frames 1024] [--batch 128] [--runs 3] [--passes 5]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402  (the frame generator of the benchmark)
from cubemapslam_b200 import config  # noqa: E402
from cubemapslam_b200._capi import KP_DTYPE  # noqa: E402


def gpu_info():
    q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader,nounits"],
                       capture_output=True, text=True).stdout.strip().split(",")
    return {"name": q[0].strip(), "power_limit_w": float(q[1]), "sm_max_mhz": float(q[2])} if len(q) == 3 else {"nvidia-smi": "unavailable"}


def copy_rates(torch):
    """Page-locked H2D and D2H GB/s of 168 MiB copies, 10 each (tools/pcie_bw.py)."""
    n = 168 * 1024 * 1024
    h = torch.empty(n, dtype=torch.uint8).pin_memory(); d = torch.empty(n, dtype=torch.uint8, device="cuda")
    out = {}
    for name, fn in (("h2d_gbs", lambda: d.copy_(h, non_blocking=True)), ("d2h_gbs", lambda: h.copy_(d, non_blocking=True))):
        fn(); torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(10):
            fn()
        torch.cuda.synchronize()
        out[name] = round(10 * n / (time.perf_counter() - t0) / 1e9, 2)
    return out


def pinned(torch, shape, dtype):
    dtype = np.dtype(dtype)
    return torch.empty(int(np.prod(shape)) * dtype.itemsize, dtype=torch.uint8, pin_memory=True).numpy().view(dtype).reshape(shape)


def same_rows(a, b):
    """Two (kps, desc, n) output sets hold the same counts and the same bytes in every frame's first n rows."""
    (ka, da, na), (kb, db, nb) = a, b
    if not np.array_equal(na, nb):
        return False
    valid = np.arange(ka.shape[1])[None, :] < na[:, None]
    return bool(np.array_equal(ka.view(np.uint8).reshape(ka.shape + (-1,))[valid], kb.view(np.uint8).reshape(kb.shape + (-1,))[valid])
                and np.array_equal(da[valid], db[valid]))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=1024)
    ap.add_argument("--batch", type=int, default=128)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--passes", type=int, default=5, help="passes over all frames per timed run")
    args = ap.parse_args()
    import torch
    from cubemapslam_b200.frontend import FrontEnd
    if not torch.cuda.is_available():
        raise SystemExit("frontend_async.py: no CUDA device")
    cfg = config.front_1024()
    assert int(cfg["ORBextractor.nFeatures"]) == 3000 and int(cfg["CubeFace.w"]) == 650
    N, B = args.frames, args.batch
    fe = FrontEnd(cfg, bench.load_mask(), max_batch=B)
    kc = fe.kp_cap
    frames_dev, _ = bench.make_frames_device(torch, cfg, N, "cuda")
    in_pin = pinned(torch, tuple(frames_dev.shape), np.uint8)
    in_pin[:] = frames_dev.cpu().numpy()
    in_page = np.array(in_pin)
    kps_dev = torch.empty((N, kc * KP_DTYPE.itemsize), dtype=torch.uint8, device="cuda")
    desc_dev = torch.empty((N, kc, 32), dtype=torch.uint8, device="cuda"); n_dev = torch.empty(N, dtype=torch.int32, device="cuda")
    outs = {k: (pinned(torch, (N, kc), KP_DTYPE), pinned(torch, (N, kc, 32), np.uint8), pinned(torch, (N,), np.int32)) for k in ("run", "submit_wait")}
    fsz = frames_dev.shape[1] * frames_dev.shape[2]
    batches = [(c, min(B, N - c)) for c in range(0, N, B)]

    def run_dev():
        for c, b in batches:
            fe.run_dev(frames_dev.data_ptr() + c * fsz, b, kps_dev.data_ptr() + c * kc * KP_DTYPE.itemsize, desc_dev.data_ptr() + c * kc * 32,
                       n_dev.data_ptr() + c * 4)
        fe.sync()

    def run(src):
        k, d, n = outs["run"]
        for c, b in batches:
            fe.run_raw(src[c:c + b], k[c:c + b], d[c:c + b], n[c:c + b])

    def submit_wait(src):
        k, d, n = outs["submit_wait"]
        prev = None
        for c, b in batches:
            t = fe.submit_raw(src[c:c + b], k[c:c + b], d[c:c + b], n[c:c + b])
            if prev is not None:
                fe.wait(prev)
            prev = t
        fe.wait(prev)

    modes = {"run_dev": run_dev, "run": lambda: run(in_pin), "submit_wait": lambda: submit_wait(in_pin),
             "run_pageable_in": lambda: run(in_page), "submit_wait_pageable_in": lambda: submit_wait(in_page)}
    for fn in modes.values():   # warm-up: first launches, arena and staging allocations
        fn()
    fps = {m: [] for m in modes}
    identical = []
    for _ in range(args.runs):
        for m, fn in modes.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for _ in range(args.passes):
                fn()
            fps[m].append(round(args.passes * N / (time.perf_counter() - t0), 1))
            if m.startswith("submit_wait"):   # run wrote the same frames just before
                identical.append(same_rows(outs["run"], outs["submit_wait"]))
    fe.close()
    print(json.dumps({"workload": "config 2: %d frames 1280x1024, 650-px faces, nFeatures 3000, batch %d, %d passes per run" % (N, B, args.passes),
                      "frames_per_s": fps, "gpu": gpu_info(), "page_locked_copy": copy_rates(torch),
                      "run_and_submit_wait_identical": all(identical)}))


if __name__ == "__main__":
    main()

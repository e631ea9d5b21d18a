"""Per-call wall time of Frame::ComputeBoW: the GPU drop-in (dropin/ComputeBoW_b200.cpp) against the reference's own body (ComputeBoW_cpu), both
on the same reference Frame objects in oracle/_ref/libdropin_bow.so, with a full-size synthetic vocabulary of ORBvoc.txt's shape (k = 10, L = 6,
10^6 words, written with ORBvoc.txt's final newline and loaded by the reference's loadFromTextFile). Each call is timed with a host clock around
the member call, which returns only after the device results are copied back and the std::maps are built. Reports the first GPU call of the
process (vocabulary import, handle creation, upload of the tree) and the steady state, at 2000 and 6000 features. One JSON line per case.

    python tools/bow_latency.py [--reps 200] [--cpu-reps 20]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def _vp(a):
    return a.ctypes.data_as(C.c_void_p)


def _gpu_name():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True,
                              timeout=30).stdout.strip()
    except Exception as e:   # noqa: BLE001
        return "unknown (%s)" % e


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=200)
    ap.add_argument("--cpu-reps", type=int, default=20)
    args = ap.parse_args()
    import oracle
    from cubemapslam_b200 import config
    from tests.test_gpu_bow_limits import balanced_tree
    from tests.test_oracle_compute_bow import dropin_lib, frame_features, load_vocabulary, write_with_newline

    L = dropin_lib()
    L.dropin_set_camera(C.byref(oracle.cam_params(config.lafida_450())))
    # one leaf short of full: a full tree plus the node the final newline adds would outgrow the node array the loader reserves, and the
    # reallocation leaves the loaded object's word list pointing at freed memory (the drop-in's import refuses such an object)
    voc = balanced_tree(10, 6, seed=3, stop_frac=0.01, drop_last_leaves=1)
    with tempfile.TemporaryDirectory() as tmp:
        path = os.path.join(tmp, "voc.txt")
        t0 = time.perf_counter(); write_with_newline(voc, path); t_write = time.perf_counter() - t0
        t0 = time.perf_counter(); h = load_vocabulary(L, path); t_load = time.perf_counter() - t0
    print(json.dumps(dict(gpu=_gpu_name(), cpu=os.cpu_count(), nodes=len(voc["parent"]) + 1, write_s=round(t_write, 1), load_s=round(t_load, 1))), flush=True)
    for n in (2000, 6000):
        d = np.ascontiguousarray(frame_features(voc, n, 700 + n))
        gpu = np.zeros(args.reps + 1); cpu = np.zeros(args.cpu_reps)
        L.dropin_time_compute_bow(h, 0, n, _vp(d), args.reps + 1, _vp(gpu))
        L.dropin_time_compute_bow(h, 1, n, _vp(d), args.cpu_reps, _vp(cpu))
        steady = gpu[1 + min(10, args.reps // 4):]
        print(json.dumps(dict(features=n, gpu_first_ms=round(gpu[0], 3), gpu_median_ms=round(float(np.median(steady)), 4),
                              gpu_p10_ms=round(float(np.percentile(steady, 10)), 4), gpu_p90_ms=round(float(np.percentile(steady, 90)), 4),
                              cpu_median_ms=round(float(np.median(cpu)), 3), cpu_min_ms=round(float(cpu.min()), 3),
                              cpu_max_ms=round(float(cpu.max()), 3))), flush=True)


if __name__ == "__main__":
    main()

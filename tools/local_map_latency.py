"""Host-call latency of the local-map SearchByProjection: cslam_search_by_projection_local_large at 1024 to 2^20 MapPoints (the local entry
runs the same kernels up to the handle's max_features), and the reference's CPU body (through oracle/_ref/libdropin_local_map.so, which also
builds its Frame / MapPoint objects outside the timed call) where that library exists. One frame of 4096 key points per call, face 650, th 5, as the
drop-in calls it; medians over --reps calls after a warm-up. Prints the card's name and power limit with the numbers, as one JSON line.
  python tools/local_map_latency.py [--reps 30]"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from cubemapslam_b200.tracker import Tracker  # noqa: E402
from tests import local_map_scenes as S  # noqa: E402

SIZES = (1024, 4096, 16384, 65536, 262144, 1 << 20)


def median_ms(fn, reps):
    fn(); fn()
    t = []
    for _ in range(reps):
        t0 = time.perf_counter(); fn(); t.append((time.perf_counter() - t0) * 1e3)
    return round(float(np.median(t)), 4)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=30)
    args = ap.parse_args()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    res = {"gpu": gpu, "reps": args.reps, "face": 650, "keypoints": 4096, "th": 5.0}
    W, th, nn = 650, 5.0, 0.8
    fr = S.frame(0, W)
    t = Tracker(max_frames=1, max_features=4096)   # the drop-in's handle
    for n in SIZES:
        mp = S.local_map(fr, n, n)
        a = (fr["k"], fr["d"], mp["in_view"], mp["proj"], mp["level"], mp["vcos"], mp["dq"], mp["obs"], fr["taken"], W, W, th, nn)
        res["large_%d" % n] = median_ms(lambda: t.SearchByProjection_local_large(*a), args.reps)
    t.close()
    lib = os.path.join(ROOT, "oracle", "_ref", "libdropin_local_map.so")
    if os.path.exists(lib):   # the reference's search alone, timed inside the library (its Frame / MapPoint objects are built untimed)
        from oracle import oracle as orc
        from cubemapslam_b200 import config
        from oracle.oracle import _p
        L = C.CDLL(lib)
        L.dropin_set_camera(C.byref(orc.cam_params(config.front_1024())))
        for n in SIZES[:4]:
            mp = S.local_map(fr, n, n)
            m = np.zeros(len(fr["k"]), np.int32); obs = mp["obs"].astype(np.int32)
            ms = []
            for _ in range(max(3, args.reps // 5)):
                t_ms = C.c_double()
                L.ref_search_by_projection_local_cpu(len(fr["k"]), _p(fr["k"]), _p(fr["d"]), n, _p(mp["in_view"]), _p(mp["proj"]), _p(mp["level"]), _p(mp["vcos"]),
                                                     _p(mp["dq"]), _p(obs), _p(fr["taken"]), C.c_float(th), C.c_float(nn), _p(m), C.byref(t_ms))
                ms.append(t_ms.value)
            res["reference_cpu_%d" % n] = round(float(np.median(ms)), 4)
    else:
        res["reference_cpu"] = "not measured (oracle/_ref/libdropin_local_map.so absent)"
    print(json.dumps(res))


if __name__ == "__main__":
    main()

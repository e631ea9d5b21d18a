"""Host-call latency of SearchForInitialization: the drop-in ORBMatcher::SearchForInitialization (-> cslam_search_for_initialization) and the
reference's CPU body, both called on the same reference Frames inside oracle/_ref/libdropin_init.so (the Frames are built outside the timed
call), on frames of 6024 key points (face 450) and 9024 (face 650) from tests/init_search_scenes.py's dense scenes (clustered: windows of up to
~1800 candidates), and on its extracted pairs (the initialisation extractor's frames of a synthetic fisheye frame),
window 100, nnratio 0.9, checkOri on, as Tracking::CubemapInitialization calls it. Medians over --reps calls after two warm-up calls. Prints the
card's name and power limit with the numbers, as one JSON line.
  python tools/init_search_latency.py [--reps 30]"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import oracle as orc  # noqa: E402
from oracle.oracle import _p  # noqa: E402
from tests import init_search_scenes as S  # noqa: E402

SIZES = ((450, 6024), (650, 9024))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=30)
    args = ap.parse_args()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    res = {"gpu": gpu, "reps": args.reps, "window": 100}
    lib = os.path.join(ROOT, "oracle", "_ref", "libdropin_init.so")
    if not os.path.exists(lib):
        res["error"] = "oracle/_ref/libdropin_init.so absent"
        print(json.dumps(res)); return
    L = C.CDLL(lib)
    for W, n in SIZES:
        L.dropin_set_camera(C.byref(orc.cam_params(S.cam_cfg(W))))
        for tag, (k1, d1, k2, d2, xy) in (("dense_%d" % n, S.dense(100 + W, W, n, n)), ("extracted_%d" % W, S.extracted(orc, W))):
            res["keypoints_" + tag] = [len(k1), len(k2)]
            for gpu_, name in ((1, "dropin"), (0, "reference_cpu")):
                ms = np.zeros(args.reps + 2)
                L.time_search_for_initialization(gpu_, len(k1), _p(k1), _p(d1), len(k2), _p(k2), _p(d2), _p(xy), 100, C.c_float(0.9), 1, args.reps + 2, _p(ms))
                res["%s_%s" % (name, tag)] = round(float(np.median(ms[2:])), 4)
    print(json.dumps(res))


if __name__ == "__main__":
    main()

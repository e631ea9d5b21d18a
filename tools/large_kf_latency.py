"""Host-call latency of the key-frame searches: the _fv / _large entries against the entries they sit beside at 3000 features (where both apply),
and the _fv / _large entries alone at 9024 (the initialisation extractor's key frames at 3000 features). One pair per call, as the drop-ins call
them; medians over --reps calls after a warm-up. Prints the card's name and power limit with the numbers, as one JSON line.
  python tools/large_kf_latency.py [--reps 50]"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from cubemapslam_b200.mapper import Mapper  # noqa: E402
from cubemapslam_b200.matcher import ORBMatcher, pack_fv  # noqa: E402
from oracle import oracle  # noqa: E402
from tests import large_kf_scenes as S  # noqa: E402


def median_ms(fn, reps):
    fn()
    t = []
    for _ in range(reps):
        t0 = time.perf_counter(); fn(); t.append((time.perf_counter() - t0) * 1e3)
    return float(np.median(t))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    args = ap.parse_args()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    res = {"gpu": gpu, "reps": args.reps}
    m = ORBMatcher(0.7, True, max_pairs=1, max_features=4096)
    mp = Mapper()
    for n in (3000, 9024):
        s = S.bow_pair(n, n, n)
        f1, f2 = pack_fv([S.csr(s["node1"], n)], n), pack_fv([S.csr(s["node2"], n)], n)
        one = lambda x: x[None]   # noqa: E731
        res["search_by_bow_fv_%d" % n] = median_ms(lambda: m.SearchByBoW_fv(one(s["d1"]), one(s["a1"]), one(s["v1"]), [n], f1, one(s["d2"]), one(s["a2"]), [n], f2), args.reps)
        res["search_by_bow_kf_fv_%d" % n] = median_ms(lambda: m.SearchByBoW_KF_fv(one(s["d1"]), one(s["a1"]), one(s["v1"]), [n], f1, one(s["d2"]), one(s["a2"]),
                                                                                  one(s["v2"]), [n], f2), args.reps)
        if n <= 4096:
            o1, o2 = S.oracle_nodes(s["node1"], 0) % 1000, S.oracle_nodes(s["node2"], 1) % 1000   # any valid ids: the timing does not depend on them
            res["search_by_bow_%d" % n] = median_ms(lambda: m.SearchByBoW(s["d1"], s["a1"], s["v1"], o1, s["d2"], s["a2"], o2), args.reps)
            res["search_by_bow_kf_%d" % n] = median_ms(lambda: m.SearchByBoW_KF(s["d1"], s["a1"], s["v1"], o1, s["d2"], s["a2"], s["v2"], o2), args.reps)
        t = S.mapping_pair(n, n)
        k1, d1, h1, nd1 = (np.ascontiguousarray(t[k][:n]) for k in ("kCur", "dCur", "hasMPCur", "nodeCur"))
        k2, d2, h2, nd2 = t["kLast"], t["dLast"], t["hasMPObs"], t["nodeObs"]
        r1, _ = oracle.key_point_rays(k1, 650, 650); r2, _ = oracle.key_point_rays(k2, 650, 650)
        T1 = t["TcwCur"].astype(np.float64); Ow = (-T1[:3, :3].T @ T1[:3, 3]).astype(np.float32)[None]
        g1, g2 = pack_fv([S.csr(nd1, n)], n), pack_fv([S.csr(nd2, n)], n)
        geo = (Ow, t["TcwLast"].reshape(1, 16), t["E12"].reshape(1, 9), t["scale"], t["level_sigma2"], 650, 650, True)
        res["triangulation_fv_%d" % n] = median_ms(lambda: mp.SearchForTriangulation_fv(k1[None], d1[None], r1[None], h1[None], [n], g1, k2[None], d2[None], r2[None], h2[None],
                                                                                         [n], g2, *geo), args.reps)
        if n <= 4096:
            res["triangulation_%d" % n] = median_ms(lambda: mp.SearchForTriangulation(k1[None], d1[None], r1[None], h1[None], nd1[None], [n], k2[None], d2[None], r2[None],
                                                                                       h2[None], nd2[None], [n], *geo), args.reps)
        mm = len(t["Xw"]); level = np.clip(t["kLast"]["octave"], 0, 7).astype(np.int32); valid = np.ones(mm, np.uint8)
        fa = (k1, d1, t["TcwCur"], valid, t["Xw"], level, t["dLast"], 3.0, t["scale"], t["inv_level_sigma2"], 650, 650)
        res["fuse_large_%d" % n] = median_ms(lambda: mp.FuseSearch(*fa, large=True), args.reps)
        if n <= 4096:
            res["fuse_%d" % n] = median_ms(lambda: mp.FuseSearch(*fa), args.reps)
    m.close(); mp.close()
    print(json.dumps(res))


if __name__ == "__main__":
    main()

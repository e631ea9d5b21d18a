#!/usr/bin/env python
"""Resident k_fast CTAs per SM at bench.py's headline shape and at CELL_MAX, from the CUDA occupancy calculator; needs a GPU and nvcc.

k_fast's dynamic shared memory (fast_smem in frontend.cu, mirrored below) depends on the level's cell size and on its longest live list.
The live list of a tile holds at most all of its work items, so the layout sized with that many is the largest the level can launch.
Per pyramid level of the front camera's 650-px faces (31-px cells at level 0), and for CELL_MAX cells with the largest live list any
front end accepts and without live lists (caller canvases), the tool compiles frontend.cu (or reads --cubin), loads k_fast through the
driver API and prints one JSON line: dynamic and static shared memory, and cuOccupancyMaxActiveBlocksPerMultiprocessor at 256 threads.

  python tools/kfast_occupancy.py [--cubin file.cubin]
"""
import argparse
import ctypes
import json
import os
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

CG, FAST_TS, CELL_MAX, ITEM_BYTES = 4, 224, 48, 32     # as in frontend.cu (sizeof(FastItem) = 32)
FAST_SW = FAST_TS // 2
K_FAST = b"_ZN5cslam6k_fastEPKhNS_9LevelGeomEiiPjS3_iPiPKNS_8FastColsES1_PKtPKj"


def fast_smem(wCell, hCell, liveCap):
    """fast_smem(g).total: the k_fast CTA's dynamic shared memory in bytes."""
    tileBytes = 16 + (hCell + 6) * FAST_TS
    liveBytes = 16 * ((liveCap + 14) // 8)
    kmax = CG * ((wCell + 1) // 2) * ((hCell + 1) // 2)
    nzCap = max(liveCap, ((CG * wCell + 6) >> 2) * hCell)
    lists = 2 * 16 * ((nzCap + 7) // 8)                  # the pass list and the nz list
    return ITEM_BYTES * (FAST_SW // 2) + lists + 2 * tileBytes + (hCell + 2) * FAST_SW * 4 + 2 * liveBytes + 4 * kmax


def level_layouts():
    """(side, wCell, hCell, largest tile item count) per level of bench.py's front-camera pyramid."""
    import numpy as np
    from fast_live_roofline import _grid
    out, s = [], np.float32(1.0)
    for _ in range(8):
        side = int(np.rint(np.float32(3 * 650) * (np.float32(1.0) / s)))
        s = np.float32(s * np.float32(1.2))
        minB, maxBX, maxBY, wCell, hCell, nColsEff, nRowsEff = _grid(side, side)
        items = 0
        for cx in range(-(-nColsEff // CG)):
            tx0 = minB + cx * CG * wCell
            nx = min(tx0 + min(CG, nColsEff - cx * CG) * wCell + 6, maxBX) - tx0 - 6
            xoff = tx0 - (tx0 & ~15) + 3
            items = max(items, ((xoff + nx + 3) >> 2) - (xoff >> 2))
        out.append((side, wCell, hCell, items * hCell))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cubin", help="read this cubin instead of compiling frontend.cu")
    args = ap.parse_args()
    with tempfile.TemporaryDirectory() as tmp:
        cubin = args.cubin
        if not cubin:
            from kfast_sass import compile_cubin
            cubin = os.path.join(tmp, "frontend.cubin")
            compile_cubin(cubin)
        cu = ctypes.CDLL("libcuda.so.1")

        def ck(r, what):
            if r != 0:
                raise SystemExit("kfast_occupancy.py: %s failed (CUresult %d)" % (what, r))
        ck(cu.cuInit(0), "cuInit")
        dev, ctx, mod, fn = ctypes.c_int(), ctypes.c_void_p(), ctypes.c_void_p(), ctypes.c_void_p()
        ck(cu.cuDeviceGet(ctypes.byref(dev), 0), "cuDeviceGet")
        ck(cu.cuDevicePrimaryCtxRetain(ctypes.byref(ctx), dev), "cuDevicePrimaryCtxRetain")
        ck(cu.cuCtxSetCurrent(ctx), "cuCtxSetCurrent")
        ck(cu.cuModuleLoad(ctypes.byref(mod), cubin.encode()), "cuModuleLoad")
        ck(cu.cuModuleGetFunction(ctypes.byref(fn), mod, K_FAST), "cuModuleGetFunction")
        static = ctypes.c_int()
        ck(cu.cuFuncGetAttribute(ctypes.byref(static), 1, fn), "cuFuncGetAttribute")   # CU_FUNC_ATTRIBUTE_SHARED_SIZE_BYTES
        gmax = fast_smem(CELL_MAX, CELL_MAX, (FAST_SW // 2) * CELL_MAX)
        ck(cu.cuFuncSetAttribute(fn, 8, gmax), "cuFuncSetAttribute")   # CU_FUNC_ATTRIBUTE_MAX_DYNAMIC_SHARED_SIZE_BYTES

        def occ(dyn):
            n = ctypes.c_int()
            ck(cu.cuOccupancyMaxActiveBlocksPerMultiprocessor(ctypes.byref(n), fn, 256, ctypes.c_size_t(dyn)), "cuOccupancyMaxActiveBlocksPerMultiprocessor")
            return n.value
        levels = [{"side": side, "cell": [w, h], "live_cap_bound": lc, "dynamic_smem": fast_smem(w, h, lc), "ctas_per_sm": occ(fast_smem(w, h, lc))}
                  for side, w, h, lc in level_layouts()]
        g0 = fast_smem(CELL_MAX, CELL_MAX, 0)
        cmax = {"cell": CELL_MAX, "longest_live_list": {"dynamic_smem": gmax, "ctas_per_sm": occ(gmax)},
                "no_live_list": {"dynamic_smem": g0, "ctas_per_sm": occ(g0)}}
        cu.cuModuleUnload(mod)
        cu.cuDevicePrimaryCtxRelease(dev)
    from match_roofline import card
    print(json.dumps({"card": card(), "static_smem": static.value, "levels": levels, "cell_max": cmax}))


if __name__ == "__main__":
    main()

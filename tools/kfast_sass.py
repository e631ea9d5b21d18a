#!/usr/bin/env python
"""Static instruction budget of k_fast (frontend.cu) from its sm_90a SASS; needs nvcc/cuobjdump, no GPU.

Compiles cubemapslam_b200/csrc/frontend.cu for sm_90a with the library's flags (or reads --cubin), disassembles k_fast and prints one JSON
object:

  registers, spill_bytes, smem_bytes   ptxas's resource report for k_fast (only when this tool compiled it)
  prologue                             instructions before the strip loop: total and the integer-division opcodes (I2F, MUFU, F2I)
  strip                                the loop over a CTA's cell rows (a loop with a barrier around >= 64 VIMNMX3 / VIMNMX: it holds phases A to C),
                                       with its BAR and ATOMG counts (`bar`, `atomg`: every path of one pass, flush of the output buffer included)
  staging                              each tile-staging loop (a loop whose body issues cp.async, LDGSTS, and no score arithmetic)
  phase_a                              each scoring loop (a loop without a barrier whose body issues >= 64 VIMNMX3 / VIMNMX), `live` when its body loads
                                       the u16 live list (staged in shared memory); `append`: the instructions of its body that append a non-zero
                                       item to the nz list (the atomic ptxas aggregates per warp and the u16 store: VOTEU, FLO, POPC, S2R, SHFL,
                                       ATOMS, STS.U16 and the uniform address arithmetic)
  phase_a0                             each compass-pretest loop (a loop without a barrier whose body issues fewer than 64 VIMNMX3 / VIMNMX, a
                                       shared-memory atomic and a u16 store: the pass-list append), with `live` and `append` as for phase_a
  phase_b                              each NMS loop (a loop with a shared-memory atomic, VIMNMX3 and no barrier)

k_fast has two phase_a0 loops (live list, caller canvases), two phase_a loops (the pass list, then round 2's deferred items) and two
phase_b loops (round 1 over nzHi, round 2 over the fallback cells).
  compaction                           the other loops with a shared-memory atomic and no barrier (NMS survivors, phase C)
  each loop                            [start, end] byte offsets, the body's instruction count and its opcode histogram

A loop is the address range from a backward branch's target to the branch. Counts are static: one pass through the body, every path
included, NOPs excluded.

  python tools/kfast_sass.py [--cubin file.cubin]
"""
import argparse
import json
import os
import re
import subprocess
import sys
import tempfile
from collections import Counter

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CUDA = os.environ.get("CUDA_HOME", "/usr/local/cuda")
INSN = re.compile(r"/\*([0-9a-f]{4,})\*/\s+(@!?U?P\w+\s+)?([A-Z][A-Z0-9_.x]*)([^;]*);")
RES = re.compile(r"Used (\d+) registers.*?(\d+) bytes smem")
APPEND = {"VOTEU", "FLO", "POPC", "S2R", "S2UR", "SHFL", "ATOMS", "UMOV", "UIADD3", "ULEA"}
SPILL = re.compile(r"(\d+) bytes spill stores, (\d+) bytes spill loads")


def compile_cubin(out):
    sys.path.insert(0, ROOT)
    from cubemapslam_b200 import build
    src = os.path.join(ROOT, "cubemapslam_b200", "csrc", "frontend.cu")
    cmd = [os.path.join(CUDA, "bin", "nvcc")] + build.ARCH + ["-O3", "-std=c++17", "-cubin", "-Xptxas", "-v", "-o", out, src]
    log = subprocess.run(cmd, check=True, capture_output=True, text=True).stderr
    res = {}
    lines = log.splitlines()
    for i, ln in enumerate(lines):
        if "Function properties for" in ln and "k_fast" in ln:
            for nxt in lines[i + 1:i + 3]:
                m, s = RES.search(nxt), SPILL.search(nxt)
                if s:
                    res["spill_bytes"] = int(s.group(1)) + int(s.group(2))
                if m:
                    res["registers"], res["smem_bytes"] = int(m.group(1)), int(m.group(2))
    return res


def k_fast_sass(cubin):
    text = subprocess.run([os.path.join(CUDA, "bin", "cuobjdump"), "-sass", cubin], check=True, capture_output=True, text=True).stdout
    insns, inside = [], False
    for ln in text.splitlines():
        if "Function :" in ln:
            inside = "k_fast" in ln
            continue
        m = INSN.search(ln) if inside else None
        if m:
            insns.append((int(m.group(1), 16), m.group(3), m.group(4)))
    if not insns:
        raise SystemExit("kfast_sass.py: no k_fast in %s" % cubin)
    return insns


def loops(insns):
    out = []
    for addr, op, args in insns:
        t = re.search(r"0x([0-9a-f]+)", args)
        if op.startswith("BRA") and t and int(t.group(1), 16) <= addr:
            out.append((int(t.group(1), 16), addr))
    return out


def body(insns, lo, hi):
    return [(op, args) for a, op, args in insns if lo <= a <= hi and op != "NOP"]


def hist(ins):
    return dict(Counter(op.split(".")[0] for op, _ in ins).most_common())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cubin", help="read this cubin instead of compiling frontend.cu")
    args = ap.parse_args()
    res = {}
    with tempfile.TemporaryDirectory() as tmp:
        cubin = args.cubin
        if not cubin:
            cubin = os.path.join(tmp, "frontend.cubin")
            res = compile_cubin(cubin)
        insns = k_fast_sass(cubin)
    strip, phase_a0, phase_a, phase_b, compaction, staging = [], [], [], [], [], []
    for lo, hi in loops(insns):
        b = body(insns, lo, hi)
        h = hist(b)
        entry = {"range": [hex(lo), hex(hi)], "instructions": len(b), "histogram": h}
        minmax = h.get("VIMNMX3", 0) + h.get("VIMNMX", 0)
        if minmax >= 64 and h.get("BAR", 0):
            entry["bar"], entry["atomg"] = h.get("BAR", 0), h.get("ATOMG", 0)
            strip.append(entry)
        elif minmax >= 64 or (h.get("ATOMS", 0) and not h.get("BAR", 0) and any(op.startswith("STS.U16") for op, _ in b)):
            entry["live"] = any(op.startswith("LDS") and ".U16" in op for op, _ in b)
            entry["append"] = sum(1 for op, _ in b if op.split(".")[0] in APPEND or op.startswith("STS.U16"))
            (phase_a if minmax >= 64 else phase_a0).append(entry)
        elif h.get("ATOMS", 0) and not h.get("BAR", 0):
            (phase_b if h.get("VIMNMX3", 0) else compaction).append(entry)
        elif h.get("LDGSTS", 0):
            staging.append(entry)
    first_a = min((int(e["range"][0], 16) for e in strip + phase_a0 + phase_a), default=insns[-1][0] + 1)
    pro = [op for a, op, _ in insns if a < first_a and op != "NOP"]
    pro_h = Counter(op.split(".")[0] for op in pro)
    out = dict(res)
    out["prologue"] = {"instructions": len(pro), "I2F": pro_h.get("I2F", 0), "MUFU": pro_h.get("MUFU", 0), "F2I": pro_h.get("F2I", 0)}
    out["strip"] = strip
    out["phase_a0"] = phase_a0
    out["phase_a"] = phase_a
    out["phase_b"] = phase_b
    out["compaction"] = compaction
    out["staging"] = staging
    print(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()

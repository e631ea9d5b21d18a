#!/usr/bin/env python
"""Static instruction budget of k_pyramid, k_distribute and k_describe (frontend.cu) from their sm_90a SASS; needs nvcc/cuobjdump, no GPU.

Compiles cubemapslam_b200/csrc/frontend.cu (or --src) for sm_90a with the library's flags, or reads --cubin, disassembles every
instantiation of the three kernels and prints one JSON object per kernel name (template instantiations are listed separately):

  registers, spill_bytes, smem_bytes   ptxas's resource report (only when this tool compiled the source)
  instructions                         static instructions of the whole kernel
  barriers                             static BAR instructions
  straight                             static instructions outside every loop
  loops                                each loop: [start, end] byte offsets, the body's instruction count and its opcode histogram

A loop is the address range from a backward branch's target to the branch. Counts are static: one pass through each body, every path
included, NOPs excluded. Dynamic counts follow from the trip counts, which the kernel's shapes give (DESIGN.md section 4).

  python tools/frontend_sass.py [--src frontend.cu | --cubin file.cubin]
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
KERNELS = ("k_pyramid", "k_distribute", "k_describe")
INSN = re.compile(r"/\*([0-9a-f]{4,})\*/\s+(@!?U?P\w+\s+)?([A-Z][A-Z0-9_.x]*)([^;]*);")
RES = re.compile(r"Used (\d+) registers")
SMEM = re.compile(r"(\d+) bytes smem")
SPILL = re.compile(r"(\d+) bytes spill stores, (\d+) bytes spill loads")


def compile_cubin(src, out):
    sys.path.insert(0, ROOT)
    from cubemapslam_b200 import build
    cmd = [os.path.join(CUDA, "bin", "nvcc")] + build.ARCH + ["-O3", "-std=c++17", "-cubin", "-Xptxas", "-v", "-o", out, src]
    log = subprocess.run(cmd, check=True, capture_output=True, text=True, cwd=os.path.dirname(src)).stderr
    res = {}
    lines = log.splitlines()
    for i, ln in enumerate(lines):
        m = re.search(r"Function properties for (\S+)", ln)
        if not m or not any(k in m.group(1) for k in KERNELS):
            continue
        r = res.setdefault(m.group(1), {})
        for nxt in lines[i + 1:i + 3]:
            mm, s, sm = RES.search(nxt), SPILL.search(nxt), SMEM.search(nxt)
            if s:
                r["spill_bytes"] = int(s.group(1)) + int(s.group(2))
            if mm:
                r["registers"], r["smem_bytes"] = int(mm.group(1)), int(sm.group(1)) if sm else 0
    return res


def functions(cubin):
    text = subprocess.run([os.path.join(CUDA, "bin", "cuobjdump"), "-sass", cubin], check=True, capture_output=True, text=True).stdout
    out, cur = {}, None
    for ln in text.splitlines():
        if "Function :" in ln:
            name = ln.split("Function :")[1].strip()
            cur = name if any(k in name for k in KERNELS) else None
            if cur:
                out[cur] = []
            continue
        m = INSN.search(ln) if cur else None
        if m:
            out[cur].append((int(m.group(1), 16), m.group(3), m.group(4)))
    if not out:
        raise SystemExit("frontend_sass.py: no %s in %s" % (" / ".join(KERNELS), cubin))
    return out


def loops(insns):
    out = []
    for addr, op, args in insns:
        t = re.search(r"0x([0-9a-f]+)", args)
        if op.startswith("BRA") and t and int(t.group(1), 16) <= addr:
            out.append((int(t.group(1), 16), addr))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--src", default=os.path.join(ROOT, "cubemapslam_b200", "csrc", "frontend.cu"), help="frontend.cu to compile")
    ap.add_argument("--cubin", help="read this cubin instead of compiling")
    args = ap.parse_args()
    res = {}
    with tempfile.TemporaryDirectory() as tmp:
        cubin = args.cubin
        if not cubin:
            cubin = os.path.join(tmp, "frontend.cubin")
            res = compile_cubin(os.path.abspath(args.src), cubin)
        fns = functions(cubin)
    out = {}
    for name, insns in sorted(fns.items()):
        live = [(a, op) for a, op, _ in insns if op != "NOP"]
        lp = loops(insns)
        inside = lambda a: any(lo <= a <= hi for lo, hi in lp)
        entry = dict(res.get(name, {}))
        entry["instructions"] = len(live)
        entry["barriers"] = sum(1 for _, op in live if op.split(".")[0] == "BAR")
        entry["straight"] = sum(1 for a, _ in live if not inside(a))
        entry["loops"] = []
        for lo, hi in lp:
            b = [op for a, op in live if lo <= a <= hi]
            entry["loops"].append({"range": [hex(lo), hex(hi)], "instructions": len(b),
                                   "histogram": dict(Counter(op.split(".")[0] for op in b).most_common())})
        out[name] = entry
    print(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()

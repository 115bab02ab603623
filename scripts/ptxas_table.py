#!/usr/bin/env python
"""Registers / spills / shared memory per kernel (ptxas -v) and the Hopper-class SASS mnemonics each kernel contains (warp
REDUX, MATCH, 64-bit shared atomics, bulk asynchronous copies UBLKCP and the mbarrier operations SYNCS they complete on).
The SASS is read from the object file the script compiles, so the table needs no prior build of the library.
usage: python scripts/ptxas_table.py > ptxas_sass.txt   (no GPU needed: nvcc cross-compiles)"""
import os, re, subprocess, sys, collections, tempfile
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from urban_road_filter_b200 import build
src = os.path.join(build.CSRC, "urf_api.cu")
obj = os.path.join(tempfile.mkdtemp(prefix="urf_ptxas_"), "urf_api.o")
out = subprocess.run([build._nvcc(), *build.NVCC_FLAGS, "-Xptxas=-v", "-c", src, "-o", obj], capture_output=True, text=True, check=True).stderr
rows = []
for m in re.finditer(r"Compiling entry function '(\S+)' for 'sm_90a'\n.*?\n\s+(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads\nptxas info\s+: Used (\d+) registers(?:, used (\d+) barriers)?(?:, (\d+) bytes cumulative stack size)?(?:, (\d+) bytes smem)?", out):
    name = subprocess.run(["c++filt", m.group(1)], capture_output=True, text=True).stdout.strip().split("(")[0].replace("urf::", "")
    rows.append((name, int(m.group(5)), int(m.group(2)), int(m.group(3)), int(m.group(4)), int(m.group(8) or 0)))
sass = subprocess.run(["cuobjdump", "-sass", obj], capture_output=True, text=True, check=True).stdout
per = collections.defaultdict(collections.Counter)
cur = None
for line in sass.splitlines():
    m = re.search(r"Function : (\S+)", line)
    if m:
        cur = subprocess.run(["c++filt", m.group(1)], capture_output=True, text=True).stdout.strip().split("(")[0].replace("urf::", "")
        continue
    m = re.match(r"\s+/\*[0-9a-f]+\*/\s+(?:@!?U?P\d+\s+)?([A-Z0-9_.]+)", line)
    if m and cur:
        op = m.group(1)
        for tag in ("REDUX", "MATCH", "ATOMS", "ATOM", "RED", "SHFL", "DSQRT", "MUFU.RSQ64H", "DFMA", "DMUL", "DADD", "LDL", "STL", "BAR.SYNC", "VOTE", "UBLKCP", "SYNCS"):
            if op.startswith(tag):
                per[cur][tag] += 1
                break
        per[cur]["total"] += 1
print("urf_api.cu compiled with:", " ".join(build.NVCC_FLAGS))
print(f"{'kernel':28s} {'regs':>4s} {'stack':>5s} {'spill_st':>8s} {'spill_ld':>8s} {'smem_B':>7s} {'sass':>6s}  notable SASS (static counts)")
for name, regs, stack, sst, sld, smem in sorted(rows):
    c = per.get(name, {})
    notes = ", ".join(f"{k} {v}" for k, v in sorted(c.items()) if k != "total" and k not in ("DFMA", "DMUL", "DADD") and v)
    print(f"{name:28s} {regs:4d} {stack:5d} {sst:8d} {sld:8d} {smem:7d} {c.get('total', 0):6d}  {notes}")
print("\nREDUX = warp-wide integer reduce; MATCH = __match_any_sync; UBLKCP = cp.async.bulk (k_scatter stages each warp's")
print("8 KB of input records with one), SYNCS = the mbarrier init / expect-tx / wait it completes on. No tensor-core")
print("instructions: the path has no dense contraction.")

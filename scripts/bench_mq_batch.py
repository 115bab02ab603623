#!/usr/bin/env python
"""Single-process throughput of one ingest stream over N GPUs (urf_mq, BASELINE config 4: OS2-128 scans), per-scan delivery
with labels read in place (urf_mq_next_view, int32 slots) against batched delivery on int8 slots (urf_mq_next_batch).
Both use the same producers (urf_mq_submit_ref from pinned buffers, tools/mq_bench modes 2 and 3). Runs the two modes
alternately `--repeats` times per GPU count and prints the medians as a markdown table, with the cards' power limit and
clocks as nvidia-smi reports them.
usage: python scripts/bench_mq_batch.py [--gpus 1,2,4,8] [--shape C4] [--scans 3000] [--producers 4] [--repeats 3]"""
import argparse, json, os, statistics, subprocess, sys, tempfile
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np
import torch
from urban_road_filter_b200.synth import SHAPES, make_scan
from urban_road_filter_b200 import build

ap = argparse.ArgumentParser()
ap.add_argument("--gpus", default="1,2,4,8")
ap.add_argument("--shape", default="C4")
ap.add_argument("--scans", type=int, default=3000)
ap.add_argument("--producers", type=int, default=4)
ap.add_argument("--slots", type=int, default=24)
ap.add_argument("--max-batch", type=int, default=16)
ap.add_argument("--max-results", type=int, default=64)
ap.add_argument("--repeats", type=int, default=3)
args = ap.parse_args()
visible = torch.cuda.device_count()
counts = [g for g in (int(x) for x in args.gpus.split(",")) if g <= visible]
if not counts:
    sys.exit(f"no GPU count of {args.gpus} is available ({visible} visible)")
exe = build.build_tools()
sh = SHAPES[args.shape]
K = 16
n = sh.rings * sh.cols
tmp = tempfile.mkdtemp(prefix="urf_mq_batch_")
path = os.path.join(tmp, f"urf_{args.shape}.bin")
with open(path, "wb") as f:
    for k in range(K):
        f.write(np.ascontiguousarray(make_scan(args.shape, 500 + k), np.float32).tobytes())
smi = subprocess.run(["nvidia-smi", "--query-gpu=index,name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                     capture_output=True, text=True).stdout.strip()
print("GPUs (index, name, power limit, SM clock, max SM clock):\n" + smi)
env = {**os.environ, "LD_LIBRARY_PATH": os.path.join(ROOT, "urban_road_filter_b200")}
MODES = {2: "next_view_int32", 3: "next_batch_int8"}
rows = []
for g in counts:
    runs = {m: [] for m in MODES}
    for r in range(args.repeats):
        for m in ((2, 3) if r % 2 == 0 else (3, 2)):              # alternated, so drift does not favour one mode
            out = subprocess.run([exe, path, str(n), str(K), str(g), str(args.producers), str(args.scans), str(args.slots),
                                  str(args.max_batch), "1", str(sh.channels), str(sh.interval), str(m), str(args.max_results)],
                                 check=True, capture_output=True, text=True, env=env).stdout
            res = json.loads(out.strip().splitlines()[-1])
            runs[m].append(res["scans_per_sec"])
    med = {m: statistics.median(v) for m, v in runs.items()}
    rows.append((g, med, runs))
    print(json.dumps({"bench_mq_batch": args.shape, "gpus": g, "producers": args.producers, "points_per_scan": n,
                      **{MODES[m] + "_scans_per_sec": round(med[m], 1) for m in MODES},
                      **{MODES[m] + "_runs": [round(x, 1) for x in runs[m]] for m in MODES}}), flush=True)
print(f"\n| GPUs | urf_mq_next_view, int32 slots (scans/s) | urf_mq_next_batch, int8 slots (scans/s) | ratio |")
print("|---|---|---|---|")
for g, med, _ in rows:
    print(f"| {g} | {med[2]:,.0f} | {med[3]:,.0f} | {med[3] / med[2]:.2f} |")
os.remove(path)
os.rmdir(tmp)

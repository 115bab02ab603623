#!/usr/bin/env python
"""Single-process throughput of one ingest stream over every visible GPU (urf_mq, BASELINE config 4: OS2-128 scans) fed with
48-byte Ouster PointCloud2 records, two ways (tools/mq_bench modes 5 and 4):
  repacked:  a float4 mq; each producer repacks the records of its scan into (x, y, z, intensity) points, inside the timed
             region, and submits them by reference (urf_mq_submit_ref) — 16 bytes per point cross PCIe;
  records:   a record mq (urf_mq_create_cloud2); each producer submits the records as they are, by reference
             (urf_mq_submit_cloud2_ref), and the device unpacks them — 48 bytes per point cross PCIe.
Both with the settings of scripts/bench_mq_batch.py: 4 producers, 24 slots per device, max_batch 16, int8 label slots,
results taken with urf_mq_next_batch. The two modes run alternately `--repeats` times; prints the median and range of
scans/s per mode and the input GB/s that crossed PCIe, as a markdown table, with the cards' power limit and clocks as
nvidia-smi reports them.
usage: python scripts/bench_mq_records.py [--gpus N] [--shape C4] [--scans 3000] [--producers 4] [--repeats 3]"""
import argparse, json, os, statistics, subprocess, sys, tempfile
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np
import torch
from urban_road_filter_b200.synth import SHAPES, make_scan
from urban_road_filter_b200 import build

STEP, OFFS = 48, (0, 4, 8, 16)       # Ouster records: x, y, z, intensity at 0, 4, 8, 16

ap = argparse.ArgumentParser()
ap.add_argument("--gpus", type=int, default=0, help="devices to shard over (default: every visible GPU)")
ap.add_argument("--shape", default="C4")
ap.add_argument("--scans", type=int, default=3000)
ap.add_argument("--producers", type=int, default=4)
ap.add_argument("--slots", type=int, default=24)
ap.add_argument("--max-batch", type=int, default=16)
ap.add_argument("--max-results", type=int, default=64)
ap.add_argument("--repeats", type=int, default=3)
args = ap.parse_args()
visible = torch.cuda.device_count()
if visible < 1:
    sys.exit("no GPU is visible")
g = args.gpus or visible
if g > visible:
    sys.exit(f"{g} GPUs asked for, {visible} visible")
exe = build.build_tools()
sh = SHAPES[args.shape]
K = 16
n = sh.rings * sh.cols
tmp = tempfile.mkdtemp(prefix="urf_mq_records_")
path = os.path.join(tmp, f"urf_{args.shape}_rec{STEP}.bin")
with open(path, "wb") as f:
    for k in range(K):
        pts = np.ascontiguousarray(make_scan(args.shape, 500 + k), np.float32)
        rec = np.random.default_rng(k).integers(0, 256, (n, STEP), dtype=np.uint8)    # the fields the filter does not read
        for j, off in enumerate(OFFS):
            rec[:, off: off + 4] = pts[:, j: j + 1].copy().view(np.uint8)
        f.write(rec.tobytes())
smi = subprocess.run(["nvidia-smi", "--query-gpu=index,name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                     capture_output=True, text=True).stdout.strip()
print("GPUs (index, name, power limit, SM clock, max SM clock):\n" + smi)
env = {**os.environ, "LD_LIBRARY_PATH": os.path.join(ROOT, "urban_road_filter_b200")}
MODES = {5: "repacked", 4: "records"}
runs = {m: [] for m in MODES}
gbs = {m: [] for m in MODES}
for r in range(args.repeats):
    for m in ((5, 4) if r % 2 == 0 else (4, 5)):                  # alternated, so drift does not favour one mode
        out = subprocess.run([exe, path, str(n), str(K), str(g), str(args.producers), str(args.scans), str(args.slots),
                              str(args.max_batch), "1", str(sh.channels), str(sh.interval), str(m), str(args.max_results), "0",
                              str(STEP), *map(str, OFFS)], check=True, capture_output=True, text=True, env=env).stdout
        res = json.loads(out.strip().splitlines()[-1])
        runs[m].append(res["scans_per_sec"])
        gbs[m].append(res["h2d_gb_per_sec"])
        print(json.dumps(res), flush=True)
med = {m: statistics.median(v) for m, v in runs.items()}
print(json.dumps({"bench_mq_records": args.shape, "gpus": g, "producers": args.producers, "points_per_scan": n,
                  **{MODES[m] + "_scans_per_sec": round(med[m], 1) for m in MODES},
                  **{MODES[m] + "_runs": [round(x, 1) for x in runs[m]] for m in MODES},
                  **{MODES[m] + "_h2d_gb_per_sec": round(statistics.median(gbs[m]), 2) for m in MODES}}), flush=True)
print(f"\n| GPUs | mode | input bytes / point over PCIe | scans/s, median | range ({args.repeats} runs) | input GB/s over PCIe |")
print("|---|---|---|---|---|---|")
for m, label in ((5, "float4, repacked on the producer"), (4, "48-byte records, by reference")):
    print(f"| {g} | {label} | {STEP if m == 4 else 16} | {med[m]:,.0f} | {min(runs[m]):,.0f} – {max(runs[m]):,.0f} | "
          f"{statistics.median(gbs[m]):.1f} |")
print(f"\nrecords / repacked: {med[4] / med[5]:.2f}")
os.remove(path)
os.rmdir(tmp)

#!/usr/bin/env python
"""What delivering the emission order costs a streaming queue (URF_QUEUE_ORDER): single-process throughput of urf_mq on
int8 label slots, results taken with urf_mq_next_batch (tools/mq_bench mode 3), with and without the order. With it every
batch runs the per-ring azimuth sort and copies 4 bytes per input point more to the host. Runs the two settings alternately
`--repeats` times per scan shape and GPU count (one GPU and every visible GPU) and prints the medians as a markdown table,
with the cards' name and power limit as nvidia-smi reports them in the same run.
usage: python scripts/bench_queue_order.py [--shapes C2,C4] [--scans 3000] [--producers 4] [--repeats 3]"""
import argparse, json, os, statistics, subprocess, sys, tempfile
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np
import torch
from urban_road_filter_b200.synth import SHAPES, make_scan
from urban_road_filter_b200 import build

ap = argparse.ArgumentParser()
ap.add_argument("--shapes", default="C2,C4")
ap.add_argument("--scans", type=int, default=3000)
ap.add_argument("--producers", type=int, default=4)
ap.add_argument("--slots", type=int, default=24)
ap.add_argument("--max-batch", type=int, default=16)
ap.add_argument("--max-results", type=int, default=64)
ap.add_argument("--repeats", type=int, default=3)
args = ap.parse_args()
visible = torch.cuda.device_count()
if visible < 1:
    sys.exit("no GPU visible")
counts = sorted({1, visible})
exe = build.build_tools()
smi = subprocess.run(["nvidia-smi", "--query-gpu=index,name,power.limit", "--format=csv,noheader"], capture_output=True,
                     text=True).stdout.strip()
print("GPUs (index, name, power limit):\n" + smi)
env = {**os.environ, "LD_LIBRARY_PATH": os.path.join(ROOT, "urban_road_filter_b200")}
K = 16
SETTINGS = {0: "without_order", 1: "with_order"}
tmp = tempfile.mkdtemp(prefix="urf_queue_order_")
rows = []
for shape in args.shapes.split(","):
    sh = SHAPES[shape]
    n = sh.rings * sh.cols
    path = os.path.join(tmp, f"urf_{shape}.bin")
    with open(path, "wb") as f:
        for k in range(K):
            f.write(np.ascontiguousarray(make_scan(shape, 500 + k), np.float32).tobytes())
    for g in counts:
        runs = {o: [] for o in SETTINGS}
        for r in range(args.repeats):
            for o in ((0, 1) if r % 2 == 0 else (1, 0)):          # alternated, so drift does not favour one setting
                out = subprocess.run([exe, path, str(n), str(K), str(g), str(args.producers), str(args.scans), str(args.slots),
                                      str(args.max_batch), "1", str(sh.channels), str(sh.interval), "3", str(args.max_results), str(o)],
                                     check=True, capture_output=True, text=True, env=env).stdout
                res = json.loads(out.strip().splitlines()[-1])
                assert res["order"] == o and (res["ordered_points"] > 0) == bool(o), res
                runs[o].append(res["scans_per_sec"])
        med = {o: statistics.median(v) for o, v in runs.items()}
        rows.append((shape, n, g, med))
        print(json.dumps({"bench_queue_order": shape, "gpus": g, "producers": args.producers, "points_per_scan": n,
                          **{SETTINGS[o] + "_scans_per_sec": round(med[o], 1) for o in SETTINGS},
                          **{SETTINGS[o] + "_runs": [round(x, 1) for x in runs[o]] for o in SETTINGS}}), flush=True)
    os.remove(path)
os.rmdir(tmp)
print("\n| scans | GPUs | without order (scans/s) | with URF_QUEUE_ORDER (scans/s) | ratio |")
print("|---|---|---|---|---|")
for shape, n, g, med in rows:
    print(f"| {shape} ({n:,} points) | {g} | {med[0]:,.0f} | {med[1]:,.0f} | {med[1] / med[0]:.3f} |")

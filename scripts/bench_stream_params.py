#!/usr/bin/env python
"""Cost of a parameter update on a running urf_queue (urf_queue_update_params): scans/s of one stream with no updates
against the same stream with one update every `--every` scans. An update costs the stream one shorter batch (the worker
ends a run at the first scan of the new generation) and, when the next small batch takes the CUDA-graph path, a graph
re-capture. The settings are those of scripts/bench_async_batch.py: full ROI with the shape's channels and interval,
batches of up to `--batch` scans, pinned scans submitted by reference by one producer thread, results taken with
urf_queue_next_batch by one consumer thread. The updates alternate between two sets with the same launch sequence
(curb_height 0.05 / 0.06). Modes alternate `--repeats` times; medians and every run are printed.
usage: python scripts/bench_stream_params.py [--shapes C2,C4] [--scans 3000] [--every 100] [--batch 16] [--repeats 3]"""
import argparse, ctypes as C, json, os, statistics, subprocess, sys, threading, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np
import torch
from urban_road_filter_b200 import FULL_ROI, api, make_params
from urban_road_filter_b200.synth import SHAPES, make_scan

ap = argparse.ArgumentParser()
ap.add_argument("--shapes", default="C2,C4")
ap.add_argument("--scans", type=int, default=3000)
ap.add_argument("--every", type=int, default=100)
ap.add_argument("--batch", type=int, default=16)
ap.add_argument("--slots", type=int, default=32)
ap.add_argument("--warmup", type=int, default=200)
ap.add_argument("--repeats", type=int, default=3)
args = ap.parse_args()
if not torch.cuda.is_available():
    sys.exit("no GPU: this benchmark measures the device")
smi = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                     capture_output=True, text=True).stdout.strip()
print("GPU 0 (name, power limit, SM clock, max SM clock): " + smi, flush=True)
lib = api.load_library()
B = args.batch


def pinned(a):
    p = lib.urf_pinned_alloc(a.nbytes)
    dst = np.ctypeslib.as_array(C.cast(p, C.POINTER(C.c_uint8)), shape=(a.nbytes,)).view(a.dtype).reshape(a.shape)
    dst[...] = a
    return p, dst


def run(q, scans, count, every, sets):
    """Wall seconds for `count` scans through the queue; an update every `every` scans (0: none). Returns (s, updates)."""
    done = [0]

    def consume():
        while done[0] < count:
            out = q.next_batch(64, 60000)
            if not out:
                raise RuntimeError("queue timed out")
            done[0] += len(out)

    cons = threading.Thread(target=consume)
    updates = 0
    t0 = time.perf_counter()
    cons.start()
    for k in range(count):
        if every and k and k % every == 0:
            q.update_params(sets[updates % 2])
            updates += 1
        if q.submit(scans[k % len(scans)], tag=k, timeout_ms=60000, by_reference=True) != api.URF_OK:
            raise RuntimeError("submit failed")
    cons.join()
    return time.perf_counter() - t0, updates


rows = []
for shape in args.shapes.split(","):
    sh = SHAPES[shape]
    clouds = [make_scan(shape, 900 + k) for k in range(B)]
    n = max(c.shape[0] for c in clouds)
    base = dict(FULL_ROI, channels=sh.channels, interval=sh.interval)
    sets = [make_params(**base, curb_height=0.06), make_params(**base, curb_height=0.05)]
    det = api.Detector(max_points=n, max_batch=B, params=make_params(**base))
    keep = [pinned(np.ascontiguousarray(c, np.float32)) for c in clouds]
    scans = [a for _, a in keep]
    q = api.ScanQueue(det, max_points=n, slots=args.slots, max_batch=B)
    run(q, scans, args.warmup, 0, sets)
    run(q, scans, args.warmup, args.every, sets)
    runs = {"no_updates": [], "updates": []}
    n_updates = 0
    for r in range(args.repeats):
        for mode in (("no_updates", "updates") if r % 2 == 0 else ("updates", "no_updates")):
            wall, u = run(q, scans, args.scans, args.every if mode == "updates" else 0, sets)
            runs[mode].append(args.scans / wall)
            n_updates = max(n_updates, u)
    st = q.stats()
    q.close()
    q.destroy()
    det.close()
    for p, _ in keep:
        lib.urf_pinned_free(p)
    med = {m: statistics.median(v) for m, v in runs.items()}
    line = {"bench_stream_params": shape, "batch": B, "points_per_scan": n, "scans": args.scans, "update_every": args.every,
            "updates_per_run": n_updates, "batches_total": st["batches"], "most_in_flight": st["most_in_flight"]}
    for m, v in runs.items():
        line[m] = {"scans_per_sec": round(med[m], 1), "runs_scans_per_sec": [round(x, 1) for x in v]}
    # per update: the extra wall time of the run with updates over the one without, divided by the updates
    line["ms_per_update"] = round(1e3 * (args.scans / med["updates"] - args.scans / med["no_updates"]) / max(n_updates, 1), 3)
    print(json.dumps(line), flush=True)
    rows.append((shape, med, line["ms_per_update"]))

print(f"\n| shape x {B} | no updates (scans/s) | one update per {args.every} scans (scans/s) | ratio | ms per update |")
print("|---|---|---|---|---|")
for shape, med, ms in rows:
    print(f"| {shape} | {med['no_updates']:,.0f} | {med['updates']:,.0f} | {med['updates'] / med['no_updates']:.3f} | {ms:.3f} |")

#!/usr/bin/env python
"""Host-buffer batches back to back from pinned buffers: a urf_process_batch loop (one batch at a time, what the queue
worker did before it kept two batches in flight) against a urf_enqueue_batch / urf_finish_batch loop with two batches in
flight (what it does now). Per shape: scans/s of both loops, alternated `--repeats` times (medians), and the device's idle
time between consecutive batches = (wall time - the sum of the batches' kernel spans, CUDA events) / batches. The labels
of both loops are compared byte for byte.
With --old-lib DIR (a liburf_b200.so of another build): tools/mq_bench (urf_mq at one GPU, the settings of
scripts/bench_mq_batch.py: urf_mq_next_view on int32 slots and urf_mq_next_batch on int8 slots) alternately against that
library and this tree's, medians and every run.
usage: python scripts/bench_async_batch.py [--shapes C2,C4] [--batch 16] [--steps 100] [--repeats 3] [--old-lib DIR]"""
import argparse, ctypes as C, json, os, statistics, subprocess, sys, tempfile, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np
import torch
from urban_road_filter_b200 import FULL_ROI, UrfResult, api, build, make_params
from urban_road_filter_b200.synth import SHAPES, make_scan

ap = argparse.ArgumentParser()
ap.add_argument("--shapes", default="C2,C4")
ap.add_argument("--batch", type=int, default=16)
ap.add_argument("--steps", type=int, default=100)
ap.add_argument("--warmup", type=int, default=5)
ap.add_argument("--repeats", type=int, default=3)
ap.add_argument("--old-lib", default=None)
ap.add_argument("--mq-scans", type=int, default=3000)
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


def check(rc, where):
    if rc != 0:
        raise RuntimeError(f"{where}: {rc} {lib.urf_last_cuda_error(det._ctx).decode()}")


rows = []
for shape in args.shapes.split(","):
    sh = SHAPES[shape]
    clouds = [make_scan(shape, 900 + k) for k in range(B)]
    n = max(c.shape[0] for c in clouds)
    det = api.Detector(max_points=n, max_batch=B, params=make_params(**FULL_ROI, channels=sh.channels, interval=sh.interval))
    keep = [pinned(np.ascontiguousarray(c, np.float32)) for c in clouds]
    ptrs = (C.c_void_p * B)(*[p for p, _ in keep])
    ns = (C.c_int * B)(*[c.shape[0] for c in clouds])
    sets = []                                                # result buffers of the two batches in flight
    for s in range(2):
        labs = [pinned(np.zeros(n, np.int32)) for _ in range(B)]
        res = (UrfResult * B)()
        for b in range(B):
            res[b].label = C.cast(labs[b][0], C.POINTER(C.c_int32))
        sets.append((res, labs))

    def run_sync(steps):
        res = sets[0][0]
        dev = 0.0
        t0 = time.perf_counter()
        for _ in range(steps):
            check(lib.urf_process_batch(det._ctx, ptrs, ns, B, res), "urf_process_batch")
            dev += lib.urf_last_device_ms(det._ctx)
        return time.perf_counter() - t0, dev

    def run_async(steps):
        dev = 0.0
        t0 = time.perf_counter()
        check(lib.urf_enqueue_batch(det._ctx, ptrs, ns, B, sets[0][0], None), "urf_enqueue_batch")
        for s in range(1, steps + 1):
            if s < steps:
                check(lib.urf_enqueue_batch(det._ctx, ptrs, ns, B, sets[s % 2][0], None), "urf_enqueue_batch")
            check(lib.urf_finish_batch(det._ctx), "urf_finish_batch")
            dev += lib.urf_last_device_ms(det._ctx)
        return time.perf_counter() - t0, dev

    run_sync(args.warmup)
    run_async(args.warmup)
    runs = {"process": [], "enqueue_finish": []}
    for r in range(args.repeats):
        for mode in (("process", "enqueue_finish") if r % 2 == 0 else ("enqueue_finish", "process")):
            wall, dev = (run_sync if mode == "process" else run_async)(args.steps)
            runs[mode].append((B * args.steps / wall, 1e3 * (wall - dev / 1e3) / args.steps, dev / args.steps))
    same = all(sets[0][1][b][1].tobytes() == sets[1][1][b][1].tobytes() for b in range(B))
    run_sync(1)                                              # set 0 from the synchronous call, set 1 from the last async one
    same &= all(sets[0][1][b][1].tobytes() == sets[1][1][b][1].tobytes() for b in range(B))
    med = {m: tuple(statistics.median(x[i] for x in v) for i in range(3)) for m, v in runs.items()}
    line = {"bench_async_batch": shape, "batch": B, "points_per_scan": n, "steps": args.steps, "labels_identical": same}
    for m, (rate, idle, dev) in med.items():
        line[m] = {"scans_per_sec": round(rate, 1), "idle_ms_per_batch": round(idle, 3), "device_ms_per_batch": round(dev, 3),
                   "runs_scans_per_sec": [round(x[0], 1) for x in runs[m]]}
    print(json.dumps(line), flush=True)
    rows.append((shape, med, same))
    det.close()
    for p, _ in keep + [x for s in sets for x in s[1]]:
        lib.urf_pinned_free(p)

print(f"\n| shape x {B} | process loop (scans/s) | enqueue/finish (scans/s) | ratio | idle ms/batch, process | idle ms/batch, enqueue/finish | labels identical |")
print("|---|---|---|---|---|---|---|")
for shape, med, same in rows:
    a, b = med["process"], med["enqueue_finish"]
    print(f"| {shape} | {a[0]:,.0f} | {b[0]:,.0f} | {b[0] / a[0]:.2f} | {a[1]:.3f} | {b[1]:.3f} | {same} |")

if args.old_lib:
    exe = build.build_tools()
    sh = SHAPES["C4"]
    K, n = 16, sh.rings * sh.cols
    tmp = tempfile.mkdtemp(prefix="urf_async_mq_")
    path = os.path.join(tmp, "urf_C4.bin")
    with open(path, "wb") as f:
        for k in range(K):
            f.write(np.ascontiguousarray(make_scan("C4", 500 + k), np.float32).tobytes())
    libs = {"old": os.path.abspath(args.old_lib), "new": os.path.join(ROOT, "urban_road_filter_b200")}
    for mode, name in ((2, "next_view_int32"), (3, "next_batch_int8")):      # tools/mq_bench modes
        runs = {k: [] for k in libs}
        for r in range(args.repeats):
            for k in (("old", "new") if r % 2 == 0 else ("new", "old")):
                out = subprocess.run([exe, path, str(n), str(K), "1", "4", str(args.mq_scans), "24", "16", "1", str(sh.channels),
                                      str(sh.interval), str(mode), "64"], check=True, capture_output=True, text=True,
                                     env={**os.environ, "LD_LIBRARY_PATH": libs[k]}).stdout
                runs[k].append(json.loads(out.strip().splitlines()[-1])["scans_per_sec"])
        med = {k: statistics.median(v) for k, v in runs.items()}
        print(json.dumps({"mq_1gpu_C4_" + name: {k: {"scans_per_sec": round(med[k], 1), "runs": [round(x, 1) for x in runs[k]]}
                                                 for k in libs}}), flush=True)
    os.remove(path)
    os.rmdir(tmp)

#!/usr/bin/env python
"""Throughput of one ingest stream carrying two LiDAR formats (OS1-64 scans, C2 of urban_road_filter_b200.synth,
131,072 points: 48-byte Ouster records and 32-byte Velodyne-like records in turn) over every visible GPU, three ways:
  (a) formats:  one formats mq (urf_mq_create_formats) with both formats in its table; producers submit by reference with
                urf_mq_submit_format_ref;
  (b) two mqs:  one record mq per format (urf_mq_create_cloud2) on the same GPUs, each fed its own half of the scans by
                reference (two device contexts, workers and slot sets per GPU, two consumers);
  (c) repack:   one float4 mq; producers repack each scan's records into (x, y, z, intensity) on the host, inside the timed
                region, and submit the points by reference.
All with `--producers` producer threads (each takes every producers-th scan), int8 label slots, `--slots` slots per device,
max_batch `--max-batch`, results taken with next_batch. The setups run alternately `--repeats` times; prints the median and
range of scans/s per setup, the device memory each setup's mqs took (free memory before and after creation) and their pinned
slot bytes, with the cards' name and power limit as nvidia-smi reports them.
usage: python scripts/bench_formats.py [--scans 3000] [--producers 4] [--repeats 3] [--gpus N]"""
import argparse
import ctypes as C
import os
import statistics
import subprocess
import sys
import threading
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np  # noqa: E402
import torch  # noqa: E402

from urban_road_filter_b200 import api  # noqa: E402
from urban_road_filter_b200.synth import SHAPES, make_scan  # noqa: E402

OS48, V32 = api.CloudFormat(48, 0, 4, 8, 16), api.CloudFormat(32, 0, 4, 8, 16)

ap = argparse.ArgumentParser()
ap.add_argument("--gpus", type=int, default=0, help="devices to shard over (default: every visible GPU)")
ap.add_argument("--shape", default="C2", help="synth shape of the scans")
ap.add_argument("--scans", type=int, default=3000)
ap.add_argument("--producers", type=int, default=4)
ap.add_argument("--slots", type=int, default=24)
ap.add_argument("--max-batch", type=int, default=16)
ap.add_argument("--repeats", type=int, default=3)
ap.add_argument("--unpack-batch", type=int, default=128, help="C2 scans per batch of the k_unpack_cloud2_batch timing (0: skip)")
args = ap.parse_args()
visible = torch.cuda.device_count()
if visible < 1:
    sys.exit("no GPU is visible")
devs = list(range(args.gpus or visible))
sh = SHAPES[args.shape]
n = sh.rings * sh.cols
K = 8                                                   # distinct scans per format, reused round-robin
pts = [np.ascontiguousarray(make_scan(args.shape, 700 + k), np.float32) for k in range(K)]


def records(p, f, seed):
    rec = np.random.default_rng(seed).integers(0, 256, (p.shape[0], f.point_step), dtype=np.uint8)
    for j, off in enumerate((f.off_x, f.off_y, f.off_z, f.off_intensity)):
        rec[:, off: off + 4] = p[:, j: j + 1].copy().view(np.uint8)
    return rec.reshape(-1)


def pinned_copy(a, lib, keep):
    p = lib.urf_pinned_alloc(a.nbytes)
    keep.append(p)
    dst = np.ctypeslib.as_array(C.cast(p, C.POINTER(C.c_uint8)), shape=(a.nbytes,))
    dst[:] = a.view(np.uint8).reshape(-1)
    return dst


lib = api.load_library()
pins = []
raws = {f: [pinned_copy(records(p, f, k), lib, pins) for k, p in enumerate(pts)] for f in (OS48, V32)}
fmt_of = [OS48 if s % 2 == 0 else V32 for s in range(args.scans)]    # the two sensors in turn
smi = subprocess.run(["nvidia-smi", "--query-gpu=index,name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
print("GPUs (index, name, power limit):\n" + smi)


def free_bytes():
    return sum(torch.cuda.mem_get_info(d)[0] for d in sorted(set(devs)))


def make(setup):
    """The mqs of a setup and the bytes of their pinned slots (records and int8 labels)."""
    kw = dict(max_points=n, slots_per_device=args.slots, max_batch=args.max_batch, label8=True)
    if setup == "formats":
        mqs = [api.MultiGpuQueue(devs, formats=[OS48, V32], **kw)]
        pinned = args.slots * len(devs) * n * (48 + 1)
    elif setup == "two mqs":
        mqs = [api.MultiGpuQueue(devs, records=OS48, **kw), api.MultiGpuQueue(devs, records=V32, **kw)]
        pinned = args.slots * len(devs) * n * (48 + 1 + 32 + 1)
    else:
        mqs = [api.MultiGpuQueue(devs, **kw)]
        pinned = args.slots * len(devs) * n * (16 + 1)
    return mqs, pinned


def submit_fn(setup, mqs):
    def submit(s):
        f = fmt_of[s]
        raw = raws[f][s % K]
        if setup == "formats":
            rc = mqs[0].submit_records(raw, n, tag=s, by_reference=True, fmt=0 if f == OS48 else 1)
        elif setup == "two mqs":
            rc = mqs[0 if f == OS48 else 1].submit_records(raw, n, tag=s, by_reference=True)
        else:                                           # the host repack the records mq saves
            rec = raw.reshape(n, f.point_step)
            xyzi = np.empty((n, 4), np.float32)
            for j, off in enumerate((f.off_x, f.off_y, f.off_z, f.off_intensity)):
                xyzi[:, j] = rec[:, off: off + 4].copy().view(np.float32).ravel()
            rc = mqs[0].submit(xyzi, tag=s, by_reference=True)
        assert rc == api.URF_OK, rc
    return submit


def run(setup):
    torch.cuda.synchronize()
    free0 = free_bytes()
    mqs, pinned = make(setup)
    dev_bytes = free0 - free_bytes()
    submit = submit_fn(setup, mqs)
    want = [sum(1 for s in range(args.scans) if setup != "two mqs" or (fmt_of[s] == OS48) == (i == 0)) for i in range(len(mqs))]

    def consume(i):
        got = 0
        while got < want[i]:
            out = mqs[i].next_batch(64, timeout_ms=600_000)
            assert out and all(r.status >= 0 for _, r in out)
            got += len(out)

    t0 = time.perf_counter()
    cons = [threading.Thread(target=consume, args=(i,)) for i in range(len(mqs))]
    prods = [threading.Thread(target=lambda p=p: [submit(s) for s in range(p, args.scans, args.producers)]) for p in range(args.producers)]
    for t in cons + prods:
        t.start()
    for t in prods + cons:
        t.join()
    dt = time.perf_counter() - t0
    for m in mqs:
        m.close()
        m.destroy()
    return args.scans / dt, dev_bytes, pinned, len(mqs) * len(devs)


SETUPS = ["formats", "two mqs", "repack"]
res = {s: [] for s in SETUPS}
mem = {}
for r in range(args.repeats):
    for s in (SETUPS if r % 2 == 0 else SETUPS[::-1]):  # alternated, so drift does not favour one setup
        sps, dev_bytes, pinned, ctxs = run(s)
        res[s].append(sps)
        mem[s] = (dev_bytes, pinned, ctxs)
        print(f"run {r} {s}: {sps:,.0f} scans/s", flush=True)
print(f"\n{args.scans} {args.shape} scans ({n} points; 48- and 32-byte records in turn), {args.producers} producers by reference, "
      f"{len(devs)} device(s) {devs}, {args.slots} slots per device, max_batch {args.max_batch}, int8 slots\n")
print("| setup | scans/s (median) | range | device contexts | device memory | pinned slots |")
print("|---|---|---|---|---|---|")
for s in SETUPS:
    v = res[s]
    dev_bytes, pinned, ctxs = mem[s]
    print(f"| {s} | {statistics.median(v):,.0f} | {min(v):,.0f}-{max(v):,.0f} | {ctxs} | {dev_bytes / 2**20:,.0f} MiB | {pinned / 2**20:,.0f} MiB |")


def unpack_ms(det, raws_, fmts, mixed, calls=7):
    """Median device time of k_unpack_cloud2_batch per batch call (torch.profiler), one-format or mixed entry point."""
    from torch.profiler import ProfilerActivity, profile
    call = (lambda: det.filtered_batch_mixed(raws_, fmts)) if mixed else (lambda: det.filtered_batch_records(raws_, *fmts[0]))
    call()
    per = []
    for _ in range(calls):
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            call()
            torch.cuda.synchronize()
        per.append(sum(e.device_time_total for e in prof.key_averages() if "k_unpack_cloud2_batch" in e.key) / 1000)
    return statistics.median(per), min(per), max(per)


if args.unpack_batch:
    B = args.unpack_batch
    c2 = [np.ascontiguousarray(make_scan("C2", 900 + k), np.float32) for k in range(B)]
    det = api.Detector(max_points=max(c.shape[0] for c in c2), max_batch=B, device=devs[0])
    one = [records(c, OS48, k) for k, c in enumerate(c2)]
    mix_f = [OS48 if k % 2 == 0 else V32 for k in range(B)]
    mix = [records(c, f, k) for k, (c, f) in enumerate(zip(c2, mix_f))]
    print(f"\nk_unpack_cloud2_batch, C2 x {B} (device ms per batch: median, min-max of 7 calls, torch.profiler):")
    for name, (r_, f_, m_) in {"one format (48-byte)": (one, [OS48] * B, False),
                               "mixed (48- and 32-byte in turn)": (mix, mix_f, True)}.items():
        med, lo, hi = unpack_ms(det, r_, f_, m_)
        print(f"  {name}: {med:.4f} ms ({lo:.4f}-{hi:.4f})")
    det.close()
for p in pins:
    lib.urf_pinned_free(p)

#!/usr/bin/env python
"""Throughput of the recorded-drive replay (urban_road_filter_b200.replay) on a seeded synthetic bag: two OS1-64 topics
(C2 of urban_road_filter_b200.synth, 131,072 points) as 48-byte Ouster records and two Velodyne-like topics (C1, VLP-16,
28,800 points) as 32-byte records, `--scans` messages per topic 0.1 s apart, written to `--out-dir` (default: a temporary
directory, removed at the end). Three runs, alternated `--repeats` times, each with the default ROI and with the full ROI:
  parse:   the producer's work alone: every message read from the bag index and decoded, no queue;
  discard: the replay with its outputs built (clouds packed, markers built) and then dropped;
  write:   the replay writing the output bag.
Prints one JSON line per run and setting: the median and range of scans/s, and the replay report's seconds of reading,
waiting on the queue, packing and writing, from which `bound` names the busiest stage, with the card's name and power
limit as nvidia-smi reports them.
usage: python scripts/bench_replay.py [--scans 50] [--repeats 3] [--devices 0] [--out-dir DIR]"""
import argparse
import json
import os
import shutil
import statistics
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402

from urban_road_filter_b200 import FULL_ROI, make_params, rosbag  # noqa: E402
from urban_road_filter_b200.replay import replay  # noqa: E402
from urban_road_filter_b200.synth import drive_bag  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--scans", type=int, default=50, help="messages per topic")
ap.add_argument("--repeats", type=int, default=3)
ap.add_argument("--devices", default="0")
ap.add_argument("--slots", type=int, default=16)
ap.add_argument("--batch", type=int, default=8)
ap.add_argument("--out-dir", help="where the bags go (default: a temporary directory, removed at the end)")
args = ap.parse_args()
if torch.cuda.device_count() < 1:
    sys.exit("no GPU is visible")
devices = tuple(int(d) for d in args.devices.split(","))
card = subprocess.run(["nvidia-smi", "--query-gpu=index,name,power.limit", "--format=csv,noheader"], capture_output=True,
                      text=True).stdout.strip().splitlines()
out_dir = args.out_dir or tempfile.mkdtemp(prefix="bench_replay_")
os.makedirs(out_dir, exist_ok=True)
src, dst = os.path.join(out_dir, "drive.bag"), os.path.join(out_dir, "replayed.bag")
sensors = [("/left_os1/os1_cloud_node/points", "C2", "ouster"), ("/right_os1/os1_cloud_node/points", "C2", "ouster"),
           ("/left_velodyne/velodyne_points", "C1", "velodyne"), ("/right_velodyne/velodyne_points", "C1", "velodyne")]
t0 = time.perf_counter()
n_msgs = drive_bag(src, sensors, args.scans, seed=2024)
print(json.dumps(dict(bag_messages=n_msgs, bag_bytes=os.path.getsize(src), generate_s=round(time.perf_counter() - t0, 2),
                      cards=card)), flush=True)


def parse_only():
    t0 = time.perf_counter()
    n = 0
    with rosbag.BagReader(src) as r:
        for topic, _, _, data in r.messages():
            msg = rosbag.decode_cloud2(data, topic)
            rosbag.cloud_format(msg, topic)
            n += 1
    return dict(scans=n, seconds=time.perf_counter() - t0, bound="host: bag parsing")


def run_replay(prm, out):
    rep = replay(src, out, devices=devices, slots=args.slots, batch=args.batch, params=prm)
    stages = dict(reading=rep.read_s, waiting=rep.wait_s, packing=rep.pack_s, writing=rep.write_s)
    busy = max(("reading", "packing", "writing"), key=stages.get)
    # the consumer waits on the queue whenever it outpaces the producer or the devices
    bound = ("queue (devices or producer)" if rep.wait_s > rep.pack_s + rep.write_s else f"host: {busy}")
    if os.path.exists(dst):
        os.remove(dst)
    return dict(scans=rep.total, seconds=rep.seconds, bound=bound, **{k: round(v, 3) for k, v in stages.items()})


settings = {"default_roi": make_params(), "full_roi": make_params(**FULL_ROI)}
runs = {"parse": lambda prm: parse_only(), "discard": lambda prm: run_replay(prm, None), "write": lambda prm: run_replay(prm, dst)}
replay(src, None, devices=devices, slots=args.slots, batch=args.batch, limit=32)        # warm-up: contexts, modules, page cache
results = {}
for rep_i in range(args.repeats):
    for sname, prm in settings.items():
        for rname, fn in runs.items():
            results.setdefault((sname, rname), []).append(fn(prm))
for (sname, rname), rs in results.items():
    rates = [r["scans"] / r["seconds"] for r in rs]
    last = rs[-1]
    print(json.dumps(dict(run=rname, setting=sname, scans=last["scans"], scans_per_s=round(statistics.median(rates), 1),
                          range=[round(min(rates), 1), round(max(rates), 1)], bound=last["bound"],
                          stages_s_last={k: last[k] for k in ("reading", "waiting", "packing", "writing") if k in last},
                          devices=list(devices), slots=args.slots, batch=args.batch, cards=card)), flush=True)
if not args.out_dir:
    shutil.rmtree(out_dir)

"""Cost of the reference tie order (urf_set_tie_order) on one GPU, device-resident batches (urf_enqueue_batch_device):
  * C2 x 128 tie-free scans: step time in the default and the reference order, alternated in one run;
  * C2 x 128 dual-return scans (every point with a second return at 2x range: every ring ties): step time in both orders,
    and the per-kernel times of k_sort_rings and k_lomuto_rings (CUDA events, urf_set_option(1, ...));
  * VLP-16 dual-return and duplicated-point scans (tests/tie_policy.py) x 128.
Prints one JSON line per measurement, the first one with the card's name and power limit read in the same run; --out
also writes them all to that file. usage: python scripts/bench_ties.py [--steps K] [--warmup W] [--rounds R] [--out F]"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from oracle.pyoracle import PortOracle  # noqa: E402
from urban_road_filter_b200 import FULL_ROI, UrfResult, api, make_params  # noqa: E402
from urban_road_filter_b200.synth import SHAPES, make_scan  # noqa: E402

import tie_policy as tp  # noqa: E402


def dual(pts):
    sec = pts.copy()
    sec[:, :3] *= np.float32(2.0)
    out = np.empty((2 * pts.shape[0], 4), np.float32)
    out[0::2], out[1::2] = pts, sec
    return out


class Batch:
    def __init__(self, clouds, prm):
        self.B = len(clouds)
        self.S = ((max(c.shape[0] for c in clouds) + 511) // 512) * 512
        self.det = api.Detector(max_points=self.S, max_batch=self.B, params=prm)
        self.x = torch.zeros((self.B, self.S, 4), dtype=torch.float32, device="cuda")
        for b, c in enumerate(clouds):
            self.x[b, : c.shape[0]] = torch.from_numpy(c).cuda()
        self.lab = torch.zeros((self.B, self.S), dtype=torch.int32, device="cuda")
        self.ns = (C.c_int * self.B)(*[c.shape[0] for c in clouds])
        self.outs = (UrfResult * self.B)()

    def step(self):
        d = self.det
        assert d.lib.urf_enqueue_batch_device(d._ctx, self.x.data_ptr(), self.S, self.ns, self.B, self.lab.data_ptr()) == 0

    def time(self, mode, steps, warmup):
        self.det.set_tie_order(mode)
        for _ in range(warmup):
            self.step()
        assert self.det.lib.urf_finish_batch_device(self.det._ctx, self.outs) == 0
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        st = torch.cuda.ExternalStream(self.det.lib.urf_stream(self.det._ctx))
        e0.record(st)
        for _ in range(steps):
            self.step()
        e1.record(st)
        assert self.det.lib.urf_finish_batch_device(self.det._ctx, self.outs) == 0
        e1.synchronize()
        return e0.elapsed_time(e1) / steps

    def kernels(self, mode, steps):
        d = self.det
        d.set_tie_order(mode)
        d.set_option(1, 1)
        acc = {}
        for _ in range(steps):
            self.step()
            assert d.lib.urf_finish_batch_device(d._ctx, self.outs) == 0
            for name, ms in d.kernel_times():
                acc[name] = acc.get(name, 0.0) + ms / steps
        d.set_option(1, 0)
        return acc


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--batch", type=int, default=128)
    ap.add_argument("--out", default=None, help="also write every line to this JSON file")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_ties.py measures on a CUDA device; none is visible")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    card = q.stdout.strip().splitlines()[0] if q.returncode == 0 else torch.cuda.get_device_name(0)
    lines = [{"card": card}]
    print(json.dumps(lines[0]), flush=True)
    sh = SHAPES["C2"]
    c2prm = make_params(channels=sh.channels, interval=sh.interval, **FULL_ROI)
    port = PortOracle()
    work = {
        "C2_tie_free": ([make_scan("C2", s) for s in range(a.batch)], c2prm),
        "C2_dual_return": ([dual(make_scan("C2", s)) for s in range(a.batch)], c2prm),
    }
    for name in ("dual_interleaved", "duplicates"):
        pts, prm = tp.CASES[name](port)
        work["VLP16_" + name] = ([pts] * a.batch, prm)
    for key, (clouds, prm) in work.items():
        bt = Batch(clouds, prm)
        t = {"input": [], "reference": []}
        for _ in range(a.rounds):                       # alternated in one run
            for mode in ("input", "reference"):
                t[mode].append(bt.time(mode, a.steps, a.warmup))
        rec = {"workload": key, "batch": a.batch, "points_per_scan": int(clouds[0].shape[0]),
               "ms_per_step": {m: sorted(v) for m, v in t.items()},
               "median_ms": {m: float(np.median(v)) for m, v in t.items()}}
        if key != "C2_tie_free":
            ks = bt.kernels("reference", max(2, a.steps // 4))
            rec["kernel_ms_reference"] = {k: round(v, 4) for k, v in ks.items() if k in ("k_sort_rings", "k_lomuto_rings", "k_label")}
        bt.det.close()
        lines.append(rec)
        print(json.dumps(rec), flush=True)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(lines, f, indent=1)


if __name__ == "__main__":
    main()

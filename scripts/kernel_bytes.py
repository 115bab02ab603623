#!/usr/bin/env python
"""Bytes each kernel of the path must move per step, and the rate that implies for measured kernel times.

  python scripts/kernel_bytes.py [--shape C2] [--batch 128] [--sample 2]            byte counts only (CPU)
  python scripts/kernel_bytes.py --shape C2 --batch 128 --bench LINE.json           + GB/s and share of 3.35 TB/s

The per-scan counts the byte models need (ROI points, registered rings, road points) come from the CPU oracle run on
the first --sample scans of the batch bench.py times (seeds 0, 1, ...) and are scaled to the batch. Every ROI point lies
in a star sector. The models count what each kernel reads and writes from DRAM once, as written in
urban_road_filter_b200/csrc/urf_kernels.cuh: per-point arrays at their element size, per-scan tables at their size.
They ignore re-reads that the code arranges to hit L1 / L2 (small tables, the threshold rows, lookup tables). Sector
sort and scan kernels are counted as if every sector were sorted whole: the near-first prefix is data-dependent, so
their rows are upper bounds.

--bench takes a line printed by `bench.py --no-cpu-baseline --no-e2e` (its `kernel_ms`) or by a full bench.py run
(`roofline.kernel_ms_per_step`). 3.35 TB/s is NVIDIA's data-sheet HBM3 bandwidth of the H100 SXM, not a measured peak.
"""
from __future__ import annotations

import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from urban_road_filter_b200 import FULL_ROI, make_params  # noqa: E402
from urban_road_filter_b200.synth import SHAPES, make_scan  # noqa: E402

HBM_DATASHEET_GBS = 3350.0      # NVIDIA H100 SXM data sheet, HBM3
CHUNK, RING_KEYS, SECT_KEYS, ELEV_BINS, DEG_BINS, T_STRIDE = 512, 256, 360, 4096, 361, 364


def scan_counts(shape: str, sample: int) -> dict:
    from oracle.pyoracle import PortOracle
    sh = SHAPES[shape]
    prm = make_params(channels=sh.channels, interval=sh.interval, **FULL_ROI)
    tot = {"n": 0, "roi": 0, "order": 0, "road": 0, "rings": 0}
    for seed in range(sample):
        pts = make_scan(shape, seed)
        r = PortOracle().run(pts, prm)
        tot["n"] += pts.shape[0]; tot["roi"] += r.n_roi; tot["order"] += r.n_order; tot["road"] += r.n_road; tot["rings"] += r.n_rings
    c = {k: v / sample for k, v in tot.items()}
    c["channels"] = sh.channels
    return c


def kernel_bytes(c: dict, batch: int) -> dict:
    """{kernel: (bytes per step, what is counted)}"""
    N, R, O, D, C = c["n"], c["roi"], c["order"], c["road"], c["channels"]
    T = -(-int(N) // CHUNK)
    hist = T * C * 4                                   # per-chunk ring histograms of a scan: one counter per channel
    per_scan = {
        "k_reset": (RING_KEYS * 28 + DEG_BINS * 20 + SECT_KEYS * 4 + (ELEV_BINS + 1) * 4 + C * DEG_BINS * 8,
                    "per-scan tables, first-index bins, curb bins"),
        "k_points": (N * (16 + 4 + 1 + 2) + R * 8, "in 16 + alpha 4 + mark 1 + sect 2 per point, az + d2 8 per ROI point"),
        "k_register": ((ELEV_BINS + 1) * (4 + 2) + RING_KEYS * 12, "first-index bins, lookup table, ring tables"),
        "k_assign": (N * (4 + 2) + hist, "alpha 4 + ringid 2 per point, histogram rows"),
        "k_scan_offsets": (2 * hist, "histogram rows read and rewritten"),
        "k_scatter": (N * (2 + 2 + 16) + O * 16 + R * 12 + hist,
                      "ringid 2 + sect 2 + in 16 per point, bpt 16 per ring point, sr + sz + sidx 12 per sector point, histogram rows"),
        "k_star_sort": (R * (4 + 4 + 8 + 4), "sr 4 + sz gather 4 + ssrz 8 + ssl 4 per sector point (whole sectors)"),
        "k_star_sort_big": (0, "work list only (empty at the bench shapes)"),
        "k_star_scan": (R * 8, "ssrz 8 per sector point (whole sectors)"),
        "k_star_refine": (0, "work list only"),
        "k_ring_detect4": (O * 16 + O * 1, "bpt 16 + mark 1 per ring point"),
        "k_tab1": (C * DEG_BINS * 8 * 2, "curb bins read, non-empty prefix counts"),
        "k_reach": (C * DEG_BINS * 2, "prefix counts"),
        "k_tab2": (2 * C * T_STRIDE * 4, "threshold tables written"),
        "k_label": (N * (2 + 4 + 4 + 1 + 4) + N / 32 + D * 16,
                    "ringid 2 + az 4 + d2 4 + mark 1 + label 4 per point, roadcnt, roadlist 16 per road point"),
        "k_markers1": (N / 32 + D * 16, "roadcnt, roadlist 16 per road point"),
    }
    return {k: (v * batch, what) for k, (v, what) in per_scan.items()}


def kernel_ms(line: dict) -> dict:
    if "kernel_ms" in line and isinstance(line["kernel_ms"], dict):
        return line["kernel_ms"]
    return line["roofline"]["kernel_ms_per_step"]


def main() -> int:
    ap = argparse.ArgumentParser()
    ap.add_argument("--shape", default="C2", choices=sorted(SHAPES))
    ap.add_argument("--batch", type=int, default=128)
    ap.add_argument("--sample", type=int, default=2, help="scans run through the CPU oracle for the per-scan counts")
    ap.add_argument("--bench", default="", help="file holding a bench.py JSON line (the last line that parses is used)")
    args = ap.parse_args()
    c = scan_counts(args.shape, args.sample)
    kb = kernel_bytes(c, args.batch)
    ms = {}
    if args.bench:
        for ln in open(args.bench):
            try:
                ms = kernel_ms(json.loads(ln))
            except (ValueError, KeyError, TypeError):
                pass
        if not ms:
            sys.exit(f"{args.bench}: no bench.py line with kernel times")
    print(f"{args.shape} x {args.batch}: {c['n']:.0f} points, {c['roi']:.0f} ROI, {c['order']:.0f} in rings, {c['road']:.0f} road "
          f"per scan (mean of {args.sample} oracle runs)")
    print(f"{'kernel':18s} {'MB/step':>9s} {'B/pt':>6s}" + (f" {'ms':>7s} {'GB/s':>7s} {'of 3.35 TB/s':>12s}" if ms else "") + "  counted")
    for k, (b, what) in sorted(kb.items(), key=lambda kv: -kv[1][0]):
        row = f"{k:18s} {b / 1e6:9.1f} {b / (c['n'] * args.batch):6.1f}"
        if ms:
            t = ms.get(k)
            row += f" {t:7.3f} {b / (t * 1e-3) / 1e9:7.0f} {b / (t * 1e-3) / 1e9 / HBM_DATASHEET_GBS:12.1%}" if t else f" {'-':>7s} {'-':>7s} {'-':>12s}"
        print(row + "  " + what)
    if ms:
        print(f"share: the rate over {HBM_DATASHEET_GBS / 1e3:.2f} TB/s, the H100 SXM data-sheet HBM3 bandwidth (not a measured peak)")
    return 0


if __name__ == "__main__":
    sys.exit(main())

#!/usr/bin/env python
"""Small asynchronous case for compute-sanitizer (memcheck, racecheck): two C1 batches of two scans each, with ring and
order, in pinned handles, enqueued back to back (slots 0 and 1), then a third into slot 0 while the second is in flight;
each result is compared with the synchronous call. No torch, so the sanitized process stays small.
usage: compute-sanitizer --tool memcheck python scripts/san_async.py"""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np  # noqa: E402
from urban_road_filter_b200 import FULL_ROI, api, make_params  # noqa: E402
from urban_road_filter_b200.synth import make_scan  # noqa: E402

a = [make_scan("C1", k, cols=1800 - 7 * k) for k in range(2)]
b = [make_scan("C1", 10 + k, order="ring", cols=1700 - 5 * k) for k in range(2)]
det = api.Detector(max_points=max(c.shape[0] for c in a + b), max_batch=2, params=make_params(**FULL_ROI), tie_order="reference")
want_a, want_b = det.filtered_batch(a), det.filtered_batch(b)
ha, hb, hc = (api.BatchHandle.of_clouds(c, True, True, False, pinned=True) for c in (a, b, a))
det.enqueue(ha)
det.enqueue(hb)
det.finish_batch()
det.enqueue(hc)
det.finish_batch()
det.finish_batch()
ok = True
for h, w in ((ha, want_a), (hb, want_b), (hc, want_a)):
    for g, e in zip(h.results, w):
        ok &= all(np.array_equal(getattr(g, f), getattr(e, f)) for f in ("label", "ring", "order", "ring_start", "vert"))
det.close()
print("san_async", "OK" if ok else "MISMATCH")
sys.exit(0 if ok else 1)

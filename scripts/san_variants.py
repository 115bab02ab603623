"""Small scans through every kernel path of the pipeline, for compute-sanitizer: both ring detectors (k_ring_detect4 at the
default curb_points, k_ring_detect at curb_points = 7), both marker searches (k_markers1, and k_markers_grid on a scan above
300,000 points), the single-stream order that per-kernel timing forces, the emission-order counting sort and its fallback,
the radius-tie path (restated std::sort by one thread), the registration repair inside k_scan_offsets, the lean and record
entries."""
import sys
sys.path.insert(0, ".")
import numpy as np
from urban_road_filter_b200 import api, make_params, FULL_ROI
from urban_road_filter_b200.synth import SHAPES, make_scan, random_cloud

prm = make_params(**FULL_ROI)
pts = make_scan("C1", 3)
det = api.Detector(max_points=30000, max_batch=4, params=prm)
base = det.filtered(pts)                                                         # k_ring_detect4, k_markers1, side stream
tie = pts.copy(); tie[1000:1300, :3] = tie[3000:3300, :3]                      # equal radii -> std::sort emulation
assert det.filtered(tie).flags & 2
assert det.filtered(random_cloud(5000, 5)).flags & 1                            # speculation refuted -> repair in k_scan_offsets
det.set_params(make_params(curb_points=7, **FULL_ROI)); det.filtered(pts)      # one-position-per-thread detector
det.set_params(prm)
rs = det.filtered_batch_records([np.ascontiguousarray(pts[:, :3]), np.ascontiguousarray(pts[:9000, :3])], 12, 0, 4, 8, -1, want_order=True)
assert np.array_equal(rs[0].label, base.label)
flat = make_scan("C1", 4).copy(); flat[:, 2] = -1.8                              # no edges: every sector refined
det.filtered(flat)
det.set_option(10, 28); rw = det.filtered(pts); det.set_option(10, 17)          # pivot too high for a prefix: whole-sector sorts
det.set_option(1, 1); r1s = det.filtered(pts); det.set_option(1, 0)              # per-kernel timing: everything on one stream
assert np.array_equal(rw.label, base.label) and np.array_equal(r1s.label, base.label)
assert np.array_equal(r1s.order, base.order) and np.array_equal(r1s.vert, base.vert)
det.close()
# OS1-64 sectors (364 points) are sorted near-first; in a flat / half-flat world the walks run off the prefix:
# k_star_refine (remainder sort behind the prefix + warp-wide resumed walk) on every / every other sector
det = api.Detector(max_points=131072, max_batch=1, params=prm)
big = make_scan("C2", 5)
ref = det.filtered(big)
for variant in ("flat", "half"):
    w = big.copy()
    w[(w[:, 0] < 0) if variant == "half" else slice(None), 2] = -1.8
    a = det.filtered(w)
    det.set_option(4, 0); b = det.filtered(w); det.set_option(4, 1)             # whole-sector sorting: same result
    assert np.array_equal(a.label, b.label) and np.array_equal(a.order, b.order), variant
det.close()
# 1,048,576 points: the marker search takes a grid of CTAs per scan (k_markers_grid<1> -> k_markers_grid<2> -> k_verts)
sh = SHAPES["C5"]
det = api.Detector(max_points=1_048_576, max_batch=1, params=make_params(channels=sh.channels, interval=sh.interval, **FULL_ROI))
r5 = det.filtered(make_scan("C5", 0))
assert r5.status == 0 and r5.n_vert > 0
flat5 = make_scan("C5", 1).copy(); flat5[:, 2] = -1.8                           # sectors of ~2,900 points refined: k_star_refine's CTA loop
assert det.filtered(flat5).status == 0
det.close()
print("ok")

"""Generates tests/golden/*.npz by running the UNMODIFIED reference (oracle/_ref/liburf_ref.so, built from the reference's
sources by `make -C oracle ref REF=<reference checkout>`) on seeded synthetic clouds. The fixtures are committed, so the
tests need neither the reference's sources nor its build.

    python tests/golden/make_golden.py                 # everything but the C5 fixtures
    python tests/golden/make_golden.py --only c5
    python tests/golden/make_golden.py --ref-checks    # tests/golden/ref/: the reference's outputs for the random-parameter
                                                       # draws of tests/test_oracle.py, the strips of tests/test_markers.py
                                                       # the tie clouds of tests/test_ties.py and the azimuth
                                                       # edge clouds of tests/test_azimuth_edges.py

Each fixture holds: params (cfg overrides), the input cloud (or, for big clouds, the generator recipe + sha256 of the
bytes it must produce), and what the reference published: per-point labels (recovered from the roi/road/curb clouds),
the road / curb / road_probably clouds as input-index lists in emission order, and the road_marker line strips with
simplification off (exact vertices) and with the cfg defaults.
"""
from __future__ import annotations

import hashlib
import json
import os
import platform
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from oracle.pyoracle import RefOracle  # noqa: E402
from urban_road_filter_b200 import FULL_ROI, make_params  # noqa: E402
from urban_road_filter_b200.synth import SHAPES, make_scan, random_cloud  # noqa: E402
from oracle.pyoracle import PortOracle  # noqa: E402
from util import MARKER_EPS, REF_DIR, cloud_digest, digest, random_param_case  # noqa: E402
import azimuth_edges  # noqa: E402
import tie_policy  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))

CASES = [
    # name, recipe, store_input, param overrides
    ("c1_full_s0", dict(kind="scan", shape="C1", seed=0, order="column"), True, dict(**FULL_ROI)),
    ("c1_default_ring_s1", dict(kind="scan", shape="C1", seed=1, order="ring"), True, dict()),
    ("c1_full_xonly", dict(kind="scan", shape="C1", seed=0, order="column"), False, dict(z_zero_method=0, star_shaped_method=0, **FULL_ROI)),
    ("c1_full_zonly", dict(kind="scan", shape="C1", seed=0, order="column"), False, dict(x_zero_method=0, star_shaped_method=0, **FULL_ROI)),
    ("c1_full_staronly_beam", dict(kind="scan", shape="C1", seed=0, order="column"), False, dict(x_zero_method=0, z_zero_method=0, starbeam_filter=1, **FULL_ROI)),
    ("c1_full_xdir1_cp3", dict(kind="scan", shape="C1", seed=0, order="column"), False, dict(xDirection=1, curb_points=3, beamZone=45.5, **FULL_ROI)),
    ("c1_full_noblind_cp12", dict(kind="scan", shape="C1", seed=0, order="column"), False, dict(blind_spots=0, curb_points=12, **FULL_ROI)),
    ("random5000_s1_ties", dict(kind="random", n=5000, seed=1), True, dict(**FULL_ROI)),
    ("random5000_s5_specfail", dict(kind="random", n=5000, seed=5), True, dict(**FULL_ROI)),
    ("tiny29", dict(kind="scan", shape="C1", seed=0, order="column", head=29), False, dict(**FULL_ROI)),
    ("c2_default_s0", dict(kind="scan", shape="C2", seed=0, order="column"), False, dict()),
    ("c2_full_ring_s1", dict(kind="scan", shape="C2", seed=1, order="ring"), False, dict(**FULL_ROI)),
    ("c3_full_s0", dict(kind="scan", shape="C3", seed=0, order="column"), False, dict(**FULL_ROI)),
    ("c4_full_s0", dict(kind="scan", shape="C4", seed=0, order="column"), False, dict(channels=128, interval=0.07, **FULL_ROI)),
    # BASELINE config 5 (256 rings x 4096 columns = 1,048,576 points) and its detector ablation. The reference needs 12.9 GB
    # for its channels x N array3D and about 80 s per call here (page faults + its O(n^2) ring sort): run with --only c5
    ("c5_full_s0", dict(kind="scan", shape="C5", seed=0, order="column"), False, dict(channels=256, interval=0.07, **FULL_ROI)),
    ("c5_full_staronly", dict(kind="scan", shape="C5", seed=0, order="column"), False, dict(channels=256, interval=0.07, x_zero_method=0, z_zero_method=0, **FULL_ROI)),
    ("c5_full_xonly", dict(kind="scan", shape="C5", seed=0, order="column"), False, dict(channels=256, interval=0.07, star_shaped_method=0, z_zero_method=0, **FULL_ROI)),
    ("c5_full_zonly", dict(kind="scan", shape="C5", seed=0, order="column"), False, dict(channels=256, interval=0.07, star_shaped_method=0, x_zero_method=0, **FULL_ROI)),
]


def cloud_from_recipe(rc: dict) -> np.ndarray:
    if rc["kind"] == "scan":
        pts = make_scan(rc["shape"], rc["seed"], order=rc["order"])
    else:
        pts = random_cloud(rc["n"], rc["seed"])
    if "head" in rc:
        pts = pts[: rc["head"]].copy()
    return pts


def strips_to_arrays(strips):
    meta = np.array([[s[0], s[1], s[2], len(s[3])] for s in strips], np.int32).reshape(-1, 4)
    pts = np.concatenate([s[3] for s in strips], 0) if strips else np.zeros((0, 3))
    return meta, pts.astype(np.float64)


def ref_checks():
    ref = RefOracle()
    os.makedirs(REF_DIR, exist_ok=True)
    draws = {}
    for seed in range(6):
        pts, prm = random_param_case(seed)
        r = ref.run(pts, prm)
        draws[str(seed)] = dict(cloud_sha256=cloud_digest(pts), published=r.published, label=digest(r.label),
                                road_ids=digest(r.road_ids), curb_ids=digest(r.curb_ids))
    with open(os.path.join(REF_DIR, "random_params.json"), "w") as f:
        json.dump(draws, f, indent=1, sort_keys=True)
        f.write("\n")
    strips = {}
    for seed in range(4):
        pts = make_scan("C1", 20 + seed)
        strips[f"s{seed}_cloud_sha256"] = cloud_digest(pts)
        for k, eps in enumerate(MARKER_EPS):
            r = ref.run(pts, make_params(poly_s_param=eps, **FULL_ROI), ghostcount=0)
            strips[f"s{seed}_e{k}_published"] = np.int32(r.markers_published)
            strips[f"s{seed}_e{k}_meta"], strips[f"s{seed}_e{k}_pts"] = strips_to_arrays(r.strips)
    np.savez_compressed(os.path.join(REF_DIR, "marker_strips.npz"), **strips)
    ref_ties(ref)
    ref_azimuth_edges(ref)


def ref_azimuth_edges(ref):
    """azimuth_edges.npz: per cloud of tests/azimuth_edges.py the points appended to its base scan (so the tests run
    exactly these points whatever libm the machine has; the base scan is checked by the cloud's sha256), what the
    reference published (labels, road / curb / road_probably input indices, as
    sha256) and its marker strips with simplification off."""
    port = PortOracle()
    meta, arrays = {}, {}
    for name, build in azimuth_edges.CASES.items():
        pts, prm = build(port)
        r = ref.run(pts, prm)
        meta[name] = dict(cloud_sha256=cloud_digest(pts), published=r.published, label=digest(r.label),
                          road_ids=digest(r.road_ids), curb_ids=digest(r.curb_ids), prob_ids=digest(r.prob_ids))
        prm.simple_poly_allow, prm.poly_z_avg_allow = 0, 0
        r = ref.run(pts, prm, ghostcount=0)
        meta[name]["markers_published"] = r.markers_published
        arrays[name + "_tail"] = pts[azimuth_edges.base_scan(name).shape[0]:]
        arrays[name + "_meta"], arrays[name + "_pts"] = strips_to_arrays(r.strips)
    np.savez_compressed(os.path.join(REF_DIR, "azimuth_edges.npz"), meta=json.dumps(meta, sort_keys=True), **arrays)


def ref_ties(ref):
    """ties.npz: per tie cloud of tests/tie_policy.py, what the reference published (labels, the road / curb /
    road_probably clouds as input indices, as sha256) and its marker strips with simplification off."""
    port = PortOracle()
    meta, arrays = {}, {}
    for name, build in tie_policy.CASES.items():
        pts, prm = build(port)
        r = ref.run(pts, prm)
        meta[name] = dict(cloud_sha256=cloud_digest(pts), published=r.published, label=digest(r.label),
                          road_ids=digest(r.road_ids), curb_ids=digest(r.curb_ids), prob_ids=digest(r.prob_ids))
        prm.simple_poly_allow, prm.poly_z_avg_allow = 0, 0
        r = ref.run(pts, prm, ghostcount=0)
        meta[name]["markers_published"] = r.markers_published
        arrays[name + "_meta"], arrays[name + "_pts"] = strips_to_arrays(r.strips)
    np.savez_compressed(os.path.join(REF_DIR, "ties.npz"), meta=json.dumps(meta, sort_keys=True), **arrays)


def main():
    if "--ref-checks" in sys.argv:
        return ref_checks()
    only = sys.argv[sys.argv.index("--only") + 1] if "--only" in sys.argv else ""      # name prefix; default: everything but c5
    ref = RefOracle()
    env = dict(machine=platform.machine(), libc=" ".join(platform.libc_ver()), python=platform.python_version(),
               numpy=np.__version__)
    for name, recipe, store, over in CASES:
        if (only and not name.startswith(only)) or (not only and name.startswith("c5")):
            continue
        pts = cloud_from_recipe(recipe)
        sha = hashlib.sha256(pts.tobytes()).hexdigest()
        r0 = ref.run(pts, make_params(simple_poly_allow=0, poly_z_avg_allow=0, **over), ghostcount=0)
        r1 = ref.run(pts, make_params(**over), ghostcount=3)
        assert np.array_equal(r0.label, r1.label)
        m0, p0 = strips_to_arrays(r0.strips)
        m1, p1 = strips_to_arrays(r1.strips)
        out = dict(meta=json.dumps(dict(name=name, recipe=recipe, params=over, sha256=sha, n=int(pts.shape[0]), env=env)),
                   published=np.int32(r0.published), label=r0.label.astype(np.int8), n_roi=np.int32(r0.n_roi),
                   road_ids=r0.road_ids, curb_ids=r0.curb_ids, prob_ids=r0.prob_ids,
                   strips_raw_meta=m0, strips_raw_pts=p0, strips_cfg_meta=m1, strips_cfg_pts=p1,
                   markers_published=np.int32(r0.markers_published), ghost_after=np.int32(r1.ghostcount))
        if store:
            out["cloud"] = pts
        np.savez_compressed(os.path.join(HERE, name + ".npz"), **out)
        print(f"{name:28s} n={pts.shape[0]:7d} published={r0.published} roi={r0.n_roi} road={r0.n_road} curb={r0.n_curb} "
              f"strips={len(r0.strips)} sha={sha[:12]}")


if __name__ == "__main__":
    main()

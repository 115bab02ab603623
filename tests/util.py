"""Shared helpers of the test-suite: golden fixtures, comparisons, the CPU model binding."""
from __future__ import annotations

import ctypes as C
import glob
import hashlib
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from oracle.pyoracle import OracleDebug  # noqa: E402
from urban_road_filter_b200 import FULL_ROI, UrfParams, UrfResult, make_params  # noqa: E402
from urban_road_filter_b200.ctypes_abi import URF_MAX_CHANNELS, URF_MAX_VERTS  # noqa: E402
from urban_road_filter_b200.synth import make_scan, random_cloud  # noqa: E402

GOLDEN_DIR = os.path.join(ROOT, "tests", "golden")
REF_DIR = os.path.join(GOLDEN_DIR, "ref")    # what the unmodified reference returned for the tests that compare with it directly
VERT_TOL = 1e-4     # metres: BASELINE.json north_star tolerance for curb-polyline vertices
MARKER_EPS = (0.05, 0.7, 3.0)                 # poly_s_param values of the marker-tail comparison (tests/test_markers.py)


def digest(a) -> str:
    """sha256 of an int32 array: stands in for reference outputs too large to store."""
    return hashlib.sha256(np.ascontiguousarray(a, np.int32).tobytes()).hexdigest()


def cloud_digest(pts) -> str:
    return hashlib.sha256(np.ascontiguousarray(pts, np.float32).tobytes()).hexdigest()


def random_param_case(seed: int):
    """Seeded random draw over the LidarFilters.cfg parameter ranges (cfg/LidarFilters.cfg:10-84) and its cloud."""
    rng = np.random.default_rng(100 + seed)
    pts = make_scan("C1", 10 + seed, order=("column", "ring")[seed % 2]) if seed % 3 else random_cloud(6000, seed, rings=12)
    prm = make_params(
        x_zero_method=int(rng.integers(0, 2)), z_zero_method=int(rng.integers(0, 2)), star_shaped_method=int(rng.integers(0, 2)),
        blind_spots=int(rng.integers(0, 2)), xDirection=int(rng.integers(0, 3)), interval=float(rng.uniform(0.05, 0.5)),
        curb_height=float(rng.uniform(0.01, 0.2)), curb_points=int(rng.integers(1, 12)), beamZone=float(rng.uniform(10, 100)),
        cylinder_deg_x=float(rng.uniform(90, 180)), cylinder_deg_z=float(rng.uniform(90, 180)),
        curb_slope_deg=float(rng.uniform(10, 90)), kdev_param=float(rng.uniform(0.5, 5)), kdist_param=float(rng.uniform(0.4, 10)),
        starbeam_filter=int(rng.integers(0, 2)), dmin_param=int(rng.integers(3, 30)),
        **(FULL_ROI if seed % 2 else dict(min_x=-20.0, max_x=40.0, min_y=-15.0, max_y=15.0, min_z=-3.0, max_z=1.0)))
    return pts, prm


HUGE_ROI = dict(min_x=-3e38, max_x=3e38, min_y=-3e38, max_y=3e38, min_z=-200.0, max_z=200.0)
SECTOR_RADII = (0.3, 2.5, 19.0, 190.0)


def _ulps(v, d):
    """float32 v moved by d ulps (d may be negative), elementwise; crosses zero through the signed subnormals."""
    v = np.asarray(v, np.float32)
    i = v.view(np.int32).astype(np.int64)
    o = np.where(i < 0, -(i & 0x7fffffff), i) + d                 # ordered integer: ... -1ulp, -0/+0, +1ulp ...
    return np.where(o < 0, (-o) | (1 << 31), o).astype(np.uint32).view(np.float32)


def sector_boundary_cloud(r: float, seed: int = 0, huge: bool = False) -> np.ndarray:
    """Points on a flat ring (z = -1.7) at planar radius r that put the star sector (star_shaped_search.cpp:164-173) on
    a knife edge: +-1..8 ulps of y (or x, whichever moves the angle more) around every integer-degree direction, around
    k +- 1e-3 degrees (the margin of the fast sector path, urf_logic.cuh star_sector_fast) +-3 ulps, points on both axes
    with +-0.0, at the 0/360 wrap (x > 0, y = -tiny) and with subnormal coordinates; with `huge`, points with |x| or
    |y| above 2^126 (need HUGE_ROI). Seeded shuffle: no ring is in azimuth order."""
    pts = []
    deg = np.arange(360, dtype=np.float64)
    for centre, spread in ((deg, range(-8, 9)), (deg + 1e-3, range(-3, 4)), (deg - 1e-3, range(-3, 4))):
        th = np.deg2rad(centre)
        x = (r * np.cos(th)).astype(np.float32)
        y = (r * np.sin(th)).astype(np.float32)
        along_y = np.abs(np.cos(th)) >= np.abs(np.sin(th))       # the angle is most sensitive to the smaller coordinate
        for d in spread:
            pts.append(np.stack([np.where(along_y, x, _ulps(x, d)), np.where(along_y, _ulps(y, d), y)], 1))
    tiny = np.float32(1e-30)
    sub = np.float32(1e-40)                                       # subnormal
    s = np.float32(r)
    special = [(s, 0.0), (s, -0.0), (-s, 0.0), (-s, -0.0), (0.0, s), (-0.0, s), (0.0, -s), (-0.0, -s),
               (s, -tiny), (s, -sub), (s, sub), (s, -np.float32(1e-45)), (s, _ulps(np.float32(0.0), -1)),
               (sub, sub), (-sub, sub), (sub, -sub), (-sub, -sub), (sub, np.float32(3e-41)), (np.float32(3e-41), -sub),
               (sub, s * np.float32(1e-3)), (-s * np.float32(1e-3), -sub)]
    pts.append(np.array(special, np.float32))
    if huge:
        big = np.float32(2.0 ** 126)
        hp = []
        for a, b in ((1.5, 0.01), (1.9, 1.3), (0.7, 1.99), (1.0, 1.0), (1.99, 1e-30), (3e-30, 1.7)):
            for sx, sy in ((1, 1), (-1, 1), (-1, -1), (1, -1)):
                hp.append((sx * a * big, sy * b * big))
                hp.append((sy * b * big, sx * a * big))
        hp += [(2.0 ** 127, 5.0), (-(2.0 ** 127), -5.0), (5.0, 2.0 ** 127), (-3.0, -(2.0 ** 127)), (1.5e38, 7.0)]
        pts.append(np.array(hp, np.float32))
    xy = np.concatenate(pts).astype(np.float32)
    out = np.zeros((xy.shape[0], 4), np.float32)
    out[:, :2] = xy
    out[:, 2] = -1.7
    out[:, 3] = 1.0
    return out[np.random.default_rng(seed).permutation(out.shape[0])]


_SCAN_CACHE: dict = {}


def cached_scan(shape, seed, order):
    """make_scan with a one-entry cache per (shape, seed, order): the four C5 fixtures share one 1M-point cloud."""
    key = (shape, seed, order)
    if key not in _SCAN_CACHE:
        if len(_SCAN_CACHE) > 3:
            _SCAN_CACHE.clear()
        _SCAN_CACHE[key] = make_scan(shape, seed, order=order)
    return _SCAN_CACHE[key]


def golden_names() -> list[str]:
    return sorted(os.path.splitext(os.path.basename(p))[0] for p in glob.glob(os.path.join(GOLDEN_DIR, "*.npz")))


class Golden:
    def __init__(self, name: str):
        z = np.load(os.path.join(GOLDEN_DIR, name + ".npz"))
        self.meta = json.loads(str(z["meta"]))
        self.name = name
        self.params_over = self.meta["params"]
        rc = self.meta["recipe"]
        if "cloud" in z.files:
            self.cloud = z["cloud"]
        else:
            self.cloud = cached_scan(rc["shape"], rc["seed"], rc["order"]) if rc["kind"] == "scan" else random_cloud(rc["n"], rc["seed"])
            if "head" in rc:
                self.cloud = self.cloud[: rc["head"]].copy()
        sha = hashlib.sha256(np.ascontiguousarray(self.cloud).tobytes()).hexdigest()
        assert sha == self.meta["sha256"], f"{name}: the synthetic generator no longer reproduces the fixture's input cloud"
        self.published = bool(z["published"])
        self.label = z["label"].astype(np.int32)
        self.road_ids, self.curb_ids, self.prob_ids = z["road_ids"], z["curb_ids"], z["prob_ids"]
        self.strips_raw = self._strips(z["strips_raw_meta"], z["strips_raw_pts"])
        self.strips_cfg = self._strips(z["strips_cfg_meta"], z["strips_cfg_pts"])
        self.markers_published = bool(z["markers_published"])
        self.ghost_after = int(z["ghost_after"])

    @staticmethod
    def _strips(meta, pts):
        out, k = [], 0
        for sid, act, red, cnt in meta:
            out.append((int(sid), int(act), int(red), pts[k: k + cnt]))
            k += cnt
        return out

    def params(self, **extra) -> UrfParams:
        return make_params(**{**self.params_over, **extra})


def assert_matches_golden(g: Golden, res, build_markers, check_order: bool = True):
    """res: anything with status/label/order/ring_start/n_rings/vert (PortResult, ScanResult, model result)."""
    if not g.published:
        assert res.status == 1, "reference published nothing (piece < 30)"
        return
    assert res.status == 0
    assert np.array_equal(res.label, g.label), f"{g.name}: labels differ at {np.nonzero(res.label != g.label)[0][:10]}"
    ties = bool(res.flags & 4)
    if check_order and res.order is not None and not ties:
        lab = res.label[res.order]
        assert np.array_equal(res.order[lab == 1], g.road_ids), "road cloud emission order"
        assert np.array_equal(res.order[lab == 2], g.curb_ids), "curb cloud emission order"
        prob = res.order[res.ring_start[10]: res.ring_start[11]] if res.n_rings > 10 else np.zeros(0, np.int32)
        assert np.array_equal(prob, g.prob_ids), "road_probably cloud"
    if ties:
        return   # reference order of equal azimuths comes from its unstable quicksort; vertices may legitimately differ
    # vertices, through the marker tail with simplification off: exact (x, y, z) of every strip point
    strips, _ = build_markers(g.params(simple_poly_allow=0, poly_z_avg_allow=0), res.vert, 0)
    compare_strips(strips, g.strips_raw, g.name + " raw strips")
    strips, ghost = build_markers(g.params(), res.vert, 3)
    compare_strips(strips, g.strips_cfg, g.name + " cfg strips")
    if g.markers_published:
        assert ghost == g.ghost_after


def compare_strips(mine, ref, what):
    assert len(mine) == len(ref), f"{what}: {len(mine)} strips vs {len(ref)}"
    for a, b in zip(mine, ref):
        assert a[0] == b[0] and a[1] == b[1], f"{what}: id/action {a[:3]} vs {b[:3]}"
        if a[1] == 2:
            continue      # DELETE markers carry no geometry
        assert a[2] == b[2], f"{what}: colour"
        assert a[3].shape == b[3].shape, f"{what}: strip {a[0]} has {a[3].shape[0]} points, reference {b[3].shape[0]}"
        assert np.all(np.abs(a[3] - b[3]) <= VERT_TOL), f"{what}: vertex off by {np.abs(a[3] - b[3]).max()} m"


def feq(a: np.ndarray, b: np.ndarray) -> bool:
    """bitwise float equality, any NaN == any NaN (x86 and the GPU produce different NaN bit patterns for 0/0)"""
    a = np.ascontiguousarray(a, np.float32)
    b = np.ascontiguousarray(b, np.float32)
    a = np.where(np.isnan(a), np.float32(np.nan), a)
    b = np.where(np.isnan(b), np.float32(np.nan), b)
    return a.shape == b.shape and np.array_equal(a.view(np.uint32), b.view(np.uint32))


def cloud2_records(pts, step, ox, oy, oz, oi, seed=0):
    """PointCloud2 record bytes of an (N, 4) cloud: x / y / z / intensity as float32 at the given byte offsets (oi < 0:
    none), seeded garbage in the other bytes of each `step`-byte record."""
    n = pts.shape[0]
    rec = np.random.default_rng(seed).integers(0, 256, (n, step), dtype=np.uint8)     # garbage in the other fields
    for k, off in enumerate((ox, oy, oz, oi)):
        if off >= 0:
            rec[:, off: off + 4] = pts[:, k: k + 1].copy().view(np.uint8)
    return rec.reshape(-1)


class ModelResult:
    pass


class CpuModel:
    """build/libmodel.so: the kernels' logic functions run sequentially on the CPU (tests/kat/model_check.cpp)."""

    def __init__(self):
        self.lib = C.CDLL(os.path.join(ROOT, "build", "libmodel.so"))
        self.lib.urf_model_run.restype = C.c_int
        self.lib.urf_model_run.argtypes = [C.c_void_p, C.c_int, C.POINTER(UrfParams), C.POINTER(UrfResult),
                                           C.POINTER(OracleDebug), C.c_int]

    def run(self, pts, prm, force_exact=0) -> ModelResult:
        pts = np.ascontiguousarray(pts, np.float32)
        n, m = pts.shape[0], max(pts.shape[0], 1)
        res = UrfResult()
        a = dict(label=np.full(m, -1, np.int32), ring=np.full(m, -1, np.int32), order=np.zeros(m, np.int32),
                 ring_start=np.zeros(URF_MAX_CHANNELS + 1, np.int32))
        for k, v in a.items():
            setattr(res, k, v.ctypes.data_as(C.POINTER(C.c_int32)))
        d = OracleDebug.arrays(n)
        dbg = OracleDebug(**{k: v.ctypes.data for k, v in d.items()})
        rc = self.lib.urf_model_run(pts.ctypes.data, n, C.byref(prm), C.byref(res), C.byref(dbg), force_exact)
        assert rc == 0, rc
        r = ModelResult()
        r.__dict__.update(a)
        r.__dict__.update(d)
        for f in ("status", "n_roi", "n_rings", "n_order", "n_road", "n_curb", "n_vert", "flags"):
            setattr(r, f, int(getattr(res, f)))
        for k in OracleDebug.PER_POINT:
            setattr(r, k, d[k][:n])
        r.label, r.ring, r.order = r.label[:n], r.ring[:n], r.order[: res.n_order]
        r.vert = np.ctypeslib.as_array(res.vert).reshape(URF_MAX_VERTS, 4)[: res.n_vert].copy()
        return r


_K = URF_MAX_CHANNELS


class ScanTab(C.Structure):
    """ctypes mirror of urf::ScanTab (urban_road_filter_b200/csrc/urf_device.cuh): the per-scan tables, debug item 8."""
    _fields_ = [("angle", C.c_float * _K), ("regidx", C.c_int * _K), ("regorder", C.c_int * _K), ("maxs", C.c_uint64 * _K),
                ("maxdist", C.c_uint32 * _K), ("A", C.c_double * _K), ("sect_start", C.c_int * 361), ("sect_cnt", C.c_int * 360),
                ("sect_cur", C.c_int * 360), ("nbig", C.c_int), ("nslow", C.c_int), ("biglist", C.c_uint16 * 360),
                ("slowlist", C.c_uint16 * 360), ("q", C.c_float * 4), ("reach", (C.c_int * 361) * 2),
                ("cutbest", C.c_uint64 * 361), ("dmax", C.c_uint32 * 361), ("best", C.c_uint64 * 361),
                ("sorted_len", C.c_int * 360), ("nrefine", C.c_int), ("pad_", C.c_int), ("refine", C.c_uint16 * 360),
                ("resume", (C.c_float * 4) * 360)]


class GpuDebug:
    """Stage intermediates of scan b of the detector's last call, re-indexed by input index like the oracle's debug run.
    The device keeps one mark for all three detectors, so there is no star_mark of its own."""

    def __init__(self, det, res, n, b=0):
        self.__dict__.update(res.__dict__ if hasattr(res, "__dict__") else {s: getattr(res, s) for s in res.__slots__})
        a = det.debug_fetch(b, 0, np.float32, n)
        self.alpha_v = np.where(a < 0, np.nan, a).astype(np.float32)
        in_ring = det.debug_fetch(b, 2, np.int16, n) >= 0
        self.az = np.where(in_ring, det.debug_fetch(b, 4, np.float32, n), np.float32(np.nan)).astype(np.float32)
        self.d2 = np.where(in_ring, det.debug_fetch(b, 5, np.float32, n), np.float32(np.nan)).astype(np.float32)
        self.star_mark = None
        self.det_label = np.where(in_ring, det.debug_fetch(b, 1, np.uint8, n).astype(np.int8), np.int8(-1)).astype(np.int8)
        self.sector = det.debug_fetch(b, 3, np.int16, n)[:n]
        size = det.lib.urf_debug_sizeof_tab()
        assert size == C.sizeof(ScanTab), f"ScanTab mirror is {C.sizeof(ScanTab)} bytes, the library's {size}"
        tab = ScanTab.from_buffer_copy(det.debug_fetch(b, 8, np.uint8, size).tobytes())
        self.tab = tab
        self.ring_angle = np.array(tab.angle, np.float32)
        self.max_dist = np.array(tab.maxdist, np.uint32).view(np.float32)
        self.q = np.array(tab.q, np.float32)
        self.A = np.array(tab.A, np.float64)
        self.reach = np.array(tab.reach, np.int32).reshape(2, 361)


def stage_diffs(o, m, n: int, check_order: bool = True) -> list[str]:
    """Names of the stages in which result m (model / GPU) differs from the oracle's debug run o. Stages m does not
    provide (attribute missing or None) are skipped.

    reach: the oracle writes -1 for window starts its loops skip (outside the loop range, or blind). Those entries are
    never read when labels are decided, and the device leaves them as it likes: k_tab1 sets every entry to n_rings,
    k_reach then overwrites the starts inside the loop range, blind or not. Only the entries the oracle defines (>= 0)
    are compared. A is compared for rings 1 .. n_rings - 1 (blind_spots.cpp:142 never uses A[0])."""
    bad = []
    if o.status != m.status:
        return ["status"]
    if o.status != 0:
        return bad
    for f in ("alpha_v", "az", "d2"):
        if getattr(m, f, None) is not None and not feq(getattr(o, f)[:n], getattr(m, f)[:n]):
            bad.append(f)
    for f in ("star_mark", "det_label", "sector"):
        if getattr(m, f, None) is not None and not np.array_equal(getattr(o, f)[:n], getattr(m, f)[:n]):
            bad.append(f)
    if getattr(m, "q", None) is not None and not feq(o.q, m.q):
        bad.append("q")
    R = o.n_rings
    if R != m.n_rings:
        bad.append("n_rings")
    else:
        for f in ("ring_angle", "max_dist"):
            if getattr(m, f, None) is not None and not feq(getattr(o, f)[:R], getattr(m, f)[:R]):
                bad.append(f)
        if getattr(m, "A", None) is not None and not np.array_equal(np.asarray(o.A[1:R]).view(np.uint64), np.asarray(m.A[1:R]).view(np.uint64)):
            bad.append("A")
        if getattr(m, "reach", None) is not None:
            defined = o.reach >= 0
            if not np.array_equal(o.reach[defined], m.reach[defined]):
                bad.append("reach")
    if m.ring is not None and not np.array_equal(o.ring, m.ring):
        bad.append("ring")
    if not np.array_equal(o.label, m.label):
        bad.append("label")
    if (o.n_roi, o.n_road, o.n_curb, o.n_order) != (m.n_roi, m.n_road, m.n_curb, m.n_order):
        bad.append("counts")
    if (o.flags & 2) != (m.flags & 2):
        bad.append("sector_tie_flag")
    ties = bool(o.flags & 4)
    if check_order and m.order is not None:
        if bool(m.flags & 4) != ties:
            bad.append("azimuth_tie_flag")
        if not ties and not np.array_equal(o.order, m.order):
            bad.append("order")
        if getattr(m, "ring_start", None) is not None and not np.array_equal(o.ring_start[: o.n_rings + 1], m.ring_start[: o.n_rings + 1]):
            bad.append("ring_start")
    if not ties and (o.n_vert != m.n_vert or not feq(o.vert, m.vert)):
        bad.append("vert")
    return bad

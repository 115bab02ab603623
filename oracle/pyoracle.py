"""ctypes bindings of the two CPU checkers. TEST INFRASTRUCTURE ONLY: importable from tests/, __graft_entry__.smoke()
and bench.py's cpu_baseline / --impl reference leg, never from the urban_road_filter_b200 package.

  RefOracle  -> oracle/_ref/liburf_ref.so : the unmodified reference sources (built by `make -C oracle ref`)
  PortOracle -> oracle/liburf_oracle.so   : our CPU restatement (urf_oracle.cpp)
"""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

from urban_road_filter_b200.ctypes_abi import URF_MAX_CHANNELS, URF_MAX_VERTS, UrfParams, UrfResult, UrfStrip

HERE = os.path.dirname(os.path.abspath(__file__))
REF_SO = os.path.join(HERE, "_ref", "liburf_ref.so")
PORT_SO = os.path.join(HERE, "liburf_oracle.so")


def _f32c(a: np.ndarray) -> np.ndarray:
    a = np.ascontiguousarray(a, dtype=np.float32)
    assert a.ndim == 2 and a.shape[1] == 4
    return a


class RefResult:
    pass


class RefOracle:
    """The reference's own Detector::filtered() (lidar_segmentation.cpp:95) behind a C entry."""

    def __init__(self, path: str = REF_SO):
        self.lib = C.CDLL(path)
        self.lib.urf_ref_run.restype = C.c_int
        self.lib.urf_ref_run.argtypes = [C.c_void_p, C.c_int, C.POINTER(UrfParams), C.c_void_p, C.c_void_p,
                                         C.c_void_p, C.c_void_p, C.POINTER(UrfStrip), C.c_int, C.c_void_p, C.c_int]
        self.lib.urf_ref_time.restype = C.c_double
        self.lib.urf_ref_time.argtypes = [C.c_void_p, C.c_int, C.POINTER(UrfParams), C.c_int]
        self.lib.urf_ref_set_ghostcount.argtypes = [C.c_int]
        self.lib.urf_ref_get_ghostcount.restype = C.c_int

    @staticmethod
    def available(path: str = REF_SO) -> bool:
        return os.path.exists(path)

    def run(self, pts: np.ndarray, prm: UrfParams, ghostcount: int | None = None) -> RefResult:
        pts = _f32c(pts)
        n = pts.shape[0]
        label = np.empty(n, np.int32)
        emit = np.empty(n, np.int32)
        prob = np.empty(n, np.int32)
        counts = np.zeros(8, np.int32)
        max_strips, max_sp = 1024, 4096
        strips = (UrfStrip * max_strips)()
        sp = np.zeros(3 * max_sp, np.float64)
        if ghostcount is not None:
            self.lib.urf_ref_set_ghostcount(ghostcount)
        rc = self.lib.urf_ref_run(pts.ctypes.data, n, C.byref(prm), label.ctypes.data, emit.ctypes.data,
                                  prob.ctypes.data, counts.ctypes.data, strips, max_strips, sp.ctypes.data, max_sp)
        assert rc == 0
        r = RefResult()
        r.published = bool(counts[0])
        r.label = label
        r.n_roi, r.n_road, r.n_curb, r.n_prob = (int(counts[i]) for i in (1, 2, 3, 4))
        r.road_ids = emit[: r.n_road].copy()
        r.curb_ids = emit[r.n_road: r.n_road + r.n_curb].copy()
        r.prob_ids = prob[: r.n_prob].copy()
        r.markers_published = bool(counts[7])
        r.strips = [(s.id, s.action, s.red, sp[3 * s.first: 3 * (s.first + s.count)].reshape(-1, 3).copy())
                    for s in strips[: counts[5]]]
        r.ghostcount = self.lib.urf_ref_get_ghostcount()
        return r

    def time(self, pts: np.ndarray, prm: UrfParams, repeat: int = 1) -> float:
        pts = _f32c(pts)
        return float(self.lib.urf_ref_time(pts.ctypes.data, pts.shape[0], C.byref(prm), repeat))


class PortResult:
    pass


class OracleDebug(C.Structure):
    """struct urf_oracle_debug (oracle/urf_oracle.cpp): per-point arrays are indexed by input point, the rest per ring /
    window start; NULL fields are not produced."""
    _fields_ = [("alpha_v", C.c_void_p), ("az", C.c_void_p), ("d2", C.c_void_p), ("star_mark", C.c_void_p),
                ("det_label", C.c_void_p), ("ring_angle", C.c_void_p), ("max_dist", C.c_void_p),
                ("sector", C.c_void_p), ("q", C.c_void_p), ("A", C.c_void_p), ("reach", C.c_void_p)]

    PER_POINT = ("alpha_v", "az", "d2", "star_mark", "det_label", "sector")

    @staticmethod
    def arrays(n: int) -> dict:
        """Host arrays for every field, holding the fill value entries keep when their stage does not reach them."""
        m = max(n, 1)
        return dict(alpha_v=np.full(m, np.nan, np.float32), az=np.full(m, np.nan, np.float32), d2=np.full(m, np.nan, np.float32),
                    star_mark=np.zeros(m, np.int8), det_label=np.full(m, -1, np.int8),
                    ring_angle=np.full(URF_MAX_CHANNELS, np.nan, np.float32), max_dist=np.full(URF_MAX_CHANNELS, np.nan, np.float32),
                    sector=np.full(m, -1, np.int16), q=np.full(4, np.nan, np.float32),
                    A=np.full(URF_MAX_CHANNELS, np.nan, np.float64), reach=np.full((2, 361), -1, np.int32))


class PortOracle:
    """Our CPU restatement of the path (oracle/urf_oracle.cpp): same outputs as urf_result plus intermediates."""

    def __init__(self, path: str = PORT_SO):
        self.lib = C.CDLL(path)
        self.lib.urf_oracle_run.restype = C.c_int
        self.lib.urf_oracle_run.argtypes = [C.c_void_p, C.c_int, C.POINTER(UrfParams), C.POINTER(UrfResult)]
        self.lib.urf_oracle_run_debug.restype = C.c_int
        self.lib.urf_oracle_run_debug.argtypes = [C.c_void_p, C.c_int, C.POINTER(UrfParams), C.POINTER(UrfResult),
                                                  C.POINTER(OracleDebug)]
        self.lib.urf_oracle_time.restype = C.c_double
        self.lib.urf_oracle_time.argtypes = [C.c_void_p, C.c_int, C.POINTER(UrfParams), C.c_int]

    @staticmethod
    def available(path: str = PORT_SO) -> bool:
        return os.path.exists(path)

    def run(self, pts: np.ndarray, prm: UrfParams, debug: bool = False) -> PortResult:
        pts = _f32c(pts)
        n = pts.shape[0]
        res = UrfResult()
        dbg = None
        if debug:
            dbg_arrays = OracleDebug.arrays(n)
            dbg = OracleDebug(**{k: v.ctypes.data for k, v in dbg_arrays.items()})
        label = np.full(max(n, 1), -1, np.int32)
        ring = np.full(max(n, 1), -1, np.int32)
        order = np.zeros(max(n, 1), np.int32)
        ring_start = np.zeros(URF_MAX_CHANNELS + 1, np.int32)
        res.label = label.ctypes.data_as(C.POINTER(C.c_int32))
        res.ring = ring.ctypes.data_as(C.POINTER(C.c_int32))
        res.order = order.ctypes.data_as(C.POINTER(C.c_int32))
        res.ring_start = ring_start.ctypes.data_as(C.POINTER(C.c_int32))
        if debug:
            rc = self.lib.urf_oracle_run_debug(pts.ctypes.data, n, C.byref(prm), C.byref(res), C.byref(dbg))
        else:
            rc = self.lib.urf_oracle_run(pts.ctypes.data, n, C.byref(prm), C.byref(res))
        assert rc == 0, rc
        r = PortResult()
        if debug:
            for k, v in dbg_arrays.items():
                setattr(r, k, v[:n] if k in OracleDebug.PER_POINT else v)
        r.status = res.status
        r.n_roi, r.n_rings, r.n_order = res.n_roi, res.n_rings, res.n_order
        r.n_road, r.n_curb, r.n_vert, r.flags = res.n_road, res.n_curb, res.n_vert, res.flags
        r.label = label[:n]
        r.ring = ring[:n]
        r.order = order[: res.n_order].copy()
        r.ring_start = ring_start[: res.n_rings + 1].copy()
        r.vert = np.ctypeslib.as_array(res.vert).reshape(URF_MAX_VERTS, 4)[: res.n_vert].copy()
        return r

    def time(self, pts: np.ndarray, prm: UrfParams, repeat: int = 1) -> float:
        pts = _f32c(pts)
        return float(self.lib.urf_oracle_time(pts.ctypes.data, pts.shape[0], C.byref(prm), repeat))

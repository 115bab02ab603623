"""ctypes binding of liburf_b200.so plus `Detector`, the host-side mirror of the reference node's interface
(`paramsCallback` -> set_params, `Detector::filtered` -> filtered / filtered_batch; src/main.cpp:4-34,
src/lidar_segmentation.cpp:95). There is no CPU fallback: loading fails loudly when the CUDA library is missing and
every compute call raises without a GPU."""
from __future__ import annotations

import collections
import ctypes as C
import os

import numpy as np

from .ctypes_abi import (UrfMqStats, QUEUE_FINISH_FN, QUEUE_PARAMS_FN, QUEUE_PROCESS_FN, URF_ERR_CLOSED, URF_ERR_TIMEOUT, URF_MAX_CHANNELS, URF_MAX_VERTS, URF_OK, URF_QUEUE_BLOCK,
                         URF_QUEUE_DROP_OLDEST, URF_QUEUE_LABEL8, URF_QUEUE_ORDER, URF_TOO_FEW_POINTS, UrfClouds, UrfCloud2Format, UrfParams,
                         UrfQueueStats, UrfResult, UrfStrip, make_params)

LIB_PATH = os.path.join(os.path.dirname(os.path.abspath(__file__)), "liburf_b200.so")

EXPORTS = ["urf_queue_next_batch", "urf_mq_next_batch", "urf_mq_create_label8", "urf_mq_create_with_label8", "urf_queue_next_view", "urf_queue_release_view", "urf_mq_next_view", "urf_queue_submit_ref", "urf_queue_create_cloud2", "urf_queue_submit_cloud2", "urf_mq_create", "urf_mq_create_with",
           "urf_mq_set_params", "urf_mq_submit", "urf_mq_submit_ref", "urf_mq_next", "urf_mq_get_stats", "urf_mq_close", "urf_mq_destroy",
           "urf_process_cloud2", "urf_process_cloud2_packed", "urf_pinned_alloc", "urf_pinned_free", "urf_queue_create",
           "urf_queue_create_with", "urf_queue_submit", "urf_queue_next", "urf_queue_get_stats", "urf_queue_close", "urf_queue_destroy",
           "urf_version", "urf_strerror", "urf_last_cuda_error", "urf_default_params", "urf_create", "urf_destroy",
           "urf_set_params", "urf_get_params", "urf_process", "urf_process_batch", "urf_process_batch_device",
           "urf_process_batch_xyz", "urf_process_cloud2_batch", "urf_enqueue_batch_device", "urf_enqueue_batch_device_ex", "urf_finish_batch_device", "urf_stream", "urf_last_device_ms",
           "urf_last_launch_count", "urf_build_markers", "urf_set_tie_order", "urf_get_tie_order", "urf_mq_set_tie_order",
           "urf_enqueue_batch", "urf_enqueue_cloud2_batch", "urf_finish_batch", "urf_queue_create_with_async",
           "urf_set_params_next", "urf_queue_update_params", "urf_mq_update_params", "urf_queue_set_params_hook",
           "urf_mq_set_params_hook", "urf_mq_create_policy", "urf_mq_create_with_policy", "urf_queue_submit_cloud2_ref",
           "urf_queue_create_cloud2_with", "urf_mq_create_cloud2", "urf_mq_create_cloud2_with", "urf_mq_submit_cloud2",
           "urf_mq_submit_cloud2_ref", "urf_process_cloud2_batch_mixed", "urf_enqueue_cloud2_batch_mixed", "urf_queue_create_formats",
           "urf_queue_create_formats_with", "urf_queue_submit_format", "urf_queue_submit_format_ref", "urf_mq_create_formats",
           "urf_mq_create_formats_with", "urf_mq_submit_format", "urf_mq_submit_format_ref"]

# One PointCloud2 record format (include/urf.h urf_cloud2_format): what a message's point_step and `fields` give. A float4 scan
# is CloudFormat(16, 0, 4, 8, 12).
CloudFormat = collections.namedtuple("CloudFormat", "point_step off_x off_y off_z off_intensity")
FLOAT4_FORMAT = CloudFormat(16, 0, 4, 8, 12)


def _format_array(formats):
    """A ctypes urf_cloud2_format array of `formats` (CloudFormat or 5-tuples)."""
    return (UrfCloud2Format * len(formats))(*[UrfCloud2Format(*(int(v) for v in f)) for f in formats])

# urf_set_tie_order modes (include/urf.h): equal azimuths inside a ring in input order, or in the reference's Lomuto order
TIE_ORDERS = {"input": 0, "reference": 1}

_lib = None


class UrfError(RuntimeError):
    def __init__(self, code: int, where: str, detail: str = ""):
        self.code = code
        super().__init__(f"{where}: urf error {code}" + (f" ({detail})" if detail else ""))


def load_library(path: str = LIB_PATH) -> C.CDLL:
    """Loads the CUDA library. Raises if it has not been built — there is deliberately no fallback."""
    global _lib
    if _lib is not None and path == LIB_PATH:
        return _lib
    if not os.path.exists(path):
        raise FileNotFoundError(f"{path} is missing: run `python -c 'import __graft_entry__ as g; g.build()'` "
                                "(urban_road_filter_b200 has no CPU fallback)")
    lib = C.CDLL(path)
    vp, ip = C.c_void_p, C.c_int
    lib.urf_version.restype = ip
    lib.urf_strerror.restype = C.c_char_p
    lib.urf_strerror.argtypes = [ip]
    lib.urf_last_cuda_error.restype = C.c_char_p
    lib.urf_last_cuda_error.argtypes = [vp]
    lib.urf_default_params.argtypes = [C.POINTER(UrfParams)]
    lib.urf_create.argtypes = [C.POINTER(vp), ip, ip, ip]
    lib.urf_destroy.argtypes = [vp]
    lib.urf_set_params.argtypes = [vp, C.POINTER(UrfParams)]
    lib.urf_set_params_next.argtypes = [vp, C.POINTER(UrfParams)]
    lib.urf_get_params.argtypes = [vp, C.POINTER(UrfParams)]
    lib.urf_set_option.argtypes = [vp, ip, ip]
    lib.urf_set_tie_order.argtypes = [vp, ip]
    lib.urf_get_tie_order.argtypes = [vp, C.POINTER(ip)]
    lib.urf_mq_set_tie_order.argtypes = [vp, ip]
    lib.urf_process.argtypes = [vp, vp, ip, C.POINTER(UrfResult)]
    lib.urf_process_batch.argtypes = [vp, C.POINTER(vp), C.POINTER(ip), ip, C.POINTER(UrfResult)]
    lib.urf_process_cloud2.argtypes = [vp, vp, ip, ip, ip, ip, ip, C.POINTER(UrfResult)]
    lib.urf_process_cloud2_packed.argtypes = [vp, vp, ip, ip, ip, ip, ip, ip, C.POINTER(UrfResult), C.POINTER(UrfClouds)]
    lib.urf_process_batch_xyz.argtypes = [vp, C.POINTER(vp), C.POINTER(ip), ip, C.POINTER(UrfResult), C.POINTER(vp)]
    lib.urf_process_cloud2_batch.argtypes = [vp, C.POINTER(vp), C.POINTER(ip), ip, ip, ip, ip, ip, ip, C.POINTER(UrfResult), C.POINTER(vp)]
    lib.urf_enqueue_batch.argtypes = [vp, C.POINTER(vp), C.POINTER(ip), ip, C.POINTER(UrfResult), C.POINTER(vp)]
    lib.urf_enqueue_cloud2_batch.argtypes = [vp, C.POINTER(vp), C.POINTER(ip), ip, ip, ip, ip, ip, ip, C.POINTER(UrfResult), C.POINTER(vp)]
    lib.urf_finish_batch.argtypes = [vp]
    lib.urf_process_batch_device.argtypes = [vp, vp, ip, C.POINTER(ip), ip, vp, C.POINTER(UrfResult)]
    lib.urf_enqueue_batch_device.argtypes = [vp, vp, ip, C.POINTER(ip), ip, vp]
    lib.urf_enqueue_batch_device_ex.argtypes = [vp, vp, ip, C.POINTER(ip), ip, vp, vp]
    lib.urf_finish_batch_device.argtypes = [vp, C.POINTER(UrfResult)]
    lib.urf_stream.restype = vp
    lib.urf_stream.argtypes = [vp]
    lib.urf_last_device_ms.restype = C.c_float
    lib.urf_last_device_ms.argtypes = [vp]
    lib.urf_last_launch_count.argtypes = [vp]
    lib.urf_build_markers.argtypes = [C.POINTER(UrfParams), vp, ip, C.POINTER(ip), C.POINTER(UrfStrip), ip, vp, ip,
                                      C.POINTER(ip)]
    lib.urf_pinned_alloc.restype = vp
    lib.urf_pinned_alloc.argtypes = [C.c_size_t]
    lib.urf_pinned_free.restype = None
    lib.urf_pinned_free.argtypes = [vp]
    lib.urf_queue_create.argtypes = [C.POINTER(vp), vp, ip, ip, ip, ip]
    lib.urf_queue_create_with.argtypes = [C.POINTER(vp), QUEUE_PROCESS_FN, vp, ip, ip, ip, ip]
    lib.urf_queue_create_with_async.argtypes = [C.POINTER(vp), QUEUE_PROCESS_FN, QUEUE_FINISH_FN, vp, ip, ip, ip, ip]
    lib.urf_queue_submit.argtypes = [vp, vp, ip, C.c_uint64, ip]
    lib.urf_queue_next.argtypes = [vp, C.POINTER(C.c_uint64), C.POINTER(UrfResult), ip]
    lib.urf_queue_get_stats.argtypes = [vp, C.POINTER(UrfQueueStats)]
    lib.urf_queue_close.restype = None
    lib.urf_queue_close.argtypes = [vp]
    lib.urf_queue_destroy.restype = None
    lib.urf_queue_destroy.argtypes = [vp]
    lib.urf_queue_submit_ref.argtypes = [vp, vp, ip, C.c_uint64, ip]
    lib.urf_queue_create_cloud2.argtypes = [C.POINTER(vp), vp, ip, ip, ip, ip, ip, ip, ip, ip, ip]
    lib.urf_queue_submit_cloud2.argtypes = [vp, vp, ip, C.c_uint64, ip]
    lib.urf_queue_submit_cloud2_ref.argtypes = [vp, vp, ip, C.c_uint64, ip]
    lib.urf_queue_create_cloud2_with.argtypes = [C.POINTER(vp), QUEUE_PROCESS_FN, vp, ip, ip, ip, ip, ip, ip, ip, ip, ip]
    lib.urf_mq_create.argtypes = [C.POINTER(vp), C.POINTER(ip), ip, ip, ip, ip, C.POINTER(UrfParams)]
    lib.urf_mq_create_with.argtypes = [C.POINTER(vp), QUEUE_PROCESS_FN, C.POINTER(vp), ip, ip, ip, ip]
    lib.urf_mq_set_params.argtypes = [vp, C.POINTER(UrfParams)]
    lib.urf_queue_update_params.argtypes = [vp, C.POINTER(UrfParams)]
    lib.urf_mq_update_params.argtypes = [vp, C.POINTER(UrfParams)]
    lib.urf_queue_set_params_hook.argtypes = [vp, QUEUE_PARAMS_FN]
    lib.urf_mq_set_params_hook.argtypes = [vp, QUEUE_PARAMS_FN]
    lib.urf_mq_submit.argtypes = [vp, vp, ip, C.c_uint64, ip]
    lib.urf_mq_submit_ref.argtypes = [vp, vp, ip, C.c_uint64, ip]
    lib.urf_mq_next.argtypes = [vp, C.POINTER(C.c_uint64), C.POINTER(UrfResult), ip]
    lib.urf_mq_get_stats.argtypes = [vp, C.POINTER(UrfMqStats)]
    lib.urf_mq_create_label8.argtypes = [C.POINTER(vp), C.POINTER(ip), ip, ip, ip, ip, C.POINTER(UrfParams)]
    lib.urf_mq_create_with_label8.argtypes = [C.POINTER(vp), QUEUE_PROCESS_FN, C.POINTER(vp), ip, ip, ip, ip]
    lib.urf_mq_create_policy.argtypes = [C.POINTER(vp), C.POINTER(ip), ip, ip, ip, ip, C.POINTER(UrfParams), ip]
    lib.urf_mq_create_with_policy.argtypes = [C.POINTER(vp), QUEUE_PROCESS_FN, C.POINTER(vp), ip, ip, ip, ip, ip]
    lib.urf_mq_create_cloud2.argtypes = [C.POINTER(vp), C.POINTER(ip), ip, ip, ip, ip, C.POINTER(UrfParams), ip, ip, ip, ip, ip, ip]
    lib.urf_mq_create_cloud2_with.argtypes = [C.POINTER(vp), QUEUE_PROCESS_FN, C.POINTER(vp), ip, ip, ip, ip, ip, ip, ip, ip, ip, ip]
    lib.urf_mq_submit_cloud2.argtypes = [vp, vp, ip, C.c_uint64, ip]
    lib.urf_mq_submit_cloud2_ref.argtypes = [vp, vp, ip, C.c_uint64, ip]
    fp = C.POINTER(UrfCloud2Format)
    lib.urf_process_cloud2_batch_mixed.argtypes = [vp, C.POINTER(vp), C.POINTER(ip), fp, ip, C.POINTER(UrfResult), C.POINTER(vp)]
    lib.urf_enqueue_cloud2_batch_mixed.argtypes = [vp, C.POINTER(vp), C.POINTER(ip), fp, ip, C.POINTER(UrfResult), C.POINTER(vp)]
    lib.urf_queue_create_formats.argtypes = [C.POINTER(vp), vp, ip, ip, ip, ip, fp, ip]
    lib.urf_queue_create_formats_with.argtypes = [C.POINTER(vp), QUEUE_PROCESS_FN, vp, ip, ip, ip, ip, fp, ip]
    lib.urf_mq_create_formats.argtypes = [C.POINTER(vp), C.POINTER(ip), ip, ip, ip, ip, C.POINTER(UrfParams), ip, fp, ip]
    lib.urf_mq_create_formats_with.argtypes = [C.POINTER(vp), QUEUE_PROCESS_FN, C.POINTER(vp), ip, ip, ip, ip, ip, fp, ip]
    for name in ("urf_queue_submit_format", "urf_queue_submit_format_ref", "urf_mq_submit_format", "urf_mq_submit_format_ref"):
        getattr(lib, name).argtypes = [vp, ip, vp, ip, C.c_uint64, ip]
    batch_args = [vp, ip, C.POINTER(C.c_uint64), C.POINTER(C.c_int32), C.POINTER(UrfResult), C.POINTER(vp), ip]
    lib.urf_queue_next_batch.argtypes = batch_args
    lib.urf_queue_next_view.argtypes = [vp, C.POINTER(C.c_uint64), C.POINTER(UrfResult), C.POINTER(vp), ip]
    lib.urf_mq_next_view.argtypes = [vp, C.POINTER(C.c_uint64), C.POINTER(UrfResult), C.POINTER(vp), ip]
    lib.urf_queue_release_view.argtypes = [vp]
    lib.urf_queue_release_view.restype = None
    lib.urf_mq_next_batch.argtypes = batch_args
    lib.urf_mq_close.argtypes = [vp]
    lib.urf_mq_close.restype = None
    lib.urf_mq_destroy.argtypes = [vp]
    lib.urf_mq_destroy.restype = None
    lib.urf_test_math.argtypes = [ip, ip, vp, vp, vp, ip]
    lib.urf_debug_fetch.argtypes = [vp, ip, ip, vp, C.c_size_t]
    lib.urf_debug_sizeof_tab.restype = C.c_size_t
    lib.urf_profile_count.argtypes = [vp]
    lib.urf_profile_slots.argtypes = [vp]
    lib.urf_profile_get.argtypes = [vp, ip, ip, C.POINTER(C.c_char_p), C.POINTER(C.c_float)]
    if path == LIB_PATH:
        _lib = lib
    return lib


class ScanResult:
    """Per-scan output of the path (urf_result, include/urf.h)."""
    __slots__ = ("status", "n_in", "n_roi", "n_rings", "n_order", "n_road", "n_curb", "n_vert", "flags", "params_gen", "label",
                 "ring", "order", "ring_start", "vert")

    @property
    def published(self) -> bool:
        return self.status == URF_OK

    def cloud_indices(self, which: str) -> np.ndarray:
        """Input indices of the `road` / `curb` / `road_probably` / `roi` clouds in the reference's emission order
        (lidar_segmentation.cpp:354-367,605-608,620)."""
        if which == "roi":
            return np.nonzero(self.label >= 0)[0].astype(np.int32)
        if self.order is None:
            raise ValueError("emission order was not requested")
        if which == "road_probably":
            if self.n_rings <= 10:
                return np.zeros(0, np.int32)
            return self.order[self.ring_start[10]: self.ring_start[11]]
        lab = self.label[self.order]
        return self.order[lab == (1 if which == "road" else 2)]


def _scan_result(res: UrfResult, label, ring=None, order=None, ring_start=None) -> ScanResult:
    """ScanResult of a filled urf_result: `label` and `ring` as given, `order` / `ring_start` (the caller's whole buffers, or
    None) cut to n_order / n_rings + 1 entries and copied, the vertices copied."""
    r = ScanResult()
    for f in ("status", "n_in", "n_roi", "n_rings", "n_order", "n_road", "n_curb", "n_vert", "flags", "params_gen"):
        setattr(r, f, int(getattr(res, f)))
    r.label, r.ring = label, ring
    r.order = None if order is None else order[: r.n_order].copy()
    r.ring_start = None if ring_start is None else ring_start[: r.n_rings + 1].copy()
    r.vert = np.ctypeslib.as_array(res.vert).reshape(URF_MAX_VERTS, 4)[: r.n_vert].copy()
    return r


def build_markers(prm: UrfParams, vert: np.ndarray, ghostcount: int = 0):
    """Marker tail (lidar_segmentation.cpp:371-598). Returns (strips, ghostcount'): strips = [(id, action, red, xyz[n,3])]."""
    lib = load_library()
    vert = np.ascontiguousarray(vert, np.float32).reshape(-1, 4)
    strips = (UrfStrip * 1024)()
    pts = np.zeros(3 * 4096, np.float64)
    gc = C.c_int(ghostcount)
    npnt = C.c_int(0)
    ns = lib.urf_build_markers(C.byref(prm), vert.ctypes.data, vert.shape[0], C.byref(gc), strips, 1024,
                               pts.ctypes.data, 4096, C.byref(npnt))
    if ns < 0:
        raise UrfError(ns, "urf_build_markers")
    out = [(s.id, s.action, s.red, pts[3 * s.first: 3 * (s.first + s.count)].reshape(-1, 3).copy()) for s in strips[:ns]]
    return out, gc.value


class BatchHandle:
    """The inputs, arguments and result buffers of one host-buffer batch call. They stay referenced here until the call has
    finished; `results` (list of ScanResult) is set by collect(), which Detector.finish_batch calls for an enqueued batch.
    step == 0: float4 scans; step > 0: PointCloud2 records of `step` bytes with x / y / z / intensity at `offs`.
    pinned: the inputs are copied into, and the results land in, page-locked memory (urf_pinned_alloc), so an enqueued
    batch's copies run asynchronously; a copy from or to pageable memory makes the enqueue wait for it. Allocating
    page-locked memory can wait for the device: build handles before enqueueing if batches are to overlap. A handle can be
    enqueued again once it is finished (collect copies the results out); its page-locked memory is freed by free() or when
    the handle is dropped. want_label=False: no label buffers (a call whose caller does not read the labels). formats (one
    CloudFormat per scan, or None): a batch of mixed record formats (urf_*_cloud2_batch_mixed); step and offs are then unused."""

    def __init__(self, inputs, ns, want_ring: bool, want_order: bool, label8: bool, step: int = 0, offs=(0, 4, 8, -1),
                 pinned: bool = False, want_label: bool = True, formats=None):
        B = len(inputs)
        self.lib = load_library()
        self.step, self.offs, self.pinned = step, tuple(offs), pinned
        self.fmts = None if formats is None else _format_array(formats)
        self._pins = []
        self.inputs = [self._array(a) for a in inputs] if pinned else inputs
        self.ptrs = (C.c_void_p * B)(*[a.ctypes.data for a in self.inputs])
        self.ns = (C.c_int * B)(*ns)
        self.res = (UrfResult * B)()
        self.l8 = (C.c_void_p * B)() if label8 else None
        self.bufs = []
        self.results = None
        for b, n in enumerate(ns):
            m = max(n, 1)
            lab = self._array(np.full(m, -1, np.int8 if label8 else np.int32)) if want_label else None
            ring = self._array(np.full(m, -1, np.int32)) if want_ring else None
            order = self._array(np.zeros(m, np.int32)) if want_order else None
            rs = self._array(np.zeros(URF_MAX_CHANNELS + 1, np.int32))
            if lab is None:
                pass
            elif label8:
                self.l8[b] = lab.ctypes.data
            else:
                self.res[b].label = lab.ctypes.data_as(C.POINTER(C.c_int32))
            if want_ring:
                self.res[b].ring = ring.ctypes.data_as(C.POINTER(C.c_int32))
            if want_order:
                self.res[b].order = order.ctypes.data_as(C.POINTER(C.c_int32))
            self.res[b].ring_start = rs.ctypes.data_as(C.POINTER(C.c_int32))
            self.bufs.append((lab, ring, order, rs))

    def _array(self, a: np.ndarray) -> np.ndarray:
        """`a` itself, or with `pinned` a page-locked copy of it."""
        if not self.pinned:
            return a
        p = self.lib.urf_pinned_alloc(max(a.nbytes, 1))
        if not p:
            raise MemoryError("urf_pinned_alloc failed")
        self._pins.append(p)
        dst = np.ctypeslib.as_array(C.cast(p, C.POINTER(C.c_uint8)), shape=(max(a.nbytes, 1),))[: a.nbytes].view(a.dtype).reshape(a.shape)
        dst[...] = a
        return dst

    @classmethod
    def of_clouds(cls, clouds, want_ring: bool, want_order: bool, label8: bool, pinned: bool = False) -> "BatchHandle":
        arrs = [np.ascontiguousarray(c, np.float32).reshape(-1, 4) for c in clouds]
        return cls(arrs, [a.shape[0] for a in arrs], want_ring, want_order, label8, pinned=pinned)

    @classmethod
    def of_records(cls, records, point_step: int, off_x: int, off_y: int, off_z: int, off_intensity: int, want_ring: bool,
                   want_order: bool, label8: bool, pinned: bool = False) -> "BatchHandle":
        raws = [np.ascontiguousarray(r).view(np.uint8).reshape(-1) for r in records]
        return cls(raws, [r.size // point_step for r in raws], want_ring, want_order, label8, point_step,
                   (off_x, off_y, off_z, off_intensity), pinned)

    @classmethod
    def of_mixed(cls, records, formats, want_ring: bool, want_order: bool, label8: bool, pinned: bool = False) -> "BatchHandle":
        """A batch of raw PointCloud2 record arrays where records[b] has the format formats[b] (CloudFormat or 5-tuple)."""
        if len(records) != len(formats):
            raise ValueError(f"{len(records)} scans but {len(formats)} formats")
        raws = [np.ascontiguousarray(r).view(np.uint8).reshape(-1) for r in records]
        return cls(raws, [r.size // int(f[0]) for r, f in zip(raws, formats)], want_ring, want_order, label8, pinned=pinned,
                   formats=[CloudFormat(*(int(v) for v in f)) for f in formats])

    def collect(self) -> list[ScanResult]:
        """ScanResults of the finished call: labels as int32 (int8 ones widened), ring cut to n_in; copies of page-locked
        buffers, so they outlive free()."""
        out = []
        for b, n in enumerate(self.ns):
            lab, ring, order, rs = self.bufs[b]
            if lab is not None:
                lab = lab[:n].astype(np.int32) if self.l8 is not None else lab[:n]
            ring = None if ring is None else ring[:n]
            if self.pinned:
                lab = None if lab is None else lab.copy()
                ring = None if ring is None else ring.copy()
            out.append(_scan_result(self.res[b], lab, ring, order, rs))
        self.results = out
        return out

    def free(self):
        """Gives the page-locked buffers back; the handle must not be in flight."""
        for p in self._pins:
            self.lib.urf_pinned_free(p)
        self._pins = []

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass


class Detector:
    """Host-side mirror of the reference's `Detector` (include/urban_road_filter/data_structures.hpp:110-141) on one GPU."""

    def __init__(self, max_points: int, max_batch: int = 1, device: int = 0, params: UrfParams | None = None,
                 tie_order: str = "input"):
        self.lib = load_library()
        self._ctx = C.c_void_p()
        self._inflight = collections.deque()         # BatchHandles of enqueue_batch*, oldest first
        rc = self.lib.urf_create(C.byref(self._ctx), device, max_points, max_batch)
        if rc != URF_OK:
            raise UrfError(rc, "urf_create", self.lib.urf_strerror(rc).decode())
        self.max_points, self.max_batch, self.device = max_points, max_batch, device
        self.params = params if params is not None else make_params()
        self.set_params(self.params)
        if tie_order != "input":
            self.set_tie_order(tie_order)
        self.ghostcount = 0      # lidar_segmentation.cpp:23

    def close(self):
        if getattr(self, "_ctx", None) and self._ctx.value:
            self.lib.urf_destroy(self._ctx)           # waits for batches in flight, whose buffers _inflight still holds
            self._ctx = C.c_void_p()
            self._inflight.clear()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _check(self, rc: int, where: str):
        if rc < 0:
            raise UrfError(rc, where, self.lib.urf_strerror(rc).decode() + ": " + self.lib.urf_last_cuda_error(self._ctx).decode())

    def set_params(self, prm: UrfParams):
        """paramsCallback (src/main.cpp:4-34)."""
        self._check(self.lib.urf_set_params(self._ctx, C.byref(prm)), "urf_set_params")
        self.params = prm

    def set_params_next(self, prm: UrfParams) -> int:
        """paramsCallback while batches are in flight (urf_set_params_next): `prm` applies from the next enqueue / filtered
        call on, batches already enqueued keep the set they were enqueued with. Returns the new parameter generation, which
        the results of later calls report as `params_gen`."""
        gen = self.lib.urf_set_params_next(self._ctx, C.byref(prm))
        self._check(gen, "urf_set_params_next")
        self.params = prm
        return gen

    def set_option(self, option: int, value: int):
        self._check(self.lib.urf_set_option(self._ctx, option, value), "urf_set_option")

    def set_tie_order(self, mode: str):
        """"input" (default: equal azimuths of a ring in input order) or "reference" (the order the reference's Lomuto
        quicksort leaves: its clouds and marker vertices bit for bit). Applies from the next call (urf_set_tie_order)."""
        if mode not in TIE_ORDERS:
            raise ValueError(f"tie order {mode!r}: expected one of {sorted(TIE_ORDERS)}")
        self._check(self.lib.urf_set_tie_order(self._ctx, TIE_ORDERS[mode]), "urf_set_tie_order")

    def tie_order(self) -> str:
        m = C.c_int()
        self._check(self.lib.urf_get_tie_order(self._ctx, C.byref(m)), "urf_get_tie_order")
        return {v: k for k, v in TIE_ORDERS.items()}[m.value]

    def filtered_batch(self, clouds, want_ring: bool = True, want_order: bool = True) -> list[ScanResult]:
        """`batch` independent Detector::filtered() calls (lidar_segmentation.cpp:95) on host (N,4) float32 arrays."""
        hb = BatchHandle.of_clouds(clouds, want_ring, want_order, label8=False)
        self._check(self.lib.urf_process_batch(self._ctx, hb.ptrs, hb.ns, len(hb.ns), hb.res), "urf_process_batch")
        return hb.collect()

    def filtered_batch_records(self, records, point_step: int, off_x: int, off_y: int, off_z: int, off_intensity: int = -1,
                               want_order: bool = False, label8: bool = True, want_ring: bool = False) -> list[ScanResult]:
        """`batch` scans given as raw PointCloud2 record arrays (uint8, n * point_step bytes each) of one sensor format,
        unpacked on the device (urf_process_cloud2_batch). point_step == 12 with offsets 0, 4, 8 is the packed-xyz lean
        input of urf_process_batch_xyz, which this method then calls. label8: labels come back as int8."""
        hb = BatchHandle.of_records(records, point_step, off_x, off_y, off_z, off_intensity, want_ring, want_order, label8)
        B = len(hb.ns)
        if point_step == 12 and (off_x, off_y, off_z) == (0, 4, 8) and off_intensity < 0:
            self._check(self.lib.urf_process_batch_xyz(self._ctx, hb.ptrs, hb.ns, B, hb.res, hb.l8), "urf_process_batch_xyz")
        else:
            self._check(self.lib.urf_process_cloud2_batch(self._ctx, hb.ptrs, hb.ns, B, point_step, off_x, off_y, off_z, off_intensity, hb.res,
                                                          hb.l8), "urf_process_cloud2_batch")
        return hb.collect()

    def filtered_batch_mixed(self, records, formats, want_order: bool = False, label8: bool = True,
                             want_ring: bool = False) -> list[ScanResult]:
        """filtered_batch_records for a batch of several sensor formats: records[b] (uint8 record bytes) has the format
        formats[b] (CloudFormat or (point_step, off_x, off_y, off_z, off_intensity)); one unpack launch for the whole batch
        (urf_process_cloud2_batch_mixed). Every result is what filtered_batch_records gives for that scan alone."""
        hb = BatchHandle.of_mixed(records, formats, want_ring, want_order, label8)
        self._check(self.lib.urf_process_cloud2_batch_mixed(self._ctx, hb.ptrs, hb.ns, hb.fmts, len(hb.ns), hb.res, hb.l8),
                    "urf_process_cloud2_batch_mixed")
        return hb.collect()

    def enqueue(self, hb: "BatchHandle") -> "BatchHandle":
        """Enqueues a prepared batch (BatchHandle.of_clouds / of_records / of_mixed; urf_enqueue_batch /
        urf_enqueue_cloud2_batch / urf_enqueue_cloud2_batch_mixed) and
        returns at once when its buffers are pinned. finish_batch fills its `results`. At most two batches are in flight;
        the detector keeps the handle alive until then. While batches are in flight every other compute call and
        set_params / set_tie_order / set_option raise (URF_ERR_INVALID); set_params_next changes the set of the next
        enqueue."""
        B = len(hb.ns)
        if hb.fmts is not None:
            rc, where = (self.lib.urf_enqueue_cloud2_batch_mixed(self._ctx, hb.ptrs, hb.ns, hb.fmts, B, hb.res, hb.l8),
                         "urf_enqueue_cloud2_batch_mixed")
        elif hb.step == 0:
            rc, where = self.lib.urf_enqueue_batch(self._ctx, hb.ptrs, hb.ns, B, hb.res, hb.l8), "urf_enqueue_batch"
        else:
            rc, where = self.lib.urf_enqueue_cloud2_batch(self._ctx, hb.ptrs, hb.ns, B, hb.step, *hb.offs, hb.res, hb.l8), "urf_enqueue_cloud2_batch"
        self._check(rc, where)
        self._inflight.append(hb)
        return hb

    def enqueue_batch(self, clouds, want_ring: bool = True, want_order: bool = True, label8: bool = False) -> "BatchHandle":
        """filtered_batch without waiting: enqueue() of a pinned handle built here. Allocating its page-locked buffers can
        wait for a batch already in flight; callers that want batches to overlap build the handles first."""
        return self.enqueue(BatchHandle.of_clouds(clouds, want_ring, want_order, label8, pinned=True))

    def enqueue_batch_records(self, records, point_step: int, off_x: int, off_y: int, off_z: int, off_intensity: int = -1,
                              want_order: bool = False, label8: bool = True, want_ring: bool = False) -> "BatchHandle":
        """filtered_batch_records without waiting (urf_enqueue_cloud2_batch); see enqueue_batch."""
        return self.enqueue(BatchHandle.of_records(records, point_step, off_x, off_y, off_z, off_intensity, want_ring, want_order, label8,
                                                   pinned=True))

    def finish_batch(self) -> "BatchHandle":
        """Waits for the oldest batch in flight (urf_finish_batch), fills its handle's `results` and returns the handle."""
        rc = self.lib.urf_finish_batch(self._ctx)
        hb = self._inflight.popleft() if self._inflight else None      # the library frees the slot whatever the outcome
        self._check(rc, "urf_finish_batch")
        hb.collect()
        return hb

    def _one_record_scan(self, data, n_points: int, point_step: int, offs, want_ring: bool, want_order: bool, want_label: bool) -> BatchHandle:
        """Input and result buffers of one scan given as raw PointCloud2 bytes, of which n_points records count."""
        raw = np.frombuffer(data, np.uint8) if isinstance(data, (bytes, bytearray)) else np.ascontiguousarray(data).view(np.uint8).reshape(-1)
        return BatchHandle([raw], [n_points], want_ring, want_order, False, point_step, offs, want_label=want_label)

    def filtered_cloud2(self, data: bytes | np.ndarray, n_points: int, point_step: int, off_x: int, off_y: int, off_z: int) -> ScanResult:
        """One scan from the raw `data` bytes of a sensor_msgs/PointCloud2 (unpacked on the device)."""
        hb = self._one_record_scan(data, n_points, point_step, (off_x, off_y, off_z, -1), True, True, True)
        self._check(self.lib.urf_process_cloud2(self._ctx, hb.ptrs[0], n_points, point_step, off_x, off_y, off_z, hb.res), "urf_process_cloud2")
        return hb.collect()[0]

    def filtered_cloud2_packed(self, data, n_points: int, point_step: int, off_x: int, off_y: int, off_z: int,
                               off_intensity: int = -1, want_labels: bool = False):
        """One scan from raw PointCloud2 bytes; returns (ScanResult, clouds) where clouds maps "road" / "curb" / "roi" /
        "road_probably" to float32 arrays [count, 8] of 32-byte pcl::PointXYZI records packed on the device in the
        reference's emission order (include/urf.h urf_clouds). Labels / order are only fetched with want_labels."""
        hb = self._one_record_scan(data, n_points, point_step, (off_x, off_y, off_z, off_intensity), False, want_labels, want_labels)
        bufs = {k: np.empty((max(n_points, 1), 8), np.float32) for k in ("road", "curb", "roi", "road_probably")}
        cl = UrfClouds()
        for k, a in bufs.items():
            setattr(cl, k, a.ctypes.data)
        self._check(self.lib.urf_process_cloud2_packed(self._ctx, hb.ptrs[0], n_points, point_step, off_x, off_y, off_z,
                                                       off_intensity, hb.res, C.byref(cl)), "urf_process_cloud2_packed")
        counts = dict(road=cl.n_road, curb=cl.n_curb, roi=cl.n_roi, road_probably=cl.n_road_probably)
        return hb.collect()[0], {k: bufs[k][: counts[k]] for k in bufs}

    def filtered(self, cloud, **kw) -> ScanResult:
        """One Detector::filtered() call."""
        return self.filtered_batch([cloud], **kw)[0]

    def markers(self, result: ScanResult):
        """road_marker MarkerArray of a scan (keeps the reference's `ghostcount` state between scans)."""
        if not result.published:
            return []
        strips, self.ghostcount = build_markers(self.params, result.vert, self.ghostcount)
        return strips

    # diagnostics -------------------------------------------------------------------------------------------------
    def last_device_ms(self) -> float:
        return float(self.lib.urf_last_device_ms(self._ctx))

    def last_launch_count(self) -> int:
        return int(self.lib.urf_last_launch_count(self._ctx))

    def kernel_times(self, slot: int = 0) -> list[tuple[str, float]]:
        """(kernel name, device ms) of the call recorded in event slot `slot`; needs set_option(1, nslots) beforehand."""
        out = []
        for i in range(self.lib.urf_profile_count(self._ctx)):
            name, ms = C.c_char_p(), C.c_float()
            self._check(self.lib.urf_profile_get(self._ctx, slot, i, C.byref(name), C.byref(ms)), "urf_profile_get")
            out.append((name.value.decode(), float(ms.value)))
        return out

    def debug_fetch(self, scan: int, what: int, dtype, count: int) -> np.ndarray:
        a = np.zeros(max(count, 1), dtype)
        self._check(self.lib.urf_debug_fetch(self._ctx, scan, what, a.ctypes.data, a.nbytes if count else 0), "urf_debug_fetch")
        return a[:count]


def _slot_ints(ptr, n: int, copy: bool) -> np.ndarray:
    """The first n int32 of a lent slot's array: a view, or with `copy` a copy."""
    if n <= 0:
        return np.zeros(0, np.int32)
    a = np.ctypeslib.as_array(ptr, shape=(n,))
    return a.copy() if copy else a


class _BatchBuffers:
    """Output arrays of urf_queue_next_batch / urf_mq_next_batch for up to `cap` scans, reused between calls."""

    def __init__(self, cap: int):
        self.cap = cap
        self.tags = (C.c_uint64 * cap)()
        self.rcs = (C.c_int32 * cap)()
        self.outs = (UrfResult * cap)()
        self.views = (C.c_void_p * cap)()

    def results(self, k: int, label8: bool, copy: bool) -> list:
        """(tag, ScanResult) of the k scans handed out. Labels, and the emission order and ring offsets of a queue that
        delivers them, are numpy views of the lent slots (labels int8 or int32) unless `copy`; a scan whose batch failed has
        status = its (negative) error code and label / order / ring_start None."""
        ct = C.c_int8 if label8 else C.c_int32
        out = []
        for j in range(k):
            res, rc = self.outs[j], int(self.rcs[j])
            lab = None
            if rc == URF_OK:
                n = int(res.n_in)
                lab = (np.ctypeslib.as_array(C.cast(self.views[j], C.POINTER(ct)), shape=(n,)) if n > 0
                       else np.zeros(0, np.int8 if label8 else np.int32))
                if copy:
                    lab = lab.copy()
            r = _scan_result(res, lab)
            if res.order:                                # URF_QUEUE_ORDER, and the scan did not fail
                r.order = _slot_ints(res.order, r.n_order, copy)
                r.ring_start = _slot_ints(res.ring_start, r.n_rings + 1, copy)
            if rc != URF_OK:
                r.status = rc
            out.append((int(self.tags[j]), r))
        return out


class _StreamQueue:
    """What ScanQueue and MultiGpuQueue share: the library handle `_h`, the arrays of by-reference submits, the reused
    batch buffers, and submit / submit_records / next / next_batch / close / destroy, written against the library functions
    `_PREFIX` + name (urf_queue_* or urf_mq_*), which have the same arguments in both families."""
    _PREFIX = ""

    def __init__(self, max_points: int, label8: bool, params: UrfParams | None = None, order: bool = False, records=None,
                 formats=None):
        if records is not None and formats is not None:
            raise ValueError("records and formats: a queue takes one record format or a table of them")
        self.lib = load_library()
        self._h = C.c_void_p()
        self.max_points = max_points
        self.label8 = label8
        self.order = order                # URF_QUEUE_ORDER: results carry order and ring_start
        # record queue: (point_step, off_x, off_y, off_z, off_intensity) of its PointCloud2 records; None: float4 scans
        self.records = None if records is None else tuple(int(v) for v in records)
        # formats queue: its table of CloudFormats (urf_*_create_formats), each submit_records naming one by index
        self.formats = None if formats is None else [CloudFormat(*(int(v) for v in f)) for f in formats]
        self._fmt_table = None if formats is None else _format_array(self.formats)
        self._cb = None                   # ctypes callbacks of a stand-in, kept alive with the queue
        self._params_cb = None            # the parameter hook of a stand-in
        self._bufs = None
        self._keep = {}                   # arrays of by-reference submits, until their results come back
        self._sets = {0: params}          # parameter generation -> set (0: the set in force at creation, None if unknown)

    def _call(self, name: str, *args) -> int:
        return getattr(self.lib, self._PREFIX + name)(self._h, *args)

    def update_params(self, prm: UrfParams) -> int:
        """New parameters for a running queue, with no drain (urf_queue_update_params / urf_mq_update_params): every scan
        submitted after this returns runs with `prm`, every scan before with the earlier sets, and no batch mixes them.
        Returns the new generation; results report theirs as `params_gen`, and params_of(gen) gives its set back."""
        gen = self._call("update_params", C.byref(prm))
        if gen < 0:
            raise UrfError(gen, self._PREFIX + "update_params")
        self._sets[gen] = UrfParams.from_buffer_copy(prm)   # a copy: the caller may change its own set afterwards
        return gen

    def params_of(self, gen: int) -> UrfParams | None:
        """The set of generation `gen` (for build_markers of a result with that params_gen); None for generation 0 when the
        queue does not know it (stand-in devices). One entry is kept per update."""
        return self._sets[gen]

    def set_params_hook(self, fn):
        """Stand-in queues only (tests): fn(user, params pointer, generation) -> int is called where a real queue's worker
        calls urf_set_params_next (urf_queue_set_params_hook / urf_mq_set_params_hook)."""
        self._params_cb = QUEUE_PARAMS_FN(fn)
        rc = self._call("set_params_hook", self._params_cb)
        if rc != URF_OK:
            raise UrfError(rc, self._PREFIX + "set_params_hook")

    def submit(self, cloud: np.ndarray, tag: int = 0, timeout_ms: int = -1, by_reference: bool = False) -> int:
        """Returns URF_OK, URF_ERR_TIMEOUT or URF_ERR_CLOSED; raises on anything else. by_reference: no copy
        (urf_queue_submit_ref / urf_mq_submit_ref): keep the array alive and unchanged until its result has come back."""
        pts = np.ascontiguousarray(cloud, np.float32)
        if by_reference:
            self._keep[tag] = pts
        rc = self._call("submit_ref" if by_reference else "submit", pts.ctypes.data, pts.shape[0], tag, timeout_ms)
        if rc not in (URF_OK, URF_ERR_TIMEOUT, URF_ERR_CLOSED):
            raise UrfError(rc, self._PREFIX + "submit")
        return rc

    def submit_records(self, data, n_points: int, tag: int = 0, timeout_ms: int = -1, by_reference: bool = False,
                       fmt: int | None = None) -> int:
        """A scan of a record queue: the raw `data` bytes of a sensor_msgs/PointCloud2 (bytes, bytearray or an array), of
        which the first n_points records count (urf_queue_submit_cloud2 / urf_mq_submit_cloud2). Returns as submit, and
        raises UrfError(URF_ERR_INVALID) on a float4 queue. by_reference: no copy (urf_*_submit_cloud2_ref): keep `data`
        alive and unchanged until its result has come back. fmt: the scan's index into the table of a formats queue
        (urf_*_submit_format[_ref]); the library refuses it on any other queue, and a formats queue refuses fmt=None."""
        raw = np.frombuffer(data, np.uint8) if isinstance(data, (bytes, bytearray)) else np.ascontiguousarray(data).view(np.uint8).reshape(-1)
        step = (self.records[0] if self.records is not None and fmt is None else
                self.formats[fmt].point_step if self.formats is not None and fmt is not None and 0 <= fmt < len(self.formats) else 0)
        if raw.size < n_points * step:
            raise ValueError(f"{raw.size} bytes hold fewer than {n_points} records of {step} bytes")
        if by_reference:
            self._keep[tag] = raw
        if fmt is None:
            name = "submit_cloud2_ref" if by_reference else "submit_cloud2"
            rc = self._call(name, raw.ctypes.data, n_points, tag, timeout_ms)
        else:
            name = "submit_format_ref" if by_reference else "submit_format"
            rc = self._call(name, fmt, raw.ctypes.data, n_points, tag, timeout_ms)
        if rc not in (URF_OK, URF_ERR_TIMEOUT, URF_ERR_CLOSED):
            raise UrfError(rc, self._PREFIX + name)
        return rc

    def next(self, timeout_ms: int = -1):
        """(tag, ScanResult) of the oldest finished scan, or None on timeout / when the closed queue is drained. With
        `order` the result's order and ring_start are copies of the scan's n_order / n_rings + 1 entries."""
        lab = np.full(self.max_points, -1, np.int32)
        res = UrfResult()
        res.label = lab.ctypes.data_as(C.POINTER(C.c_int32))
        order = rs = None
        if self.order:
            order, rs = np.zeros(self.max_points, np.int32), np.zeros(URF_MAX_CHANNELS + 1, np.int32)
            res.order = order.ctypes.data_as(C.POINTER(C.c_int32))
            res.ring_start = rs.ctypes.data_as(C.POINTER(C.c_int32))
        tag = C.c_uint64()
        rc = self._call("next", C.byref(tag), C.byref(res), timeout_ms)
        if rc in (URF_ERR_TIMEOUT, URF_ERR_CLOSED):
            return None
        if rc != URF_OK:
            raise UrfError(rc, self._PREFIX + "next")
        self._keep.pop(tag.value, None)
        return tag.value, _scan_result(res, lab[: res.n_in].copy(), order=order, ring_start=rs)

    def next_batch(self, max_results: int, timeout_ms: int = -1, copy: bool = False) -> list:
        """[(tag, ScanResult)] of the run of finished scans that starts with the oldest one (urf_queue_next_batch /
        urf_mq_next_batch), at most max_results; [] on timeout / when the closed queue is drained. Labels (int8 with
        label8), and with `order` the emission order and ring_start, are views of the lent slots, valid until the next
        next* call, unless `copy`. A scan whose batch failed has status < 0 and label / order / ring_start None."""
        if max_results < 1:
            raise ValueError("max_results must be >= 1")
        if self._bufs is None or self._bufs.cap < max_results:
            self._bufs = _BatchBuffers(max_results)
        b = self._bufs
        k = self._call("next_batch", max_results, b.tags, b.rcs, b.outs, b.views, timeout_ms)
        if k in (URF_ERR_TIMEOUT, URF_ERR_CLOSED):
            return []
        if k < 0:
            raise UrfError(k, self._PREFIX + "next_batch")
        out = b.results(k, self.label8, copy)
        for t, _ in out:
            self._keep.pop(t, None)
        return out

    def close(self):
        if self._h:
            self._call("close")

    def destroy(self):
        if self._h:
            self._call("destroy")
            self._h = C.c_void_p()


class MultiGpuQueue(_StreamQueue):
    """One ingest stream over several GPUs (include/urf.h urf_mq, BASELINE config 4): a context + streaming queue per device,
    every scan goes to the device with the fewest scans in flight, results come back in submission order. Any number of
    producer threads, one consumer. `by_reference` submits hand the array to the library without a copy: keep it alive and
    unchanged until its result has come back. label8: int8 label slots on every device, order: the emission order and ring
    offsets with every result, records: a record mq (urf_mq_create_cloud2) fed with submit_records (see ScanQueue), formats:
    a formats mq (urf_mq_create_formats) whose submit_records name each scan's format (see ScanQueue)."""
    _PREFIX = "urf_mq_"
    _m = property(lambda self: self._h)      # the library handle, under the name this class has always had for it

    def __init__(self, devices, max_points: int, slots_per_device: int = 8, max_batch: int = 4, params: UrfParams | None = None,
                 process_fn=None, label8: bool = False, order: bool = False, records=None, formats=None):
        super().__init__(max_points, label8, None if process_fn is not None else params if params is not None else make_params(), order,
                         records, formats)
        policy = URF_QUEUE_BLOCK | (URF_QUEUE_LABEL8 if label8 else 0) | (URF_QUEUE_ORDER if order else 0)
        fmt = self.records or (() if formats is None else (self._fmt_table, len(self.formats)))
        kind = "cloud2" if self.records else "formats" if formats is not None else "policy"
        if process_fn is not None:                      # tests: stand-in devices, no GPU
            self._cb = QUEUE_PROCESS_FN(process_fn)
            create = getattr(self.lib, "urf_mq_create_with_policy" if kind == "policy" else f"urf_mq_create_{kind}_with")
            rc = create(C.byref(self._h), self._cb, None, len(devices), max_points, slots_per_device, max_batch, policy, *fmt)
        else:
            dv = (C.c_int * len(devices))(*devices)
            create = getattr(self.lib, f"urf_mq_create_{kind}")
            rc = create(C.byref(self._h), dv, len(devices), max_points, slots_per_device, max_batch,
                        C.byref(params) if params is not None else None, policy, *fmt)
        if rc != URF_OK:
            raise UrfError(rc, "urf_mq_create", self.lib.urf_last_cuda_error(None).decode())

    def set_params(self, prm: UrfParams):
        rc = self._call("set_params", C.byref(prm))
        if rc != URF_OK:
            raise UrfError(rc, "urf_mq_set_params")

    def set_tie_order(self, mode: str):
        """Detector.set_tie_order on every device; like set_params, only while nothing is in flight."""
        if mode not in TIE_ORDERS:
            raise ValueError(f"tie order {mode!r}: expected one of {sorted(TIE_ORDERS)}")
        rc = self._call("set_tie_order", TIE_ORDERS[mode])
        if rc != URF_OK:
            raise UrfError(rc, "urf_mq_set_tie_order")

    def stats(self) -> dict:
        st = UrfMqStats()
        self._call("get_stats", C.byref(st))
        n = st.n_devices
        return dict(n_devices=n, pending=st.pending, submitted=list(st.submitted[:n]), delivered=list(st.delivered[:n]),
                    batches=list(st.batches[:n]), largest_batch=list(st.largest_batch[:n]))


class ScanQueue(_StreamQueue):
    """Streaming ingest (include/urf.h urf_queue, SURVEY.md §8 f4): producers `submit` scans from any thread, one worker
    thread batches whatever is pending through the detector, `next` returns results in submission order and `next_batch`
    every result that is ready at once. With `process_fn` (a Python callable with urf_process_batch's arguments) the queue
    runs without a GPU — tests only; with `enqueue_fn` and `finish_fn` instead (urf_enqueue_batch's arguments / none) it
    runs the real queue's two-batches-in-flight schedule around them. label8: int8 label slots (URF_QUEUE_LABEL8) — a
    quarter of the label traffic and memory; `next` still returns int32 labels, `next_batch` int8 ones. order
    (URF_QUEUE_ORDER): every result also carries its emission order and ring_start, so that cloud_indices("road" | "curb" |
    "road_probably") works on it; the batches then run the ring sort and copy 4 bytes per point more. records
    (point_step, off_x, off_y, off_z, off_intensity): a queue of raw PointCloud2 records of that one format
    (urf_queue_create_cloud2, or urf_queue_create_cloud2_with around process_fn), fed with submit_records and unpacked on
    the device; `submit` then raises, as submit_records does on a float4 queue. formats (a list of CloudFormat or 5-tuples,
    1..URF_MAX_FORMATS): a queue of several record formats (urf_queue_create_formats[_with]); submit_records(..., fmt=k)
    names each scan's format, and batches mix formats."""
    _PREFIX = "urf_queue_"
    _q = property(lambda self: self._h)      # the library handle, under the name this class has always had for it

    def __init__(self, detector: "Detector | None", max_points: int, slots: int = 8, max_batch: int = 4,
                 policy: int = URF_QUEUE_BLOCK, process_fn=None, label8: bool = False, enqueue_fn=None, finish_fn=None,
                 order: bool = False, records=None, formats=None):
        order = order or bool(policy & URF_QUEUE_ORDER)
        super().__init__(max_points, label8, detector.params if detector is not None else None, order, records, formats)
        fmt = self.records or (() if formats is None else (self._fmt_table, len(self.formats)))
        kind = "_cloud2" if self.records else "_formats" if formats is not None else ""
        if label8:
            policy |= URF_QUEUE_LABEL8
        if order:
            policy |= URF_QUEUE_ORDER
        if enqueue_fn is not None:
            if fmt:
                raise ValueError("records / formats: a record queue has no asynchronous stand-in")
            self._cb = (QUEUE_PROCESS_FN(enqueue_fn), QUEUE_FINISH_FN(lambda user: finish_fn()))
            rc = self.lib.urf_queue_create_with_async(C.byref(self._h), *self._cb, None, max_points, slots, max_batch, policy)
        elif process_fn is not None:
            self._cb = QUEUE_PROCESS_FN(process_fn)
            create = getattr(self.lib, f"urf_queue_create{kind}_with")
            rc = create(C.byref(self._h), self._cb, None, max_points, slots, max_batch, policy, *fmt)
        else:
            assert detector is not None and detector.max_batch >= max_batch and detector.max_points >= max_points
            self._det = detector          # keeps the ctx alive; nobody else may use it while the queue exists
            create = getattr(self.lib, f"urf_queue_create{kind}")
            rc = create(C.byref(self._h), detector._ctx, max_points, slots, max_batch, policy, *fmt)
        if rc != URF_OK:
            raise UrfError(rc, "urf_queue_create")

    def release(self):
        """Gives the slots lent by next_batch back before the next call (urf_queue_release_view)."""
        self._call("release_view")

    def stats(self) -> dict:
        st = UrfQueueStats()
        self._call("get_stats", C.byref(st))
        return {k: int(getattr(st, k)) for k, _ in UrfQueueStats._fields_}

"""ctypes mirror of include/urf.h (struct layouts and constants only; no library is loaded here)."""
from __future__ import annotations

import ctypes as C

URF_MAX_VERTS = 361
URF_STAR_SECTORS = 360
URF_MAX_CHANNELS = 256

URF_OK = 0
URF_TOO_FEW_POINTS = 1
URF_ERR_INVALID = -1
URF_ERR_NO_DEVICE = -2
URF_ERR_CUDA = -3
URF_ERR_NOMEM = -4
URF_ERR_CAPACITY = -5

LABEL_OUTSIDE, LABEL_NONE, LABEL_ROAD, LABEL_CURB = -1, 0, 1, 2


class UrfParams(C.Structure):
    """urf_params — the 27 fields of cfg/LidarFilters.cfg:10-84 (+ channels, lidar_segmentation.cpp:4)."""
    _fields_ = [
        ("fixed_frame", C.c_char * 128),
        ("topic_name", C.c_char * 128),
        ("x_zero_method", C.c_int),
        ("z_zero_method", C.c_int),
        ("star_shaped_method", C.c_int),
        ("blind_spots", C.c_int),
        ("xDirection", C.c_int),
        ("interval", C.c_double),
        ("curb_height", C.c_double),
        ("curb_points", C.c_int),
        ("beamZone", C.c_double),
        ("min_x", C.c_double), ("max_x", C.c_double),
        ("min_y", C.c_double), ("max_y", C.c_double),
        ("min_z", C.c_double), ("max_z", C.c_double),
        ("cylinder_deg_x", C.c_double),
        ("cylinder_deg_z", C.c_double),
        ("curb_slope_deg", C.c_double),
        ("kdev_param", C.c_double),
        ("kdist_param", C.c_double),
        ("starbeam_filter", C.c_int),
        ("dmin_param", C.c_int),
        ("simple_poly_allow", C.c_int),
        ("poly_s_param", C.c_double),
        ("poly_z_manual", C.c_double),
        ("poly_z_avg_allow", C.c_int),
        ("channels", C.c_int),
    ]


class _ResultGen(C.Union):
    """urf_result's anonymous union: `reserved` under its old name, `params_gen` the parameter generation."""
    _fields_ = [("reserved", C.c_int32), ("params_gen", C.c_int32)]


class UrfResult(C.Structure):
    _anonymous_ = ("_gen",)
    _fields_ = [
        ("status", C.c_int32), ("n_in", C.c_int32), ("n_roi", C.c_int32), ("n_rings", C.c_int32),
        ("n_order", C.c_int32), ("n_road", C.c_int32), ("n_curb", C.c_int32), ("n_vert", C.c_int32),
        ("flags", C.c_int32), ("_gen", _ResultGen),
        ("label", C.POINTER(C.c_int32)),
        ("ring", C.POINTER(C.c_int32)),
        ("order", C.POINTER(C.c_int32)),
        ("ring_start", C.POINTER(C.c_int32)),
        ("vert", (C.c_float * 4) * URF_MAX_VERTS),
    ]


class UrfStrip(C.Structure):
    _fields_ = [("id", C.c_int32), ("action", C.c_int32), ("red", C.c_int32), ("first", C.c_int32),
                ("count", C.c_int32)]


class UrfPointXYZI(C.Structure):
    """pcl::PointXYZI as the reference stores it (32 bytes)."""
    _fields_ = [("x", C.c_float), ("y", C.c_float), ("z", C.c_float), ("w", C.c_float),
                ("intensity", C.c_float), ("pad", C.c_float * 3)]


class UrfClouds(C.Structure):
    _fields_ = [("road", C.c_void_p), ("curb", C.c_void_p), ("roi", C.c_void_p), ("road_probably", C.c_void_p),
                ("n_road", C.c_int32), ("n_curb", C.c_int32), ("n_roi", C.c_int32), ("n_road_probably", C.c_int32)]


class UrfQueueStats(C.Structure):
    _fields_ = [("submitted", C.c_uint64), ("processed", C.c_uint64), ("dropped", C.c_uint64), ("delivered", C.c_uint64),
                ("batches", C.c_uint64), ("largest_batch", C.c_int32), ("pending", C.c_int32), ("most_in_flight", C.c_int32)]


URF_MQ_MAX_DEVICES = 16


class UrfMqStats(C.Structure):
    _fields_ = [("n_devices", C.c_int32), ("pending", C.c_int32), ("submitted", C.c_uint64 * URF_MQ_MAX_DEVICES),
                ("delivered", C.c_uint64 * URF_MQ_MAX_DEVICES), ("batches", C.c_uint64 * URF_MQ_MAX_DEVICES),
                ("largest_batch", C.c_int32 * URF_MQ_MAX_DEVICES)]


URF_QUEUE_BLOCK, URF_QUEUE_DROP_OLDEST = 0, 1
URF_QUEUE_LABEL8 = 2          # OR-ed into the policy: int8 label slots
URF_QUEUE_ORDER = 4           # OR-ed into the policy: every result also carries its emission order and ring offsets
URF_ERR_TIMEOUT, URF_ERR_CLOSED = -6, -7
# int (*)(void* user, const float* const* xyzi, const int* n, int batch, urf_result* outs)
QUEUE_PROCESS_FN = C.CFUNCTYPE(C.c_int, C.c_void_p, C.POINTER(C.c_void_p), C.POINTER(C.c_int), C.c_int, C.POINTER(UrfResult))
# int (*)(void* user): finishes the oldest batch of an asynchronous stand-in (urf_queue_create_with_async)
QUEUE_FINISH_FN = C.CFUNCTYPE(C.c_int, C.c_void_p)
# int (*)(void* user, const urf_params* p, int32_t gen): a stand-in queue's parameter hook (urf_queue_set_params_hook)
QUEUE_PARAMS_FN = C.CFUNCTYPE(C.c_int, C.c_void_p, C.POINTER(UrfParams), C.c_int32)


class UrfCloud2User(C.Structure):
    """urf_cloud2_user: what a record stand-in's batch function and parameter hook get as `user` (the record format and the
    creator's user)."""
    _fields_ = [("user", C.c_void_p), ("point_step", C.c_int32), ("off_x", C.c_int32), ("off_y", C.c_int32),
                ("off_z", C.c_int32), ("off_intensity", C.c_int32)]


URF_MAX_FORMATS = 8


class UrfCloud2Format(C.Structure):
    """urf_cloud2_format: one PointCloud2 record format (point_step and the byte offsets of x, y, z and intensity, -1: none)."""
    _fields_ = [("point_step", C.c_int32), ("off_x", C.c_int32), ("off_y", C.c_int32), ("off_z", C.c_int32),
                ("off_intensity", C.c_int32)]


class UrfFormatsUser(C.Structure):
    """urf_formats_user: what a formats stand-in's batch function and parameter hook get as `user` (the creator's user, the
    format table, and during a batch call each scan's index into it)."""
    _fields_ = [("user", C.c_void_p), ("formats", C.POINTER(UrfCloud2Format)), ("n_formats", C.c_int32),
                ("fmt", C.POINTER(C.c_int32))]


# cfg/LidarFilters.cfg:10-84 defaults
DEFAULTS = dict(
    fixed_frame=b"left_os1/os1_lidar", topic_name=b"/left_os1/os1_cloud_node/points",
    x_zero_method=1, z_zero_method=1, star_shaped_method=1, blind_spots=1, xDirection=0,
    interval=0.18, curb_height=0.05, curb_points=5, beamZone=30.0,
    min_x=0.0, max_x=30.0, min_y=-10.0, max_y=10.0, min_z=-3.0, max_z=-1.0,
    cylinder_deg_x=150.0, cylinder_deg_z=140.0, curb_slope_deg=50.0,
    kdev_param=1.225, kdist_param=2.0, starbeam_filter=0, dmin_param=10,
    simple_poly_allow=1, poly_s_param=0.7, poly_z_manual=-1.5, poly_z_avg_allow=1, channels=64,
)

FULL_ROI = dict(min_x=-200.0, max_x=200.0, min_y=-200.0, max_y=200.0, min_z=-200.0, max_z=200.0)


def make_params(**over) -> UrfParams:
    """LidarFilters.cfg defaults, overridden by keyword (same names as the cfg)."""
    p = UrfParams()
    vals = dict(DEFAULTS)
    for k, v in over.items():
        if k not in vals:
            raise KeyError(f"unknown LidarFilters parameter {k!r}")
        vals[k] = v
    for k, v in vals.items():
        if isinstance(v, str):
            v = v.encode()
        setattr(p, k, v)
    return p

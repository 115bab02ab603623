"""The reference-side binding: ros/urf_node.cpp (thin ROS1 glue around the C-ABI) compiled against the shim ROS/PCL headers.
Without a GPU: it compiles, links against liburf_b200.so and exports its test entry. With a GPU: a cloud pushed through the
glue node's scan callback publishes exactly what the unmodified reference node published for the same cloud and parameters
(roi / road / curb / road_probably clouds point for point and in order, road_marker strips vertex for vertex)."""
import ctypes as C
import os

import numpy as np
import pytest

from urban_road_filter_b200 import UrfParams, UrfStrip
from util import ROOT, Golden, compare_strips, golden_names


def _lib():
    lib = C.CDLL(os.path.join(ROOT, "build", "libglue.so"))
    lib.urf_glue_run.restype = C.c_int
    lib.urf_glue_run.argtypes = [C.c_void_p, C.c_int, C.POINTER(UrfParams), C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p,
                                 C.c_void_p, C.POINTER(UrfStrip), C.c_int, C.c_void_p, C.c_int]
    lib.urf_glue_run_cloud2.restype = C.c_int
    lib.urf_glue_run_cloud2.argtypes = [C.c_void_p, C.c_int, C.POINTER(UrfParams), C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p,
                                        C.c_void_p, C.c_void_p, C.POINTER(UrfStrip), C.c_int, C.c_void_p, C.c_int]
    return lib


def test_glue_compiles_against_shims_and_links():
    assert hasattr(_lib(), "urf_glue_run") and hasattr(_lib(), "urf_glue_run_cloud2")
    for node in ("urf_node.cpp", "urf_node_cloud2.cpp"):
        src = open(os.path.join(ROOT, "ros", node)).read()
        for topic in ('"road"', '"curb"', '"roi"', '"road_probably"', '"road_marker"'):      # lidar_segmentation.cpp:55-59
            assert topic in src


def test_catkin_package_files_name_what_exists():
    """ros/CMakeLists.txt, package.xml and the launch file (compile-checked only: no ROS here) refer to files and targets
    that exist, and keep the reference's node name and namespace (launch/demo1.launch:2-7 of the reference)."""
    cm = open(os.path.join(ROOT, "ros", "CMakeLists.txt")).read()
    for f in ("urf_node.cpp", "urf_node_cloud2.cpp"):
        assert f in cm and os.path.exists(os.path.join(ROOT, "ros", f))
    assert "urban_road_filter" in cm and "urf_b200" in cm
    import xml.etree.ElementTree as ET
    pkg = ET.parse(os.path.join(ROOT, "ros", "package.xml")).getroot()
    assert pkg.find("name").text == "urban_road_filter_b200"
    assert "urban_road_filter" in [d.text for d in pkg.findall("depend")]
    launch = ET.parse(os.path.join(ROOT, "ros", "launch", "demo1_b200.launch")).getroot()
    nodes = [n for g in launch.findall("group") if g.get("ns") == "urban_road_filter" for n in g.findall("node")]
    assert {n.get("type") for n in nodes} == {"lidar_road_b200", "lidar_road_b200_cloud2"}
    assert all(n.get("name") == "urban_road_filt" and n.get("pkg") == "urban_road_filter_b200" for n in nodes)


def _run(lib, g: Golden, prm, ghost_in, cloud2_step=0):
    pts = np.ascontiguousarray(g.cloud, np.float32)
    n = pts.shape[0]
    label, emit, prob = np.empty(n, np.int32), np.empty(n, np.int32), np.empty(n, np.int32)
    counts = np.zeros(8, np.int32)
    strips = (UrfStrip * 1024)()
    sp = np.zeros(3 * 4096, np.float64)
    if cloud2_step:
        ghost = lib.urf_glue_run_cloud2(pts.ctypes.data, n, C.byref(prm), max(n, 1024), ghost_in, cloud2_step, label.ctypes.data,
                                        emit.ctypes.data, prob.ctypes.data, counts.ctypes.data, strips, 1024, sp.ctypes.data, 4096)
    else:
        ghost = lib.urf_glue_run(pts.ctypes.data, n, C.byref(prm), max(n, 1024), ghost_in, label.ctypes.data, emit.ctypes.data,
                                 prob.ctypes.data, counts.ctypes.data, strips, 1024, sp.ctypes.data, 4096)
    assert ghost >= 0
    out = [(s.id, s.action, s.red, sp[3 * s.first: 3 * (s.first + s.count)].reshape(-1, 3).copy()) for s in strips[: counts[5]]]
    return label, emit, prob, counts, out, ghost


@pytest.mark.gpu
@pytest.mark.parametrize("step", [0, 48, 32])
@pytest.mark.parametrize("name", [n for n in golden_names() if "ties" not in n and not n.startswith("c5")])
def test_glue_publishes_what_the_reference_published(name, step):
    """step 0: ros/urf_node.cpp (PCL-typed callback); 48 / 32: ros/urf_node_cloud2.cpp fed a PointCloud2 with Ouster- or
    Velodyne-sized records."""
    lib = _lib()
    g = Golden(name)
    label, emit, prob, counts, strips, _ = _run(lib, g, g.params(simple_poly_allow=0, poly_z_avg_allow=0), 0, step)
    assert bool(counts[0]) == g.published
    if not g.published:
        return
    assert np.array_equal(label, g.label)
    assert np.array_equal(emit[: counts[2]], g.road_ids) and np.array_equal(emit[counts[2]: counts[2] + counts[3]], g.curb_ids)
    assert np.array_equal(prob[: counts[4]], g.prob_ids)
    assert bool(counts[7]) == g.markers_published
    compare_strips(strips, g.strips_raw, name + " raw strips")
    _, _, _, _, strips, ghost = _run(lib, g, g.params(), 3, step)
    compare_strips(strips, g.strips_cfg, name + " cfg strips")
    if g.markers_published:
        assert ghost == g.ghost_after

"""The ROS 2 node: ros2/urf_ros2_node.cpp (rclcpp component urf_b200::RoadFilterNode) compiled against the shim headers
of tests/ros2_shim, driven through the C entries of tests/kat/ros2_glue_entry.cpp.

Without a GPU: the library builds and exports its entries; the node's parameter table matches the reference's
LidarFilters.cfg (tests/golden/ref/lidarfilters_cfg.json) and ctypes_abi.DEFAULTS; the table checks refuse what they must;
a bad override stops the node before it touches a GPU; the ament package, CMake file and launch file name what exists.
With a GPU: every scan fed to the node's subscription publishes what the unmodified reference published (roi / road / curb /
road_probably point for point and in order, road_marker strip for strip, the input header on every cloud), parameter
updates apply from the next scan and refused ones change nothing, ghostcount carries from scan to scan, and refused
messages publish nothing and log one error."""
import ast
import ctypes as C
import json
import math
import os
import xml.etree.ElementTree as ET

import numpy as np
import pytest

from urban_road_filter_b200 import DEFAULTS, LABEL_CURB, LABEL_NONE, LABEL_OUTSIDE, LABEL_ROAD, make_params
from util import REF_DIR, ROOT, Golden, cloud2_records, compare_strips, golden_names

ROS2 = os.path.join(ROOT, "ros2")
CFG = json.load(open(os.path.join(REF_DIR, "lidarfilters_cfg.json")))
CFG_TYPES = {r["name"]: r["type"] for r in CFG}
READ_ONLY = {"topic_name", "device", "max_points", "channels", "reference_tie_order"}
TOPICS = ("road", "curb", "roi", "road_probably")
GOLDEN = [n for n in golden_names() if "ties" not in n and not n.startswith("c5")]
TYPE_CODE = {"bool": 1, "integer": 2, "double": 3, "string": 4}      # rclcpp::ParameterType
_P = [C.c_int, C.POINTER(C.c_char_p), C.POINTER(C.c_int), C.POINTER(C.c_double), C.POINTER(C.c_char_p)]

_LIB = None


def _lib():
    global _LIB
    if _LIB is None:
        lib = C.CDLL(os.path.join(ROOT, "build", "libglue_ros2.so"))
        lib.urf_ros2_create.restype = C.c_void_p
        lib.urf_ros2_create.argtypes = _P + [C.c_char_p, C.c_int]
        lib.urf_ros2_destroy.argtypes = [C.c_void_p]
        lib.urf_ros2_feed.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, C.c_int, C.c_int, C.POINTER(C.c_char_p),
                                      C.POINTER(C.c_int), C.POINTER(C.c_int), C.c_void_p, C.c_size_t, C.c_int32, C.c_uint32, C.c_char_p]
        lib.urf_ros2_cloud.argtypes = [C.c_void_p, C.c_char_p, C.c_char_p, C.c_int, C.c_void_p, C.c_size_t]
        lib.urf_ros2_markers.argtypes = [C.c_void_p, C.c_char_p, C.c_int]
        lib.urf_ros2_logs.argtypes = [C.c_char_p, C.c_int]
        lib.urf_ros2_set.argtypes = [C.c_void_p, C.c_int] + _P + [C.c_char_p, C.c_int]
        lib.urf_ros2_ghostcount.argtypes = [C.c_void_p, C.c_int]
        lib.urf_ros2_info.argtypes = [C.c_void_p, C.c_char_p, C.c_int]
        lib.urf_ros2_table.argtypes = [C.c_char_p, C.c_int]
        lib.urf_ros2_check.argtypes = _P + [C.c_char_p, C.c_int]
        _LIB = lib
    return _LIB


def _plist(params: dict):
    """rclcpp::Parameter list as C arrays: the Python type picks the parameter type (None: not set)."""
    n = len(params)
    names, types, nums, strs = (C.c_char_p * n)(), (C.c_int * n)(), (C.c_double * n)(), (C.c_char_p * n)()
    for k, (name, v) in enumerate(params.items()):
        names[k] = name.encode()
        if v is None:
            types[k] = 0
        elif isinstance(v, bool):
            types[k], nums[k] = 1, float(v)
        elif isinstance(v, int):
            types[k], nums[k] = 2, float(v)
        elif isinstance(v, float):
            types[k], nums[k] = 3, v
        else:
            types[k], strs[k] = 4, (v if isinstance(v, bytes) else str(v).encode())
    return n, names, types, nums, strs


def _json(fn, *args):
    size = fn(*args, None, 0)
    buf = C.create_string_buffer(size + 1)
    fn(*args, buf, size + 1)
    return json.loads(buf.value.decode())


def ros_params(over: dict) -> dict:
    """LidarFilters values (cfg names, cfg ints for bools as in make_params) as typed ROS 2 parameter values."""
    out = {}
    for k, v in over.items():
        t = CFG_TYPES.get(k, "int")
        out[k] = bool(v) if t == "bool" else int(v) if t == "int" else float(v) if t == "double" else v
    return out


def check(params: dict):
    """The node's table checks of one request against the default set: (accepted, reason)."""
    reason = C.create_string_buffer(1024)
    ok = _lib().urf_ros2_check(*_plist(params), reason, 1024)
    return bool(ok), reason.value.decode()


class NodeRefused(Exception):
    pass


class Node:
    """One RoadFilterNode created through its component registration with parameter overrides."""

    def __init__(self, **overrides):
        self.lib = _lib()
        err = C.create_string_buffer(1024)
        self.h = self.lib.urf_ros2_create(*_plist(overrides), err, 1024)
        if not self.h:
            raise NodeRefused(err.value.decode())

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.lib.urf_ros2_destroy(self.h)
        self.h = None

    def feed(self, data: bytes, width: int, height: int = 1, point_step: int = 48, row_step: int | None = None, fields=None,
             bigendian: bool = False, stamp=(1700000000, 123456789), frame: str = "os_sensor"):
        """fields: [(name, offset, datatype)], default x / y / z / intensity FLOAT32 at 0 / 4 / 8 / 16."""
        fields = fields if fields is not None else [("x", 0, 7), ("y", 4, 7), ("z", 8, 7), ("intensity", 16, 7)]
        nf = len(fields)
        fn = (C.c_char_p * nf)(*[f[0].encode() for f in fields])
        fo, ft = (C.c_int * nf)(*[f[1] for f in fields]), (C.c_int * nf)(*[f[2] for f in fields])
        buf = np.frombuffer(data, np.uint8)
        rs = width * point_step if row_step is None else row_step
        rc = self.lib.urf_ros2_feed(self.h, width, height, point_step, rs, int(bigendian), nf, fn, fo, ft, buf.ctypes.data, buf.size,
                                    stamp[0], stamp[1], frame.encode())
        assert rc == 0

    def cloud(self, topic: str):
        """(messages published on topic by the last feed, layout and header of the last one, its data)"""
        meta = C.create_string_buffer(4096)
        count = self.lib.urf_ros2_cloud(self.h, topic.encode(), meta, 4096, None, 0)
        assert count >= 0, topic
        m = json.loads(meta.value.decode())
        if m is None:
            return count, None, b""
        data = np.zeros(m["size"], np.uint8)
        self.lib.urf_ros2_cloud(self.h, topic.encode(), meta, 4096, data.ctypes.data, data.size)
        return count, m, data.tobytes()

    def markers(self):
        buf = C.create_string_buffer(1 << 22)
        count = self.lib.urf_ros2_markers(self.h, buf, 1 << 22)
        assert count >= 0
        return count, json.loads(buf.value.decode())

    def set(self, params: dict, atomic: bool = True):
        """(accepted requests, reasons of the refused ones)"""
        reason = C.create_string_buffer(4096)
        ok = self.lib.urf_ros2_set(self.h, int(atomic), *_plist(params), reason, 4096)
        return ok, reason.value.decode()

    def ghostcount(self, set_to: int = -1) -> int:
        return self.lib.urf_ros2_ghostcount(self.h, set_to)

    def info(self):
        return _json(self.lib.urf_ros2_info, self.h)

    def everything(self):
        """What the last feed published, byte for byte."""
        return [self.cloud(t) for t in TOPICS] + [self.markers()]


def logs():
    return _json(_lib().urf_ros2_logs)


# ---------------------------------------------------------------------------------------------------------- CPU

def test_ros2_glue_compiles_against_shims_and_links():
    lib = _lib()
    for entry in ("urf_ros2_create", "urf_ros2_destroy", "urf_ros2_feed", "urf_ros2_cloud", "urf_ros2_markers", "urf_ros2_logs",
                  "urf_ros2_set", "urf_ros2_ghostcount", "urf_ros2_info", "urf_ros2_table", "urf_ros2_check"):
        assert hasattr(lib, entry), entry
    src = open(os.path.join(ROS2, "urf_ros2_node.cpp")).read()
    for topic in ('"road"', '"curb"', '"roi"', '"road_probably"', '"road_marker"'):      # lidar_segmentation.cpp:55-59
        assert topic in src
    assert '"urban_road_filt"' in src and "RCLCPP_COMPONENTS_REGISTER_NODE(urf_b200::RoadFilterNode)" in src


def test_parameter_table_matches_the_reference_cfg():
    table = _json(_lib().urf_ros2_table)
    rows = {r["descriptor"]["name"]: r for r in table}
    assert len(rows) == len(table)
    cfg_rows = [r for r in table if r["cfg_field"] and r["descriptor"]["name"] != "channels"]
    assert [r["descriptor"]["name"] for r in cfg_rows] == [c["name"] for c in CFG]
    for c in CFG:
        r = rows[c["name"]]
        d = r["descriptor"]
        assert d["type"] == TYPE_CODE[{"int": "integer"}.get(c["type"], c["type"])], c["name"]
        assert r["default"] == c["default"] and type(r["default"]) is type(c["default"]), c["name"]
        assert d["description"], c["name"]
        if c["type"] == "double":
            assert d["floating_point_range"] == [[c["min"], c["max"], 0.0]] and d["integer_range"] == [], c["name"]
        elif c["type"] == "int":
            assert d["integer_range"] == [[c["min"], c["max"], 1]] and d["floating_point_range"] == [], c["name"]
        else:
            assert d["integer_range"] == [] and d["floating_point_range"] == [], c["name"]
        want = DEFAULTS[c["name"]]
        assert (want.decode() if isinstance(want, bytes) else want) == r["default"], c["name"]
    # the node parameters of the ROS1 nodes' private namespace, with the same defaults
    assert rows["channels"]["default"] == DEFAULTS["channels"] == 64
    assert rows["channels"]["descriptor"]["integer_range"] == [[1, 256, 1]]
    assert rows["device"]["default"] == 0 and rows["max_points"]["default"] == 1 << 20
    assert rows["reference_tie_order"]["default"] is False
    assert set(rows) == {c["name"] for c in CFG} | {"channels", "device", "max_points", "reference_tie_order"}
    assert {n for n, r in rows.items() if r["descriptor"]["read_only"]} == READ_ONLY
    assert rows["fixed_frame"]["descriptor"]["read_only"] is False


def test_table_checks_refuse_out_of_range_values():
    for bad in (dict(curb_points=31), dict(curb_points=0), dict(interval=0.005), dict(interval=10.5), dict(xDirection=3),
                dict(min_x=-200.5), dict(poly_s_param=1.0000001), dict(dmin_param=2), dict(max_z=math.inf)):
        ok, why = check(bad)
        (name,) = bad
        assert not ok and why.startswith(name + ":") and "outside" in why, (bad, why)
    for good in (dict(curb_points=30), dict(curb_points=1), dict(interval=0.01), dict(interval=10.0), dict(min_x=-200.0),
                 dict(poly_s_param=0.0), dict(xDirection=2)):
        assert check(good) == (True, ""), good
    # NaN passes a range check in rclcpp and here alike; urf_set_params decides it (GPU test below)
    assert check(dict(interval=math.nan)) == (True, "")


def test_table_checks_refuse_wrong_types():
    for bad in (dict(interval=1), dict(interval="0.2"), dict(x_zero_method=1), dict(curb_points=5.0), dict(curb_points=True),
                dict(fixed_frame=3), dict(starbeam_filter=None)):
        ok, why = check(bad)
        (name,) = bad
        assert not ok and why.startswith(name + ": expected a "), (bad, why)
    assert check(dict(fixed_frame="x" * 128)) == (False, "fixed_frame: longer than 127 bytes")
    assert check(dict(fixed_frame="base_link", x_zero_method=False, curb_points=7, interval=0.5)) == (True, "")


def test_table_checks_refuse_unknown_and_read_only_names():
    assert check(dict(no_such_parameter=1)) == (False, "no_such_parameter: no such parameter")
    assert check(dict(Interval=0.2))[0] is False
    for name, v in (("topic_name", "/points"), ("device", 1), ("max_points", 1000), ("channels", 32), ("reference_tie_order", True)):
        ok, why = check({name: v})
        assert not ok and why.startswith(name + ": read-only"), why


def test_one_bad_entry_refuses_the_whole_request():
    ok, why = check(dict(curb_points=12, interval=0.005, min_x=-20.0))
    assert not ok and why.startswith("interval:")
    ok, why = check(dict(curb_points=12, min_x=-20.0, channels=128))
    assert not ok and why.startswith("channels: read-only")


def test_bad_overrides_stop_the_node_before_it_touches_a_gpu():
    for over, start in ((dict(curb_points=31), "curb_points:"), (dict(interval=1), "interval: expected a double"),
                        (dict(channels=0), "channels:"), (dict(max_points=0), "max_points:"), (dict(max_points=(1 << 24) + 1), "max_points:"),
                        (dict(topic_name=5), "topic_name: expected a string")):
        with pytest.raises(NodeRefused) as e:
            Node(**over)
        assert str(e.value).startswith(start), (over, str(e.value))


def test_ament_package_files_name_what_exists():
    """ros2/package.xml, CMakeLists.txt and the launch file (compile-checked only: no ROS 2 here) refer to files and targets
    that exist, and keep the reference's node name and namespace."""
    pkg = ET.parse(os.path.join(ROS2, "package.xml")).getroot()
    assert pkg.get("format") == "3" and pkg.find("name").text == "urban_road_filter_b200"
    assert pkg.find("buildtool_depend").text == "ament_cmake" and pkg.find("export/build_type").text == "ament_cmake"
    deps = {d.text for d in pkg.findall("depend")}
    assert {"rclcpp", "rclcpp_components", "rcl_interfaces", "sensor_msgs", "visualization_msgs"} <= deps
    assert "urban_road_filter" not in deps and "dynamic_reconfigure" not in deps

    cm = open(os.path.join(ROS2, "CMakeLists.txt")).read()
    assert "add_library(urf_ros2_node SHARED urf_ros2_node.cpp)" in cm and os.path.exists(os.path.join(ROS2, "urf_ros2_node.cpp"))
    assert 'rclcpp_components_register_node(urf_ros2_node PLUGIN "urf_b200::RoadFilterNode" EXECUTABLE lidar_road_b200)' in cm
    assert "URF_B200_ROOT" in cm and "NAMES urf_b200" in cm and "ament_package()" in cm
    for d in ("rclcpp", "rclcpp_components", "rcl_interfaces", "sensor_msgs", "visualization_msgs"):
        assert f"find_package({d} REQUIRED)" in cm
    assert "install(DIRECTORY launch" in cm and os.path.isdir(os.path.join(ROS2, "launch"))

    tree = ast.parse(open(os.path.join(ROS2, "launch", "demo1_b200.launch.py")).read())
    calls = [n for n in ast.walk(tree) if isinstance(n, ast.Call) and isinstance(n.func, ast.Name)]
    nodes = [c for c in calls if c.func.id == "Node"]
    assert len(nodes) == 1
    kw = {k.arg: k.value for k in nodes[0].keywords}
    assert {k: ast.literal_eval(kw[k]) for k in ("package", "executable", "namespace", "name")} == dict(
        package="urban_road_filter_b200", executable="lidar_road_b200", namespace="urban_road_filter", name="urban_road_filt")
    args = {ast.literal_eval(c.args[0]) for c in calls if c.func.id == "DeclareLaunchArgument"}
    assert args == {"device", "max_points", "channels"}
    (params,) = kw["parameters"].elts
    assert {ast.literal_eval(k) for k in params.keys} == args
    launch_args = {ast.literal_eval(c.args[0]) for c in calls if c.func.id == "LaunchConfiguration"}
    assert launch_args == args
    assert {r["descriptor"]["name"] for r in _json(_lib().urf_ros2_table)} >= args


# ---------------------------------------------------------------------------------------------------------- GPU

def records(cloud, step: int, seed: int = 0):
    """The cloud as PointCloud2 records of `step` bytes, x / y / z at 0 / 4 / 8, the point's index (exact below 2^24) as the
    FLOAT32 intensity at 16 (at 12 in 16-byte records), other bytes seeded garbage. Returns (data, fields)."""
    pts = np.ascontiguousarray(cloud, np.float32).copy()
    pts[:, 3] = np.arange(pts.shape[0], dtype=np.float32)
    oi = 16 if step >= 20 else 12
    return cloud2_records(pts, step, 0, 4, 8, oi, seed).tobytes(), [("x", 0, 7), ("y", 4, 7), ("z", 8, 7), ("intensity", oi, 7)]


XYZI_FIELDS = [["x", 0, 7, 1], ["y", 4, 7, 1], ["z", 8, 7, 1], ["intensity", 16, 7, 1]]


def published_ids(node: Node, cloud, stamp, frame):
    """Input indices of the four published clouds (None when nothing was published), after checking each message's layout,
    header and records against the input."""
    cloud = np.ascontiguousarray(cloud, np.float32)
    out = {}
    for t in TOPICS:
        count, m, data = node.cloud(t)
        if count == 0:
            out[t] = None
            continue
        assert count == 1, t
        assert (m["frame_id"], m["sec"], m["nanosec"]) == (frame, stamp[0], stamp[1]), t
        assert m["fields"] == XYZI_FIELDS and m["point_step"] == 32 and m["height"] == 1, t
        assert m["row_step"] == 32 * m["width"] and m["size"] == m["row_step"] and not m["is_bigendian"] and m["is_dense"], t
        rec = np.frombuffer(data, np.float32).reshape(-1, 8)
        ids = rec[:, 4].astype(np.int64)
        assert np.array_equal(rec[:, 4], ids.astype(np.float32)) and ((ids >= 0) & (ids < cloud.shape[0])).all(), t
        assert np.array_equal(rec[:, :3].view(np.uint32), cloud[ids, :3].view(np.uint32)), t
        assert (rec[:, 3] == 1.0).all(), t
        out[t] = ids
    return out


def published_strips(node: Node, fixed_frame: str):
    """road_marker strips as (id, action, red, xyz) once the constant fields of every Marker are checked, or None."""
    count, markers = node.markers()
    if count == 0:
        return None
    assert count == 1
    out = []
    for m in markers:
        assert m["frame_id"] == fixed_frame and (m["sec"], m["nanosec"]) == (0, 0) and m["type"] == 4 and m["action"] in (0, 2)
        assert m["orientation"] == [0, 0, 0, 1] and m["scale"] == [0.5, 0.5, 0.5] and m["lifetime"] == [0, 0]
        assert m["color"] in ([1, 0, 0, 1], [0, 1, 0, 1])
        out.append((m["id"], m["action"], int(m["color"][0] == 1), np.array(m["points"], np.float64).reshape(-1, 3)))
    return out


def run_scan(node: Node, cloud, step: int = 48, height: int = 1, stamp=(1700000000, 123456789), frame="os_sensor", ghost=None):
    if ghost is not None:
        node.ghostcount(ghost)
    data, fields = records(cloud, step)
    n = cloud.shape[0]
    assert n % height == 0
    node.feed(data, n // height, height, step, fields=fields, stamp=stamp, frame=frame)
    return published_ids(node, cloud, stamp, frame)


def assert_golden_clouds(g: Golden, ids):
    assert (ids["roi"] is not None) == g.published
    if not g.published:
        assert all(v is None for v in ids.values())
        return
    label = np.full(g.cloud.shape[0], LABEL_OUTSIDE, np.int32)
    label[ids["roi"]] = LABEL_NONE
    label[ids["road"]] = LABEL_ROAD
    label[ids["curb"]] = LABEL_CURB
    assert np.array_equal(ids["roi"], np.sort(ids["roi"])), "roi keeps the input order"
    assert np.array_equal(label, g.label)
    assert np.array_equal(ids["road"], g.road_ids) and np.array_equal(ids["curb"], g.curb_ids)
    assert np.array_equal(ids["road_probably"], g.prob_ids)


def golden_overrides(g: Golden, **extra):
    return ros_params({**g.params_over, **extra})


@pytest.mark.gpu
@pytest.mark.parametrize("step", [48, 32, 16])
@pytest.mark.parametrize("name", GOLDEN)
def test_ros2_node_publishes_what_the_reference_published(name, step):
    g = Golden(name)
    mp = max(g.cloud.shape[0], 1024)
    with Node(max_points=mp, **golden_overrides(g, simple_poly_allow=0, poly_z_avg_allow=0)) as node:
        assert_golden_clouds(g, run_scan(node, g.cloud, step))
        strips = published_strips(node, DEFAULTS["fixed_frame"].decode())
        assert (strips is not None) == g.markers_published
        if strips is not None:
            compare_strips(strips, g.strips_raw, name + " raw strips")
        assert logs() == []
    if not g.markers_published:
        return
    with Node(max_points=mp, **golden_overrides(g)) as node:
        assert_golden_clouds(g, run_scan(node, g.cloud, step, ghost=3))
        compare_strips(published_strips(node, DEFAULTS["fixed_frame"].decode()), g.strips_cfg, name + " cfg strips")
        assert node.ghostcount() == g.ghost_after


@pytest.mark.gpu
def test_ros2_node_organized_cloud():
    """height > 1 with row_step = width * point_step: the rows are one run of records."""
    g = Golden("c1_full_s0")
    with Node(max_points=g.cloud.shape[0], **golden_overrides(g)) as node:
        assert_golden_clouds(g, run_scan(node, g.cloud, 32, height=16, ghost=3))
        compare_strips(published_strips(node, DEFAULTS["fixed_frame"].decode()), g.strips_cfg, "organized cfg strips")


@pytest.mark.gpu
def test_ros2_node_name_topics_qos_and_declared_parameters():
    with Node(max_points=4096, topic_name="/sensing/lidar/points", fixed_frame="base_link", curb_points=7) as node:
        info = node.info()
        assert info["name"] == "urban_road_filt" and info["callbacks"] == 1
        assert info["subscriptions"] == {"/sensing/lidar/points": {"reliability": "best_effort", "depth": 1}}
        rel = {"reliability": "reliable", "depth": 1}
        assert info["publishers"] == {"road": ["PointCloud2", rel], "curb": ["PointCloud2", rel], "roi": ["PointCloud2", rel],
                                      "road_probably": ["PointCloud2", rel], "road_marker": ["MarkerArray", rel]}
        table = {r["descriptor"]["name"]: r for r in _json(_lib().urf_ros2_table)}
        assert set(info["parameters"]) == set(table)
        for name, p in info["parameters"].items():
            assert p["descriptor"] == table[name]["descriptor"], name
        vals = {k: p["value"] for k, p in info["parameters"].items()}
        assert vals["topic_name"] == "/sensing/lidar/points" and vals["fixed_frame"] == "base_link" and vals["curb_points"] == 7
        assert vals["max_points"] == 4096 and vals["interval"] == 0.18
        assert [lvl for lvl, _ in logs()] == ["I"]


@pytest.mark.gpu
def test_ros2_node_parameter_updates_apply_from_the_next_scan():
    # one parameter (set_parameters): everything but curb_points at construction, then curb_points alone
    g = Golden("c1_full_noblind_cp12")
    over = golden_overrides(g)
    curb_points = over.pop("curb_points")
    with Node(max_points=g.cloud.shape[0], **over) as node:
        before = run_scan(node, g.cloud, 48, ghost=3)
        assert not np.array_equal(before["curb"], g.curb_ids), "the fixture's curb_points changes the curb cloud"
        assert node.set({"curb_points": curb_points}, atomic=False) == (1, "")
        assert_golden_clouds(g, run_scan(node, g.cloud, 48, ghost=3))
        compare_strips(published_strips(node, DEFAULTS["fixed_frame"].decode()), g.strips_cfg, "single update cfg strips")
        assert node.ghostcount() == g.ghost_after
    # several parameters in one atomic request, from a node started with the defaults
    g = Golden("c1_full_xdir1_cp3")
    with Node(max_points=g.cloud.shape[0]) as node:
        assert run_scan(node, g.cloud, 32)["roi"] is not None
        assert node.set(golden_overrides(g, simple_poly_allow=0, poly_z_avg_allow=0, fixed_frame="map")) == (1, "")
        assert_golden_clouds(g, run_scan(node, g.cloud, 32, ghost=0))
        compare_strips(published_strips(node, "map"), g.strips_raw, "atomic update raw strips")
        assert node.set(dict(simple_poly_allow=True, poly_z_avg_allow=True)) == (1, "")
        assert_golden_clouds(g, run_scan(node, g.cloud, 32, ghost=3))
        compare_strips(published_strips(node, "map"), g.strips_cfg, "atomic update cfg strips")


@pytest.mark.gpu
def test_ros2_node_refused_updates_change_nothing():
    g = Golden("c1_full_xonly")
    with Node(max_points=g.cloud.shape[0], **golden_overrides(g)) as node:
        assert run_scan(node, g.cloud, 48, ghost=0)["roi"] is not None
        before = node.everything()
        assert before[-1][0] == 1
        for req, atomic, start in ((dict(curb_points=31), True, "curb_points:"),
                                   (dict(interval=1), True, "interval: expected a double"),
                                   (dict(channels=128), True, "channels: read-only"),
                                   (dict(topic_name="/other"), False, "topic_name: read-only"),
                                   (dict(no_such_parameter=1.0), False, "no_such_parameter: no such parameter"),
                                   (dict(interval=math.nan), True, "urf_set_params refused"),
                                   (dict(curb_height=math.nan), False, "urf_set_params refused"),
                                   (dict(curb_points=12, blind_spots=False, interval=0.005), True, "interval:")):
            ok, why = node.set(req, atomic=atomic)
            assert ok == 0 and why.startswith(start), (req, why)
            assert run_scan(node, g.cloud, 48, ghost=0)["roi"] is not None
            assert node.everything() == before, req
        assert node.info()["parameters"]["curb_points"]["value"] == 5


@pytest.mark.gpu
def test_ros2_node_carries_ghostcount_between_scans():
    from urban_road_filter_b200 import api
    a, b = Golden("c2_default_s0"), Golden("c1_default_ring_s1")
    with Node(max_points=a.cloud.shape[0]) as node:
        run_scan(node, a.cloud, 48)
        ghost_a = node.ghostcount()
        assert_golden_clouds(b, run_scan(node, b.cloud, 32))
        strips = published_strips(node, DEFAULTS["fixed_frame"].decode())
        ghost_b = node.ghostcount()
    det = api.Detector(max_points=b.cloud.shape[0], params=make_params())
    try:
        want, want_ghost = api.build_markers(make_params(), det.filtered(b.cloud).vert, ghost_a)
    finally:
        det.close()
    assert any(s[1] == 2 for s in want), "the second scan deletes ghosts of the first"
    assert len(strips) == len(want) and ghost_b == want_ghost
    for s, w in zip(strips, want):
        assert s[:3] == w[:3] and np.array_equal(s[3], w[3])


@pytest.mark.gpu
def test_ros2_node_refused_messages_publish_nothing_and_log_one_error():
    g = Golden("c1_full_s0")
    n = g.cloud.shape[0]
    data, fields = records(g.cloud, 48)
    bigger, _ = records(np.concatenate([g.cloud, g.cloud[:1]]), 48)
    wide = np.frombuffer(records(g.cloud, 64)[0], np.uint8).reshape(n, 64)
    step72 = np.concatenate([wide, np.zeros((n, 8), np.uint8)], 1).tobytes()
    cases = {
        "no z field": dict(data=data, width=n, fields=[f for f in fields if f[0] != "z"]),
        "z not FLOAT32": dict(data=data, width=n, fields=[(f[0], f[1], 8 if f[0] == "z" else 7) for f in fields]),
        "big-endian": dict(data=data, width=n, fields=fields, bigendian=True),
        "point_step 72": dict(data=step72, width=n, point_step=72, fields=fields),
        "more than max_points": dict(data=bigger, width=n + 1, fields=fields),
        "truncated data": dict(data=data[:-1], width=n, fields=fields),
        "padded rows": dict(data=data + bytes(16 * 8), width=n // 16, height=16, row_step=(n // 16) * 48 + 8, fields=fields),
    }
    with Node(max_points=n, **golden_overrides(g)) as node:
        for what, kw in cases.items():
            node.feed(**kw)
            assert all(node.cloud(t)[0] == 0 for t in TOPICS) and node.markers()[0] == 0, what
            errs = logs()
            assert len(errs) == 1 and errs[0][0] == "E" and "unsupported PointCloud2" in errs[0][1], (what, errs)
            assert_golden_clouds(g, run_scan(node, g.cloud, 48, ghost=3))
            compare_strips(published_strips(node, DEFAULTS["fixed_frame"].decode()), g.strips_cfg, what)
            assert logs() == []
        tiny = Golden("tiny29")
        assert all(v is None for v in run_scan(node, tiny.cloud, 48).values())
        assert node.markers()[0] == 0 and logs() == []

"""ROS1 bag reading and writing (urban_road_filter_b200/rosbag.py) and the replay around stand-in devices
(urban_road_filter_b200/replay.py), without a GPU.

The reader is checked against bags built byte by byte here, from the format specification (wiki.ros.org/Bags/Format/2.0)
and without the writer: uncompressed and bz2 chunks, several chunks whose times interleave, two connections on one topic,
and the lz4 / unindexed / wrong-version refusals. The writer is checked by reading its bags back, here and with the
reader, down to the 4096-byte bag header and the index fields. The md5sums are pinned to the ROS Noetic values."""
import bz2
import ctypes as C
import struct

import numpy as np
import pytest

from urban_road_filter_b200 import api, make_params, rosbag
from urban_road_filter_b200.api import build_markers
from urban_road_filter_b200.ctypes_abi import URF_TOO_FEW_POINTS, UrfFormatsUser
from urban_road_filter_b200.replay import ReplayError, parse_sets, replay
from urban_road_filter_b200.rosbag import (BagError, BagReader, BagWriter, Header, Marker, PointCloud2, PointField, Time,
                                           cloud_format)

# ---------------------------------------------------------------------------------------------------------------------
# a bag, byte by byte


def u32(v):
    return struct.pack("<I", v)


def record(fields, data=b""):
    h = b"".join(u32(len(k) + 1 + len(v)) + k.encode() + b"=" + v for k, v in fields)
    return u32(len(h)) + h + u32(len(data)) + data


def conn_record(cid, topic, typ="std_msgs/String"):
    conn = b"".join(u32(len(k) + 1 + len(v)) + k.encode() + b"=" + v for k, v in
                    [("topic", topic.encode()), ("type", typ.encode()), ("md5sum", b"992ce8a1687cec8c8bd883ec73ca41d1"),
                     ("message_definition", b"string data\n")])
    return record([("op", b"\x07"), ("conn", u32(cid)), ("topic", topic.encode())], conn)


def build_bag(chunks, conns, version=b"#ROSBAG V2.0\n", indexed=True):
    """chunks: [(compression, [(conn id, (secs, nsecs), payload)])]; conns: {id: topic}. Returns the bag's bytes."""
    body, infos, seen = b"", [], set()
    base = len(version) + 4096
    for comp, msgs in chunks:
        raw, index = b"", {}
        for cid, (s, ns), payload in msgs:
            if cid not in seen:
                raw += conn_record(cid, conns[cid])
                seen.add(cid)
            index.setdefault(cid, []).append((s, ns, len(raw)))
            raw += record([("op", b"\x02"), ("conn", u32(cid)), ("time", struct.pack("<II", s, ns))], payload)
        data = bz2.compress(raw) if comp == "bz2" else raw
        pos = base + len(body)
        body += record([("op", b"\x05"), ("compression", comp.encode()), ("size", u32(len(raw)))], data)
        for cid, ents in sorted(index.items()):
            body += record([("op", b"\x04"), ("ver", u32(1)), ("conn", u32(cid)), ("count", u32(len(ents)))],
                           b"".join(struct.pack("<III", *e) for e in ents))
        times = [t for _, t, _ in msgs]
        infos.append((pos, min(times), max(times), {c: len(e) for c, e in sorted(index.items())}))
    index_pos = base + len(body)
    for cid, topic in conns.items():
        body += conn_record(cid, topic)
    for pos, t0, t1, counts in infos:
        body += record([("op", b"\x06"), ("ver", u32(1)), ("chunk_pos", struct.pack("<Q", pos)),
                        ("start_time", struct.pack("<II", *t0)), ("end_time", struct.pack("<II", *t1)),
                        ("count", u32(len(counts)))], b"".join(struct.pack("<II", c, m) for c, m in counts.items()))
    h = record([("op", b"\x03"), ("index_pos", struct.pack("<Q", index_pos if indexed else 0)), ("conn_count", u32(len(conns))),
                ("chunk_count", u32(len(infos)))])
    hdr = h[:-4]
    header = hdr + u32(4096 - len(hdr) - 4) + b" " * (4096 - len(hdr) - 4)
    assert len(header) == 4096
    return version + header + body


def parse_records(buf, pos, end=None):
    """[(position, header fields, data)] of the records from pos to end."""
    end = len(buf) if end is None else end
    out = []
    while pos < end:
        (hl,) = struct.unpack_from("<I", buf, pos)
        fields, p = {}, pos + 4
        while p < pos + 4 + hl:
            (n,) = struct.unpack_from("<I", buf, p)
            k, _, v = buf[p + 4: p + 4 + n].partition(b"=")
            fields[k.decode()] = v
            p += 4 + n
        (dl,) = struct.unpack_from("<I", buf, p)
        out.append((pos, fields, buf[p + 4: p + 4 + dl]))
        pos = p + 4 + dl
    return out


def write(tmp_path, name, data):
    p = tmp_path / name
    p.write_bytes(data)
    return str(p)


MSGS = {  # chunk contents: times interleave across chunks, connections 0 and 1 share /a
    "c0": [(0, (5, 0), b"a5"), (2, (1, 500), b"b1.5"), (0, (2, 0), b"a2")],
    "c1": [(1, (3, 0), b"a3-other-publisher"), (2, (4, 0), b"b4"), (0, (5, 0), b"a5-second")],
}
CONNS = {0: "/a", 1: "/a", 2: "/b"}


@pytest.mark.parametrize("comps", [("none", "none"), ("bz2", "bz2"), ("none", "bz2")])
def test_reader_reads_a_bag_built_from_the_specification(tmp_path, comps):
    path = write(tmp_path, "in.bag", build_bag([(comps[0], MSGS["c0"]), (comps[1], MSGS["c1"])], CONNS))
    with BagReader(path) as r:
        assert {c.id: c.topic for c in r.connections.values()} == CONNS
        assert all(c.type == "std_msgs/String" and c.message_definition == "string data\n" for c in r.connections.values())
        assert len(r.chunks) == 2 and [sum(ci.counts.values()) for ci in r.chunks] == [3, 3]
        got = [(topic, conn.id, tuple(t), bytes(d)) for topic, conn, t, d in r.messages()]
        # time order; equal times (5, 0) in file order
        assert got == [("/b", 2, (1, 500), b"b1.5"), ("/a", 0, (2, 0), b"a2"), ("/a", 1, (3, 0), b"a3-other-publisher"),
                       ("/b", 2, (4, 0), b"b4"), ("/a", 0, (5, 0), b"a5"), ("/a", 0, (5, 0), b"a5-second")]
        assert [bytes(d) for _, _, _, d in r.messages({"/a"})] == [b"a2", b"a3-other-publisher", b"a5", b"a5-second"]
        if comps[0] == "none":         # a view of the file's mapping, not a copy
            _, _, _, d = next(iter(r.messages({"/b"})))
            assert isinstance(d, memoryview) and d.obj is r._buf.obj


@pytest.mark.parametrize("case, msg", [
    ("lz4", "lz4-compressed chunks are not supported"),
    ("unindexed", "not indexed (index_pos 0): run `rosbag reindex`"),
    ("v12", "bag version 1.2; only 2.0 is supported"),
    ("garbage", "not a ROS bag"),
])
def test_reader_refusals(tmp_path, case, msg):
    if case == "lz4":
        data = build_bag([("lz4", MSGS["c0"])], CONNS)
    elif case == "unindexed":
        data = build_bag([("none", MSGS["c0"])], CONNS, indexed=False)
    elif case == "v12":
        data = build_bag([("none", MSGS["c0"])], CONNS, version=b"#ROSBAG V1.2\n")
    else:
        data = b"not a bag at all\n" * 10
    with pytest.raises(BagError, match=msg.replace("(", r"\(").replace(")", r"\)").replace(".", r"\.")):
        BagReader(write(tmp_path, "bad.bag", data))


@pytest.mark.parametrize("compression", ["none", "bz2"])
def test_writer_round_trip_and_index_fields(tmp_path, compression):
    path = str(tmp_path / "out.bag")
    rng = np.random.default_rng(1)
    sent = []
    with BagWriter(path, compression, chunk_threshold=2000) as w:
        for k in range(40):
            topic = ("/x", "/y/z", "/w")[k % 3]
            t = Time(100 + k // 2, 1000 * k)
            payload = rng.integers(0, 256, int(rng.integers(1, 300)), dtype=np.uint8).tobytes()
            w.write(topic, rosbag.POINTCLOUD2 if topic != "/w" else rosbag.MARKERARRAY, t, payload)
            sent.append((topic, t, payload))
    buf = open(path, "rb").read()
    assert buf[:13] == b"#ROSBAG V2.0\n"
    recs = parse_records(buf, 13)
    pos0, hdr, pad = recs[0]
    assert hdr["op"] == b"\x03" and recs[1][0] == 13 + 4096 and set(pad) == {0x20}      # the header record is 4096 bytes
    index_pos = struct.unpack("<Q", hdr["index_pos"])[0]
    conn_count, chunk_count = struct.unpack("<I", hdr["conn_count"])[0], struct.unpack("<I", hdr["chunk_count"])[0]
    ops = [f["op"][0] for _, f, _ in recs]
    assert ops.count(5) == chunk_count > 2 and conn_count == 3
    tail = [(p, f) for p, f, _ in recs if p >= index_pos]
    assert tail[0][0] == index_pos and [f["op"][0] for _, f in tail] == [7] * 3 + [6] * chunk_count
    conns = {struct.unpack("<I", f["conn"])[0]: f["topic"].decode() for _, f in tail[:3]}
    assert sorted(conns.values()) == ["/w", "/x", "/y/z"]
    chunk_pos = [p for p, f, _ in recs if f["op"] == b"\x05"]
    infos = [(p, f, d) for p, f, d in recs if f["op"] == b"\x06"]
    assert [struct.unpack("<Q", f["chunk_pos"])[0] for _, f, _ in infos] == chunk_pos
    total = 0
    for _, f, d in infos:
        counts = dict(struct.iter_unpack("<II", d))
        assert len(counts) == struct.unpack("<I", f["count"])[0]
        total += sum(counts.values())
    assert total == 40
    for p, f, d in recs:
        if f["op"] == b"\x05":
            assert f["compression"].decode() == compression
            raw = bz2.decompress(d) if compression == "bz2" else d
            assert len(raw) == struct.unpack("<I", f["size"])[0]
    with BagReader(path) as r:
        got = [(topic, tuple(t), bytes(d)) for topic, _, t, d in r.messages()]
        types = {c.topic: (c.type, c.md5sum) for c in r.connections.values()}
    assert got == [(topic, tuple(t), p) for topic, t, p in sent]
    assert types["/w"] == ("visualization_msgs/MarkerArray", "d155b9ce5188fbaf89745847fd5882d7")
    assert types["/x"] == ("sensor_msgs/PointCloud2", "1158d486dd51d683ce2f1be655c3c181")


def test_md5sums_are_the_noetic_values():
    assert rosbag.POINTCLOUD2.md5sum == "1158d486dd51d683ce2f1be655c3c181"
    assert rosbag.MARKERARRAY.md5sum == "d155b9ce5188fbaf89745847fd5882d7"
    assert rosbag.md5sum("std_msgs/Header") == "2176decaecbce78abc3b96ef049fabed"
    assert rosbag.md5sum("visualization_msgs/Marker") == "4048c9de2a16f4ae8e0538085ebf1b97"
    d = rosbag.MARKERARRAY.definition
    assert d.startswith("Marker[] markers\n") and [ln for ln in d.splitlines() if ln.startswith("MSG: ")] == [
        "MSG: visualization_msgs/Marker", "MSG: std_msgs/Header", "MSG: geometry_msgs/Pose", "MSG: geometry_msgs/Point",
        "MSG: geometry_msgs/Quaternion", "MSG: geometry_msgs/Vector3", "MSG: std_msgs/ColorRGBA"]


OUSTER_FIELDS = [PointField("x", 0, 7, 1), PointField("y", 4, 7, 1), PointField("z", 8, 7, 1), PointField("intensity", 16, 7, 1),
                 PointField("t", 20, 6, 1), PointField("reflectivity", 24, 4, 1), PointField("ring", 26, 2, 1),
                 PointField("ambient", 28, 4, 1), PointField("range", 32, 6, 1)]
VELO22_FIELDS = [PointField("x", 0, 7, 1), PointField("y", 4, 7, 1), PointField("z", 8, 7, 1), PointField("intensity", 12, 7, 1),
                 PointField("ring", 16, 4, 1), PointField("time", 18, 7, 1)]


def cloud(fields, step, width, height=1, data=None, row_step=None, big=False, stamp=Time(7, 8), frame="os1"):
    data = bytes(range(256)) * (width * height * step // 256 + 1) if data is None else data
    return PointCloud2(Header(3, stamp, frame), height, width, fields, big, step,
                       width * step if row_step is None else row_step, data[: width * height * step], True)


def test_pointcloud2_and_markerarray_round_trip():
    msg = cloud(OUSTER_FIELDS, 48, 5, 2)
    back = rosbag.decode_cloud2(rosbag.encode_cloud2(msg))
    assert back.header == msg.header and back.fields == msg.fields and bytes(back.data) == msg.data
    assert (back.height, back.width, back.point_step, back.row_step, back.is_bigendian, back.is_dense) == (2, 5, 48, 240, False, True)
    ms = [Marker(Header(1, Time(2, 3), "map"), "ns", 4, 4, 0, (1.0, 2.0, 3.0), (0.0, 0.0, 0.5, 0.5), (0.5, 0.5, 0.5),
                 (1.0, 0.0, 0.0, 1.0), (5, 6), True, [(1.5, 2.5, -1.0), (3.0, 4.0, -1.25)], [(0.0, 1.0, 0.0, 1.0)], "t", "m", True),
          Marker(action=2, id=7)]
    assert rosbag.decode_marker_array(rosbag.encode_marker_array(ms)) == ms
    for n in (0, 3):                                       # clouds given as numpy record arrays, empty ones included
        packed = np.arange(8 * n, dtype=np.float32).reshape(n, 8)
        back = rosbag.decode_cloud2(rosbag.encode_cloud2(PointCloud2(msg.header, 1, n, msg.fields, False, 32, 32 * n, packed, True)))
        assert back.width == n and bytes(back.data) == packed.tobytes()
    with pytest.raises(BagError, match="ends inside a field"):
        rosbag.decode_cloud2(rosbag.encode_cloud2(msg)[:-3])


def test_record_formats_of_the_topics():
    assert cloud_format(cloud(OUSTER_FIELDS, 48, 4), "/os1") == api.CloudFormat(48, 0, 4, 8, 16)
    assert cloud_format(cloud(VELO22_FIELDS, 22, 4), "/velo") == api.CloudFormat(22, 0, 4, 8, 12)
    assert cloud_format(cloud(OUSTER_FIELDS[:3], 16, 4), "/xyz") == api.CloudFormat(16, 0, 4, 8, -1)
    uint_i = OUSTER_FIELDS[:3] + [PointField("intensity", 12, 4, 1)]           # not FLOAT32: no intensity, as the glue node
    assert cloud_format(cloud(uint_i, 16, 4), "/u") == api.CloudFormat(16, 0, 4, 8, -1)
    org = cloud(OUSTER_FIELDS, 48, 8, 4)
    assert cloud_format(org, "/org") == api.CloudFormat(48, 0, 4, 8, 16) and org.width * org.height == 32
    f64 = [PointField("x", 0, 8, 1), PointField("y", 8, 7, 1), PointField("z", 12, 7, 1)]
    for msg, err in [(cloud(f64, 16, 4), "/t: field 'x' is FLOAT64, not FLOAT32"),
                     (cloud(OUSTER_FIELDS[1:], 48, 4), "/t: PointCloud2 has no field 'x'"),
                     (cloud(OUSTER_FIELDS, 48, 4, big=True), "/t: big-endian"),
                     (cloud(OUSTER_FIELDS, 48, 4, 2, row_step=200), r"/t: row_step 200 != width 4 \* point_step 48"),
                     (cloud(OUSTER_FIELDS, 48, 4, data=b"\0" * 100), "/t: 100 data bytes hold fewer than 4 x 1 records"),
                     (cloud(OUSTER_FIELDS, 80, 4), r"/t: point_step 80 is outside \[12, 64\]")]:
        with pytest.raises(BagError, match=err):
            cloud_format(msg, "/t")


# ---------------------------------------------------------------------------------------------------------------------
# the replay around stand-in devices

XYZI16 = [PointField("x", 0, 7, 1), PointField("y", 4, 7, 1), PointField("z", 8, 7, 1), PointField("intensity", 12, 7, 1)]


def scan_points(n, ctrl, seed):
    """n points whose first y carries the stand-in's control value `ctrl` (-1: fail the batch, else marker colour runs)."""
    p = np.random.default_rng(seed).uniform(-20, 20, (n, 4)).astype(np.float32)
    if n:
        p[0, 1] = ctrl
    return p


def as_message(p, fmt_fields, step, stamp):
    rec = np.zeros((p.shape[0], step), np.uint8)
    offs = {f.name: f.offset for f in fmt_fields}
    for k, name in enumerate(("x", "y", "z", "intensity")):
        if name in offs:
            rec[:, offs[name]: offs[name] + 4] = p[:, k: k + 1].copy().view(np.uint8)
    return rosbag.encode_cloud2(cloud(fmt_fields, step, p.shape[0], data=rec.tobytes(), stamp=stamp, frame="lidar"))


def vertices(ctrl):
    """3 * ctrl marker vertices in colour runs of 3 (ctrl runs: ctrl - 1 colour changes)."""
    v = np.zeros((3 * ctrl, 4), np.float32)
    v[:, 0] = np.arange(3 * ctrl)
    v[:, 1] = 0.5 * np.arange(3 * ctrl)
    v[:, 2] = -1.5
    v[:, 3] = (np.arange(3 * ctrl) // 3) % 2
    return v


def stand_in(user, xyzi, n, batch, outs):
    """Labels (i % 4) - 1, the ROI points in reverse input order as the emission order over 12 rings, and the vertices
    of scan_points' control value; fewer than 5 points: URF_TOO_FEW_POINTS; control -1: the batch fails."""
    u = C.cast(user, C.POINTER(UrfFormatsUser)).contents
    for j in range(batch):
        f = u.formats[u.fmt[j]]
        nj = n[j]
        rec = np.ctypeslib.as_array(C.cast(xyzi[j], C.POINTER(C.c_uint8)), shape=(max(nj, 1) * f.point_step,))
        rec = rec[: nj * f.point_step].reshape(nj, f.point_step)
        ctrl = int(rec[0, f.off_y: f.off_y + 4].copy().view(np.float32)[0]) if nj else 0
        if ctrl == -1:
            return -3
        out = outs[j]
        out.n_in = nj
        if nj < 5:
            out.status, out.n_roi, out.n_order, out.n_rings, out.n_vert = URF_TOO_FEW_POINTS, 0, 0, 0, 0
            continue
        lab = (np.arange(nj) % 4 - 1).astype(np.int32)
        np.ctypeslib.as_array(out.label, shape=(nj,))[:] = lab
        order = np.flatnonzero(lab >= 0)[::-1].astype(np.int32)
        np.ctypeslib.as_array(out.order, shape=(order.size,))[:] = order
        rs = np.linspace(0, order.size, 13).astype(np.int32)
        np.ctypeslib.as_array(out.ring_start, shape=(13,))[:] = rs
        v = vertices(ctrl)
        np.ctypeslib.as_array(out.vert)[: v.shape[0]] = v
        out.status, out.n_roi, out.n_order, out.n_rings, out.n_vert = 0, order.size, order.size, 12, v.shape[0]
    return 0


def expected_clouds(p):
    n = p.shape[0]
    rec = np.zeros((n, 8), np.float32)
    rec[:, :3], rec[:, 3], rec[:, 4] = p[:, :3], 1.0, p[:, 3]
    lab = np.arange(n) % 4 - 1
    order = np.flatnonzero(lab >= 0)[::-1]
    rs = np.linspace(0, order.size, 13).astype(np.int32)
    return {"roi": rec[lab >= 0], "road": rec[order[lab[order] == 1]], "curb": rec[order[lab[order] == 2]],
            "road_probably": rec[order[rs[10]: rs[11]]]}


# (topic, time, points, control); /velo has 22-byte packed records, /os1_* 48-byte ones
SCANS = [("/os1_a/points", (10, 0), 40, 5), ("/velo/points", (10, 5), 30, 1), ("/os1_b/points", (10, 9), 3, 2),
         ("/os1_a/points", (11, 0), 44, 2), ("/velo/points", (11, 1), 36, 3), ("/os1_b/points", (11, 2), 20, 2),
         ("/os1_a/points", (12, 0), 48, 1), ("/velo/points", (12, 2), 12, 1)]


def drive(tmp_path, scans=SCANS, name="drive.bag"):
    path = str(tmp_path / name)
    pts = {}
    with BagWriter(path, chunk_threshold=3000) as w:
        for k, (topic, t, n, ctrl) in enumerate(reversed(scans)):        # written out of time order; the index sorts
            p = scan_points(n, ctrl, k)
            pts[(topic, t)] = p
            fields, step = (VELO22_FIELDS, 22) if topic.startswith("/velo") else (OUSTER_FIELDS, 48)
            w.write(topic, rosbag.POINTCLOUD2, Time(*t), as_message(p, fields, step, Time(*t)))
    return path, pts


def read_all(path):
    out = {}
    with BagReader(path) as r:
        for topic, conn, t, d in r.messages():
            out.setdefault(topic, []).append((conn.type, tuple(t), bytes(d)))
    return out


def test_replay_around_stand_in_devices(tmp_path):
    src, pts = drive(tmp_path)
    prm = make_params(fixed_frame="base_link")
    rep = replay(src, str(tmp_path / "out.bag"), devices=(0, 1, 2), slots=2, batch=2, params=prm, process_fn=stand_in)
    assert rep.scans == {"/os1_a/points": 3, "/os1_b/points": 2, "/velo/points": 3}
    assert rep.published == {"/os1_a/points": 3, "/os1_b/points": 1, "/velo/points": 3}
    out = read_all(str(tmp_path / "out.bag"))
    topics = {s[0] for s in SCANS}
    # /os1_b/points' first scan (3 points) is URF_TOO_FEW_POINTS: nothing written for it. Scans whose control value is 1
    # have 3 vertices of one colour and get a MarkerArray too.
    assert set(out) == {f"{t}/{k}" for t in topics for k in ("road", "curb", "roi", "road_probably", "road_marker")}
    for topic in topics:
        mine = [(t, n, c) for tp, t, n, c in SCANS if tp == topic and n >= 5]
        ghost = 0
        for (t, n, ctrl), (typ, tm, data) in zip(mine, out[f"{topic}/road_marker"]):
            assert typ == "visualization_msgs/MarkerArray" and tm == t
            strips, ghost = build_markers(prm, vertices(ctrl), ghost)                # the topic's own ghostcount
            ms = rosbag.decode_marker_array(data)
            assert [(m.id, m.action) for m in ms] == [(s[0], 2 if s[1] == 2 else 0) for s in strips]
            for m, s in zip(ms, strips):
                assert m.header.frame_id == "base_link" and m.type == 4 and m.scale == (0.5, 0.5, 0.5)
                assert m.color == ((1.0, 0.0, 0.0, 1.0) if s[2] else (0.0, 1.0, 0.0, 1.0)) and m.orientation == (0, 0, 0, 1)
                np.testing.assert_array_equal(np.array(m.points).reshape(-1, 3), s[3])
        assert len(out[f"{topic}/road_marker"]) == len(mine)
        for k in ("road", "curb", "roi", "road_probably"):
            got = out[f"{topic}/{k}"]
            assert [tm for _, tm, _ in got] == [t for t, _, _ in mine]                # per-topic time order
            for (t, n, ctrl), (typ, tm, data) in zip(mine, got):
                msg = rosbag.decode_cloud2(data)
                exp = expected_clouds(pts[(topic, t)])[k]
                assert typ == "sensor_msgs/PointCloud2" and msg.header == Header(3, Time(*t), "lidar")
                assert [f[:3] for f in msg.fields] == [("x", 0, 7), ("y", 4, 7), ("z", 8, 7), ("intensity", 16, 7)]
                assert (msg.height, msg.width, msg.point_step, msg.row_step, msg.is_dense) == (1, exp.shape[0], 32, 32 * exp.shape[0], True)
                assert bytes(msg.data) == exp.tobytes(), (topic, t, k)
    # /os1_a/points: 5 colour runs, then 2, then 1: the second and third MarkerArrays delete the ghosts of the first
    acts = [[m.action for m in rosbag.decode_marker_array(d)] for _, _, d in out["/os1_a/points/road_marker"]]
    assert acts[1].count(2) == 3 and acts[2].count(2) == 1


def test_replay_stops_at_a_failed_scan(tmp_path):
    src, _ = drive(tmp_path, SCANS[:4] + [("/velo/points", (11, 1), 36, -1)] + SCANS[5:])
    with pytest.raises(ReplayError, match=r"/velo/points: the scan at 11\.000000001 failed with urf error -3"):
        replay(src, str(tmp_path / "out.bag"), devices=(0, 1), slots=2, batch=1, process_fn=stand_in)


def test_replay_options(tmp_path):
    src, _ = drive(tmp_path)
    rep = replay(src, None, topics=["/velo/points"], devices=(0,), slots=2, batch=2, limit=2, process_fn=stand_in)
    assert rep.scans == {"/velo/points": 2} and "replayed 2 scans" in str(rep)
    with pytest.raises(ReplayError, match="/nope: no sensor_msgs/PointCloud2 topic"):
        replay(src, None, topics=["/nope"], process_fn=stand_in)
    prm = parse_sets(["curb_points=7", "max_x=40.5", "fixed_frame=map", "channels=128"])
    assert (prm.curb_points, prm.max_x, prm.fixed_frame, prm.channels) == (7, 40.5, b"map", 128)
    for bad in ("curb_points", "nope=1", "curb_points=1.5"):
        with pytest.raises(ReplayError):
            parse_sets([bad])


def test_replay_refuses_a_format_change_and_too_many_formats(tmp_path):
    path = str(tmp_path / "change.bag")
    p = scan_points(8, 1, 0)
    with BagWriter(path) as w:
        w.write("/a", rosbag.POINTCLOUD2, Time(1, 0), as_message(p, OUSTER_FIELDS, 48, Time(1, 0)))
        w.write("/a", rosbag.POINTCLOUD2, Time(2, 0), as_message(p, VELO22_FIELDS, 22, Time(2, 0)))
    with pytest.raises(ReplayError, match="/a: record format changes"):
        replay(path, None, process_fn=stand_in)
    path = str(tmp_path / "many.bag")
    with BagWriter(path) as w:
        for k in range(9):
            w.write(f"/s{k}", rosbag.POINTCLOUD2, Time(1, k), as_message(p, XYZI16, 16 + 4 * k, Time(1, k)))
    with pytest.raises(ReplayError, match=r"9 distinct record formats, at most 8 .*CloudFormat\(point_step=48.*\(/s8\)"):
        replay(path, None, process_fn=stand_in)

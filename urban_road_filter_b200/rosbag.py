"""ROS1 bag files (format 2.0) and the two message types the replay reads and writes, with the Python standard library
only: no ROS installation and no `rosbag` package. Written from the format specification (wiki.ros.org/Bags/Format/2.0).

A bag is the version line `#ROSBAG V2.0`, a bag header record padded to 4096 bytes, chunk records (each followed by one
index data record per connection in it), and from `index_pos` on the connection records and the chunk info records. Every
record is a header (length-prefixed `name=value` fields, `op` naming the record kind) and a length-prefixed data part.

- BagReader: connections and messages of chosen topics in time order, uncompressed chunks read from an mmap without a copy,
  `bz2` chunks decompressed. lz4 chunks, unindexed bags and other versions are refused with their cause.
- BagWriter: what `rosbag record` writes: chunks (uncompressed, or `bz2`), index data, then the connection and chunk info
  records, and the bag header rewritten with index_pos, conn_count and chunk_count.
- sensor_msgs/PointCloud2 and visualization_msgs/MarkerArray: (de)serialisers, their message definitions and md5sums
  computed by the genmsg rule.
"""
from __future__ import annotations

import bz2
import collections
import dataclasses
import hashlib
import mmap
import os
import struct

from .api import CloudFormat
from .ctypes_abi import URF_MAX_FORMATS

VERSION_LINE = b"#ROSBAG V2.0\n"
BAG_HEADER_LEN = 4096                       # the bag header record, padded with spaces
OP_MSG, OP_BAG_HEADER, OP_INDEX, OP_CHUNK, OP_CHUNK_INFO, OP_CONNECTION = 0x02, 0x03, 0x04, 0x05, 0x06, 0x07
CHUNK_THRESHOLD = 768 * 1024                # rosbag's default chunk size

Time = collections.namedtuple("Time", "secs nsecs")       # ros::Time; sorts in time order
Connection = collections.namedtuple("Connection", "id topic type md5sum message_definition fields")
_U32, _U64, _TIME = struct.Struct("<I"), struct.Struct("<Q"), struct.Struct("<II")


class BagError(ValueError):
    """A file that is not a bag this module can read, or a message it cannot take."""


# ---------------------------------------------------------------------------------------------------------------------
# message definitions and md5sums

_DEFINITIONS = {
    "std_msgs/Header": "uint32 seq\ntime stamp\nstring frame_id",
    "sensor_msgs/PointField": ("uint8 INT8    = 1\nuint8 UINT8   = 2\nuint8 INT16   = 3\nuint8 UINT16  = 4\n"
                               "uint8 INT32   = 5\nuint8 UINT32  = 6\nuint8 FLOAT32 = 7\nuint8 FLOAT64 = 8\n\n"
                               "string name\nuint32 offset\nuint8  datatype\nuint32 count"),
    "sensor_msgs/PointCloud2": ("Header header\n\nuint32 height\nuint32 width\n\nPointField[] fields\n\nbool    is_bigendian\n"
                                "uint32  point_step\nuint32  row_step\nuint8[] data\n\nbool is_dense"),
    "geometry_msgs/Point": "float64 x\nfloat64 y\nfloat64 z",
    "geometry_msgs/Quaternion": "float64 x\nfloat64 y\nfloat64 z\nfloat64 w",
    "geometry_msgs/Pose": "Point position\nQuaternion orientation",
    "geometry_msgs/Vector3": "float64 x\nfloat64 y\nfloat64 z",
    "std_msgs/ColorRGBA": "float32 r\nfloat32 g\nfloat32 b\nfloat32 a",
    "visualization_msgs/Marker": (
        "uint8 ARROW=0\nuint8 CUBE=1\nuint8 SPHERE=2\nuint8 CYLINDER=3\nuint8 LINE_STRIP=4\nuint8 LINE_LIST=5\n"
        "uint8 CUBE_LIST=6\nuint8 SPHERE_LIST=7\nuint8 POINTS=8\nuint8 TEXT_VIEW_FACING=9\nuint8 MESH_RESOURCE=10\n"
        "uint8 TRIANGLE_LIST=11\n\nuint8 ADD=0\nuint8 MODIFY=0\nuint8 DELETE=2\nuint8 DELETEALL=3\n\n"
        "Header header\nstring ns\nint32 id\nint32 type\nint32 action\ngeometry_msgs/Pose pose\ngeometry_msgs/Vector3 scale\n"
        "std_msgs/ColorRGBA color\nduration lifetime\nbool frame_locked\ngeometry_msgs/Point[] points\n"
        "std_msgs/ColorRGBA[] colors\nstring text\nstring mesh_resource\nbool mesh_use_embedded_materials"),
    "visualization_msgs/MarkerArray": "Marker[] markers",
}
_BUILTIN = {"bool", "int8", "uint8", "int16", "uint16", "int32", "uint32", "int64", "uint64", "float32", "float64",
            "string", "time", "duration", "byte", "char"}


def _statements(text: str):
    """(type, name, value or None) of each field and constant of a .msg text, comments and blank lines skipped."""
    for line in text.splitlines():
        line = line.split("#", 1)[0].strip()
        if not line:
            continue
        typ, rest = line.split(None, 1)
        if "=" in rest:
            name, val = rest.split("=", 1)
            yield typ, name.strip(), val.strip()
        else:
            yield typ, rest.strip(), None


def _resolve(typ: str, package: str) -> str:
    base = typ.split("[", 1)[0]
    if base == "Header":
        return "std_msgs/Header"
    return base if "/" in base else f"{package}/{base}"


def md5sum(name: str) -> str:
    """genmsg's md5: constants first as `type NAME=value`, then fields, each nested type replaced by its own md5sum."""
    pkg = name.split("/")[0]
    consts, fields = [], []
    for typ, fname, val in _statements(_DEFINITIONS[name]):
        if val is not None:
            consts.append(f"{typ} {fname}={val}")
        elif typ.split("[", 1)[0] in _BUILTIN:
            fields.append(f"{typ} {fname}")
        else:
            fields.append(f"{md5sum(_resolve(typ, pkg))} {fname}")
    return hashlib.md5("\n".join(consts + fields).encode()).hexdigest()


def _dependencies(name: str, out: list) -> list:
    pkg = name.split("/")[0]
    for typ, _, val in _statements(_DEFINITIONS[name]):
        if val is None and typ.split("[", 1)[0] not in _BUILTIN:
            dep = _resolve(typ, pkg)
            if dep not in out:
                out.append(dep)
                _dependencies(dep, out)
    return out


def message_definition(name: str) -> str:
    """The full definition text rosbag stores with a connection: the type's text, then each nested type after a line of
    80 '=' and `MSG: pkg/Type` (genmsg compute_full_text). Field and constant lines only, without the .msg comments."""
    parts = [_DEFINITIONS[name] + "\n"]
    for dep in _dependencies(name, []):
        parts.append("=" * 80 + f"\nMSG: {dep}\n" + _DEFINITIONS[dep] + "\n")
    return "".join(parts)


@dataclasses.dataclass(frozen=True)
class MsgType:
    name: str
    md5sum: str
    definition: str

    @classmethod
    def of(cls, name: str) -> "MsgType":
        return cls(name, md5sum(name), message_definition(name))


POINTCLOUD2 = MsgType.of("sensor_msgs/PointCloud2")
MARKERARRAY = MsgType.of("visualization_msgs/MarkerArray")

# ---------------------------------------------------------------------------------------------------------------------
# message codecs

FLOAT32 = 7
DATATYPE_NAMES = {1: "INT8", 2: "UINT8", 3: "INT16", 4: "UINT16", 5: "INT32", 6: "UINT32", 7: "FLOAT32", 8: "FLOAT64"}
Header = collections.namedtuple("Header", "seq stamp frame_id")
PointField = collections.namedtuple("PointField", "name offset datatype count")


@dataclasses.dataclass
class PointCloud2:
    header: Header
    height: int
    width: int
    fields: list
    is_bigendian: bool
    point_step: int
    row_step: int
    data: bytes | memoryview               # a memoryview into the bag when read
    is_dense: bool


@dataclasses.dataclass
class Marker:
    header: Header = Header(0, Time(0, 0), "")
    ns: str = ""
    id: int = 0
    type: int = 0
    action: int = 0
    position: tuple = (0.0, 0.0, 0.0)
    orientation: tuple = (0.0, 0.0, 0.0, 1.0)          # x, y, z, w
    scale: tuple = (0.0, 0.0, 0.0)
    color: tuple = (0.0, 0.0, 0.0, 0.0)                # r, g, b, a (float32 on the wire)
    lifetime: tuple = (0, 0)                           # duration secs, nsecs
    frame_locked: bool = False
    points: list = dataclasses.field(default_factory=list)     # [(x, y, z)]
    colors: list = dataclasses.field(default_factory=list)     # [(r, g, b, a)]
    text: str = ""
    mesh_resource: str = ""
    mesh_use_embedded_materials: bool = False


LINE_STRIP, ADD, DELETE = 4, 0, 2


def _string(s: str) -> bytes:
    b = s.encode()
    return _U32.pack(len(b)) + b


def _header(h: Header) -> bytes:
    return struct.pack("<III", h.seq, h.stamp[0], h.stamp[1]) + _string(h.frame_id)


class _Cursor:
    """Reads ROS1-serialised fields from a buffer, refusing reads past its end."""

    def __init__(self, buf, what: str):
        self.buf, self.pos, self.what = buf, 0, what

    def take(self, fmt: struct.Struct):
        if self.pos + fmt.size > len(self.buf):
            raise BagError(f"{self.what}: message ends inside a field")
        v = fmt.unpack_from(self.buf, self.pos)
        self.pos += fmt.size
        return v

    def bytes(self, n: int):
        if self.pos + n > len(self.buf):
            raise BagError(f"{self.what}: message ends inside a field")
        v = self.buf[self.pos: self.pos + n]
        self.pos += n
        return v

    def string(self) -> str:
        return bytes(self.bytes(self.take(_U32)[0])).decode()

    def header(self) -> Header:
        seq, s, ns = self.take(_HDR)
        return Header(seq, Time(s, ns), self.string())


_HDR = struct.Struct("<III")
_FIELD_TAIL = struct.Struct("<IBI")
_CLOUD_MID = struct.Struct("<?II")
_MARKER_MID = struct.Struct("<iii10d4fiiB")
_COLOR = struct.Struct("<4f")
_POINT = struct.Struct("<3d")


def cloud2_parts(msg: PointCloud2) -> list:
    """The serialised message as a list of buffers (the point data not copied), for BagWriter.write."""
    out = [_header(msg.header), struct.pack("<III", msg.height, msg.width, len(msg.fields))]
    for f in msg.fields:
        out += [_string(f.name), _FIELD_TAIL.pack(f.offset, f.datatype, f.count)]
    data = memoryview(msg.data)
    data = data.cast("B") if data.nbytes else memoryview(b"")     # a view with a zero in its shape cannot be cast
    out += [_CLOUD_MID.pack(bool(msg.is_bigendian), msg.point_step, msg.row_step), _U32.pack(data.nbytes), data,
            struct.pack("<?", bool(msg.is_dense))]
    return out


def encode_cloud2(msg: PointCloud2) -> bytes:
    return b"".join(cloud2_parts(msg))


def decode_cloud2(buf, what: str = "PointCloud2") -> PointCloud2:
    """A PointCloud2 whose `data` is a memoryview into `buf` (no copy)."""
    c = _Cursor(memoryview(buf).cast("B"), what)
    header = c.header()
    height, width, nf = c.take(_HDR)
    fields = []
    for _ in range(nf):
        name = c.string()
        fields.append(PointField(name, *c.take(_FIELD_TAIL)))
    big, step, row = c.take(_CLOUD_MID)
    data = c.bytes(c.take(_U32)[0])
    (dense,) = c.take(struct.Struct("<?"))
    return PointCloud2(header, height, width, fields, big, step, row, data, dense)


def encode_marker_array(markers) -> bytes:
    out = [_U32.pack(len(markers))]
    for m in markers:
        out += [_header(m.header), _string(m.ns),
                _MARKER_MID.pack(m.id, m.type, m.action, *m.position, *m.orientation, *m.scale, *m.color, *m.lifetime,
                                 bool(m.frame_locked)),
                _U32.pack(len(m.points))]
        out += [_POINT.pack(*p) for p in m.points]
        out.append(_U32.pack(len(m.colors)))
        out += [_COLOR.pack(*c) for c in m.colors]
        out += [_string(m.text), _string(m.mesh_resource), struct.pack("<?", bool(m.mesh_use_embedded_materials))]
    return b"".join(out)


def decode_marker_array(buf, what: str = "MarkerArray") -> list:
    c = _Cursor(memoryview(buf).cast("B"), what)
    out = []
    for _ in range(c.take(_U32)[0]):
        header, ns = c.header(), c.string()
        v = c.take(_MARKER_MID)
        points = [c.take(_POINT) for _ in range(c.take(_U32)[0])]
        colors = [c.take(_COLOR) for _ in range(c.take(_U32)[0])]
        text, mesh = c.string(), c.string()
        (emb,) = c.take(struct.Struct("<?"))
        out.append(Marker(header, ns, v[0], v[1], v[2], v[3:6], v[6:10], v[10:13], v[13:17], v[17:19], bool(v[19]), points,
                          colors, text, mesh, emb))
    return out


def cloud_format(msg: PointCloud2, topic: str) -> CloudFormat:
    """The record format of a PointCloud2 as ros/urf_node_cloud2.cpp reads it: FLOAT32 fields `x`, `y`, `z` and `intensity`
    (-1 when absent or not FLOAT32). Refuses, naming the topic, what the device unpack cannot read: a missing or
    non-FLOAT32 coordinate, big-endian data, rows with padding (row_step != width * point_step), a point_step outside
    [12, 64], a field past the end of the record and data shorter than width * height records."""
    off = {}
    for f in msg.fields:
        if f.name in ("x", "y", "z", "intensity") and f.name not in off:
            off[f.name] = f
    for axis in ("x", "y", "z"):
        f = off.get(axis)
        if f is None:
            raise BagError(f"{topic}: PointCloud2 has no field {axis!r}")
        if f.datatype != FLOAT32:
            raise BagError(f"{topic}: field {axis!r} is {DATATYPE_NAMES.get(f.datatype, f.datatype)}, not FLOAT32")
    if msg.is_bigendian:
        raise BagError(f"{topic}: big-endian PointCloud2 data")
    if msg.row_step != msg.width * msg.point_step:
        raise BagError(f"{topic}: row_step {msg.row_step} != width {msg.width} * point_step {msg.point_step} (padded rows)")
    if not 12 <= msg.point_step <= 64:
        raise BagError(f"{topic}: point_step {msg.point_step} is outside [12, 64]")
    oi = off.get("intensity")
    fmt = CloudFormat(msg.point_step, off["x"].offset, off["y"].offset, off["z"].offset,
                      oi.offset if oi is not None and oi.datatype == FLOAT32 else -1)
    for name, o in zip(("x", "y", "z", "intensity"), fmt[1:]):
        if o >= 0 and o + 4 > msg.point_step:
            raise BagError(f"{topic}: field {name!r} at byte {o} ends past point_step {msg.point_step}")
    if len(msg.data) < msg.width * msg.height * msg.point_step:
        raise BagError(f"{topic}: {len(msg.data)} data bytes hold fewer than {msg.width} x {msg.height} records")
    return fmt


# ---------------------------------------------------------------------------------------------------------------------
# records

def _fields(buf, pos: int, end: int, where: str) -> dict:
    out = {}
    while pos < end:
        if pos + 4 > end:
            raise BagError(f"{where}: truncated header field")
        (n,) = _U32.unpack_from(buf, pos)
        pos += 4
        if pos + n > end:
            raise BagError(f"{where}: header field runs past its header")
        name, sep, val = bytes(buf[pos: pos + n]).partition(b"=")
        if not sep:
            raise BagError(f"{where}: header field without '='")
        out[name.decode()] = val
        pos += n
    return out


def _read_record(buf, pos: int, where: str):
    """(header fields, data start, data length, next record position) of the record at pos."""
    if pos + 4 > len(buf):
        raise BagError(f"{where}: truncated record at byte {pos}")
    (hlen,) = _U32.unpack_from(buf, pos)
    dpos = pos + 4 + hlen
    if dpos + 4 > len(buf):
        raise BagError(f"{where}: truncated record header at byte {pos}")
    header = _fields(buf, pos + 4, dpos, where)
    (dlen,) = _U32.unpack_from(buf, dpos)
    if dpos + 4 + dlen > len(buf):
        raise BagError(f"{where}: truncated record data at byte {pos}")
    return header, dpos + 4, dlen, dpos + 4 + dlen


def _op(h: dict, where: str) -> int:
    if len(h.get("op", b"")) != 1:
        raise BagError(f"{where}: record without an op field")
    return h["op"][0]


def _field(h: dict, name: str, fmt: struct.Struct, where: str):
    v = h.get(name)
    if v is None or len(v) != fmt.size:
        raise BagError(f"{where}: record field {name!r} is missing or malformed")
    r = fmt.unpack(v)
    return r[0] if len(r) == 1 else Time(*r)


def _header_bytes(fields: list) -> bytes:
    """Header fields [(name, value bytes)] as length-prefixed `name=value` entries."""
    return b"".join(_U32.pack(len(k) + 1 + len(v)) + k.encode() + b"=" + v for k, v in fields)


def _record_bytes(fields: list, data=b"") -> list:
    """A record as buffers: fields [(name, value bytes)], then the data (bytes-like or a list of them)."""
    hdr = _header_bytes(fields)
    parts = data if isinstance(data, list) else [data]
    dlen = sum(memoryview(p).nbytes for p in parts)
    return [_U32.pack(len(hdr)), hdr, _U32.pack(dlen), *parts]


ChunkInfo = collections.namedtuple("ChunkInfo", "pos start_time end_time counts")


class BagReader:
    """An indexed ROS1 bag (format 2.0). `connections` maps connection id to Connection, `chunks` lists ChunkInfo, and
    messages() yields (topic, connection, time, memoryview of the serialised message) in time order (equal times in file
    order). Messages of uncompressed chunks are views of the file's mmap; keep the reader open while they are used."""

    def __init__(self, path: str):
        self.path = path
        self._file = open(path, "rb")
        try:
            size = os.fstat(self._file.fileno()).st_size
            self._mm = mmap.mmap(self._file.fileno(), 0, access=mmap.ACCESS_READ) if size else None
            self._buf = memoryview(self._mm if size else b"")
            self._open()
        except BaseException:
            self.close()
            raise

    def _open(self):
        buf, where = self._buf, self.path
        line = bytes(buf[: len(VERSION_LINE)])
        if line != VERSION_LINE:
            if line.startswith(b"#ROSBAG V"):
                raise BagError(f"{where}: bag version {line[9:].strip().decode(errors='replace')}; only 2.0 is supported")
            raise BagError(f"{where}: not a ROS bag (no '#ROSBAG V2.0' line)")
        h, _, _, _ = _read_record(buf, len(VERSION_LINE), where)
        if _op(h, where) != OP_BAG_HEADER:
            raise BagError(f"{where}: the first record is not a bag header")
        index_pos = _field(h, "index_pos", _U64, where)
        if index_pos == 0:
            raise BagError(f"{where}: the bag is not indexed (index_pos 0): run `rosbag reindex` on it")
        conn_count = _field(h, "conn_count", _U32, where)
        chunk_count = _field(h, "chunk_count", _U32, where)
        pos = index_pos
        self.connections = {}
        for _ in range(conn_count):
            h, d, n, pos = _read_record(buf, pos, where)
            if _op(h, where) != OP_CONNECTION:
                raise BagError(f"{where}: expected a connection record at byte {pos}")
            cid = _field(h, "conn", _U32, where)
            ch = _fields(buf, d, d + n, where)
            for k in ("type", "md5sum", "message_definition"):
                if k not in ch:
                    raise BagError(f"{where}: connection {cid} has no {k!r}")
            self.connections[cid] = Connection(cid, h["topic"].decode(), ch["type"].decode(), ch["md5sum"].decode(),
                                               ch["message_definition"].decode(), ch)
        self.chunks = []
        for _ in range(chunk_count):
            h, d, n, pos = _read_record(buf, pos, where)
            if _op(h, where) != OP_CHUNK_INFO:
                raise BagError(f"{where}: expected a chunk info record")
            counts = {}
            for k in range(_field(h, "count", _U32, where)):
                c, m = struct.unpack_from("<II", buf, d + 8 * k)
                counts[c] = m
            self.chunks.append(ChunkInfo(_field(h, "chunk_pos", _U64, where), _field(h, "start_time", _TIME, where),
                                         _field(h, "end_time", _TIME, where), counts))
        self._entries = []               # (time, chunk number, offset in the chunk's data, connection id)
        self._chunk_data = []            # (compression, data start, data length, uncompressed size)
        for k, ci in enumerate(self.chunks):
            h, d, n, pos = _read_record(buf, ci.pos, where)
            if _op(h, where) != OP_CHUNK:
                raise BagError(f"{where}: chunk info points at byte {ci.pos}, which holds no chunk")
            comp = h.get("compression", b"").decode()
            if comp == "lz4":
                raise BagError(f"{where}: lz4-compressed chunks are not supported (there is no lz4 in the Python standard "
                               "library): run `rosbag decompress` on the bag first")
            if comp not in ("none", "bz2"):
                raise BagError(f"{where}: unknown chunk compression {comp!r}")
            self._chunk_data.append((comp, d, n, _field(h, "size", _U32, where)))
            for _ in range(len(ci.counts)):
                h, d, n, pos = _read_record(buf, pos, where)
                if _op(h, where) != OP_INDEX:
                    raise BagError(f"{where}: expected the index data of the chunk at byte {ci.pos}")
                cid = _field(h, "conn", _U32, where)
                cnt = _field(h, "count", _U32, where)
                if n < 12 * cnt:
                    raise BagError(f"{where}: index data of connection {cid} is truncated")
                for s, ns, off in struct.iter_unpack("<III", buf[d: d + 12 * cnt]):
                    self._entries.append((Time(s, ns), k, off, cid))
        self._entries.sort()
        self._cache = collections.OrderedDict()

    def _chunk(self, k: int):
        """The uncompressed data of chunk k: a view of the mmap, or the decompressed bytes (the last few are cached)."""
        comp, d, n, size = self._chunk_data[k]
        if comp == "none":
            return self._buf[d: d + n]
        data = self._cache.get(k)
        if data is None:
            data = memoryview(bz2.decompress(self._buf[d: d + n]))
            if len(data) != size:
                raise BagError(f"{self.path}: chunk {k} decompresses to {len(data)} bytes, its header says {size}")
            self._cache[k] = data
            if len(self._cache) > 4:
                self._cache.popitem(last=False)
        return data

    def topics(self) -> dict:
        """topic -> message type, over every connection."""
        return {c.topic: c.type for c in self.connections.values()}

    def messages(self, topics=None):
        """(topic, connection, time, memoryview) of every message whose topic is in `topics` (None: all), in time order."""
        for t, k, off, cid in self._entries:
            conn = self.connections.get(cid)
            if conn is None:
                raise BagError(f"{self.path}: index names connection {cid}, which has no connection record")
            if topics is not None and conn.topic not in topics:
                continue
            data = self._chunk(k)
            h, d, n, _ = _read_record(data, off, self.path)
            if _op(h, self.path) != OP_MSG or _field(h, "conn", _U32, self.path) != cid:
                raise BagError(f"{self.path}: index entry at chunk {k} offset {off} is not a message of connection {cid}")
            yield conn.topic, conn, t, data[d: d + n]

    def close(self):
        self._cache = collections.OrderedDict()
        try:
            if getattr(self, "_buf", None) is not None:
                self._buf.release()
            if getattr(self, "_mm", None) is not None:
                self._mm.close()
        except BufferError:              # message views are still alive: the mapping goes when they do
            pass
        self._buf = self._mm = None
        self._file.close()

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()


class BagWriter:
    """Writes a ROS1 bag (format 2.0) as `rosbag record` lays it out, readable by `rosbag info` / `rosbag play`. One
    connection per topic, created at its first message. compression "none" (default) or "bz2"; a chunk is closed once
    its uncompressed size passes chunk_threshold bytes."""

    def __init__(self, path: str, compression: str = "none", chunk_threshold: int = CHUNK_THRESHOLD):
        if compression not in ("none", "bz2"):
            raise ValueError(f"chunk compression {compression!r}: expected 'none' or 'bz2'")
        self.compression, self.chunk_threshold = compression, chunk_threshold
        self._f = open(path, "wb")
        self._f.write(VERSION_LINE)
        self._write_bag_header(0, 0, 0)
        self._conns = {}                  # topic -> (id, MsgType)
        self._chunk_infos = []            # ChunkInfo
        self._new_chunk()

    def _new_chunk(self):
        self._chunk = bytearray()
        self._index = {}                  # connection id -> [(time, offset)]
        self._start = self._end = None

    def _write_bag_header(self, index_pos: int, conn_count: int, chunk_count: int):
        parts = _record_bytes([("op", bytes([OP_BAG_HEADER])), ("index_pos", _U64.pack(index_pos)),
                               ("conn_count", _U32.pack(conn_count)), ("chunk_count", _U32.pack(chunk_count))])
        used = sum(len(p) for p in parts)
        pad = BAG_HEADER_LEN - used
        self._f.write(b"".join(parts[:2]) + _U32.pack(pad) + b" " * pad)

    def _connection_record(self, cid: int, topic: str, mt: MsgType) -> list:
        conn = _header_bytes([("topic", topic.encode()), ("type", mt.name.encode()), ("md5sum", mt.md5sum.encode()),
                              ("message_definition", mt.definition.encode())])
        return _record_bytes([("op", bytes([OP_CONNECTION])), ("conn", _U32.pack(cid)), ("topic", topic.encode())], conn)

    def write(self, topic: str, msgtype: MsgType, t: Time, data):
        """One message: `data` is the serialised message, bytes-like or a list of bytes-like parts."""
        entry = self._conns.get(topic)
        if entry is None:
            entry = self._conns[topic] = (len(self._conns), msgtype)
            self._chunk += b"".join(self._connection_record(entry[0], topic, msgtype))
        elif entry[1] != msgtype:
            raise BagError(f"{topic}: written as {entry[1].name} and as {msgtype.name}")
        cid = entry[0]
        t = Time(*t)
        self._index.setdefault(cid, []).append((t, len(self._chunk)))
        for p in _record_bytes([("op", bytes([OP_MSG])), ("conn", _U32.pack(cid)), ("time", _TIME.pack(*t))], data):
            self._chunk += p
        self._start = t if self._start is None else min(self._start, t)
        self._end = t if self._end is None else max(self._end, t)
        if len(self._chunk) >= self.chunk_threshold:
            self._flush_chunk()

    def _flush_chunk(self):
        if not self._index:
            return
        pos = self._f.tell()
        body = bz2.compress(self._chunk) if self.compression == "bz2" else self._chunk
        parts = _record_bytes([("op", bytes([OP_CHUNK])), ("compression", self.compression.encode()),
                               ("size", _U32.pack(len(self._chunk)))], body)
        for cid in sorted(self._index):
            ents = self._index[cid]
            parts += _record_bytes([("op", bytes([OP_INDEX])), ("ver", _U32.pack(1)), ("conn", _U32.pack(cid)),
                                    ("count", _U32.pack(len(ents)))],
                                   b"".join(struct.pack("<III", t.secs, t.nsecs, off) for t, off in ents))
        self._f.write(b"".join(parts))
        self._chunk_infos.append(ChunkInfo(pos, self._start, self._end, {c: len(e) for c, e in sorted(self._index.items())}))
        self._new_chunk()

    def close(self):
        if self._f.closed:
            return
        self._flush_chunk()
        index_pos = self._f.tell()
        parts = []
        for topic, (cid, mt) in self._conns.items():
            parts += self._connection_record(cid, topic, mt)
        for ci in self._chunk_infos:
            parts += _record_bytes([("op", bytes([OP_CHUNK_INFO])), ("ver", _U32.pack(1)), ("chunk_pos", _U64.pack(ci.pos)),
                                    ("start_time", _TIME.pack(*ci.start_time)), ("end_time", _TIME.pack(*ci.end_time)),
                                    ("count", _U32.pack(len(ci.counts)))],
                                   b"".join(struct.pack("<II", c, m) for c, m in ci.counts.items()))
        self._f.write(b"".join(parts))
        self._f.seek(len(VERSION_LINE))
        self._write_bag_header(index_pos, len(self._conns), len(self._chunk_infos))
        self._f.close()

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()


def topic_formats(reader: BagReader, topics, limit: int | None = None):
    """The first pass of a replay over the bag index: (format of each topic, the largest message in points, the number
    of messages), over the first `limit` messages of `topics`. Every message of a topic must have its first message's
    format; more than URF_MAX_FORMATS distinct formats are refused, listing them."""
    fmts, largest, count = {}, 0, 0
    for topic, conn, t, data in reader.messages(topics):
        if limit is not None and count >= limit:
            break
        if conn.type != POINTCLOUD2.name:
            raise BagError(f"{topic}: type {conn.type}, not {POINTCLOUD2.name}")
        msg = decode_cloud2(data, topic)
        f = cloud_format(msg, topic)
        if fmts.setdefault(topic, f) != f:
            raise BagError(f"{topic}: record format changes from {fmts[topic]} to {f} at {t.secs}.{t.nsecs:09d}")
        largest = max(largest, msg.width * msg.height)
        count += 1
    distinct = sorted(set(fmts.values()))
    if len(distinct) > URF_MAX_FORMATS:
        raise BagError(f"{len(distinct)} distinct record formats, at most {URF_MAX_FORMATS} fit one stream: "
                       + "; ".join(f"{f} ({', '.join(t for t in fmts if fmts[t] == f)})" for f in distinct))
    return fmts, largest, count

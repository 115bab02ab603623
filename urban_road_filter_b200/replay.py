"""Replay of a recorded drive: the PointCloud2 topics of a ROS1 bag classified on the GPU, and what the reference node would
have published for every scan written to a new bag, without ROS.

    python -m urban_road_filter_b200.replay IN.bag OUT.bag [--topics T1,T2] [--devices 0,1] [--slots 16] [--batch 8]
        [--set name=value ...] [--reference-tie-order] [--bz2] [--limit N]

For each input topic T the output bag holds T/road, T/curb, T/roi, T/road_probably (sensor_msgs/PointCloud2) and
T/road_marker (visualization_msgs/MarkerArray): the reference's topic names (lidar_segmentation.cpp:55-59) under the input
topic, so that several sensors stay apart. Every output message carries its input message's bag time.

One pass over the bag index gives the topics, their record formats (rosbag.cloud_format) and the largest scan. One formats
MultiGpuQueue (urf_mq_create_formats, one table entry per distinct format, int8 labels and the emission order) carries
every scan: a producer thread submits each message's `data` in bag time order, and a consumer thread takes the results in
the same order, packs the four clouds on the host from the input records, the labels and the emission order, as
ros/urf_node_cloud2.cpp publishes them, builds the MarkerArray from urf_build_markers with a ghostcount kept per input
topic (ros/urf_glue_common.hpp), and writes them. A scan with too few points writes nothing, as the reference publishes
nothing (lidar_segmentation.cpp:124-126); a failed scan stops the replay with its topic, time and error code.
"""
from __future__ import annotations

import argparse
import collections
import dataclasses
import sys
import threading
import time

import numpy as np

from . import rosbag
from .api import MultiGpuQueue, UrfError, build_markers, load_library
from .ctypes_abi import DEFAULTS, URF_ERR_CLOSED, URF_TOO_FEW_POINTS, UrfParams, make_params
from .rosbag import MARKERARRAY, POINTCLOUD2, BagReader, BagWriter, Header, Marker, PointCloud2, PointField, Time

CLOUDS = ("road", "curb", "roi", "road_probably")
# the field layout pcl_ros gives a pcl::PointCloud<pcl::PointXYZI> (32-byte records), as ros/urf_node_cloud2.cpp publishes
XYZI_FIELDS = [PointField("x", 0, rosbag.FLOAT32, 1), PointField("y", 4, rosbag.FLOAT32, 1),
               PointField("z", 8, rosbag.FLOAT32, 1), PointField("intensity", 16, rosbag.FLOAT32, 1)]


class ReplayError(RuntimeError):
    """A scan the library failed on, or an input the replay refuses."""


def output_topics(topic: str) -> dict:
    """Output topic of each published name: the reference node's topic names under the input topic."""
    return {k: f"{topic}/{k}" for k in CLOUDS + ("road_marker",)}


def pack_clouds(records: np.ndarray, fmt, r) -> dict:
    """The four clouds of scan result r (labels and emission order) as float32 [count, 8] arrays of 32-byte
    pcl::PointXYZI records (x, y, z, 1.0, intensity or 0, zero padding), taken from the scan's raw `records` (uint8) of
    format fmt: road and curb in emission order, roi in input order, road_probably the ring-10 segment."""
    roi = r.cloud_indices("roi")
    rec = records[: r.n_in * fmt.point_step].reshape(r.n_in, fmt.point_step)[roi]
    packed = np.zeros((roi.size, 8), np.float32)
    b = packed.view(np.uint8)
    for k, off in enumerate((fmt.off_x, fmt.off_y, fmt.off_z)):
        b[:, 4 * k: 4 * k + 4] = rec[:, off: off + 4]
    packed[:, 3] = 1.0
    if fmt.off_intensity >= 0:
        b[:, 16:20] = rec[:, fmt.off_intensity: fmt.off_intensity + 4]
    at = np.empty(r.n_in, np.int32)                   # input index -> row of `packed`; every ordered point is in the ROI
    at[roi] = np.arange(roi.size, dtype=np.int32)
    out = {"roi": packed}
    for k in ("road", "curb", "road_probably"):
        out[k] = packed[at[r.cloud_indices(k)]]
    return out


def cloud_message(header: Header, packed: np.ndarray) -> PointCloud2:
    n = packed.shape[0]
    return PointCloud2(header, 1, n, XYZI_FIELDS, False, 32, 32 * n, packed, True)


def marker_array(strips, frame_id: str) -> list:
    """The road_marker MarkerArray of urf_build_markers' strips, as ros/urf_glue_common.hpp build_marker_array fills it."""
    out = []
    for sid, action, red, pts in strips:
        out.append(Marker(header=Header(0, Time(0, 0), frame_id), id=sid, type=rosbag.LINE_STRIP,
                          action=rosbag.DELETE if action == 2 else rosbag.ADD, scale=(0.5, 0.5, 0.5),
                          color=(1.0, 0.0, 0.0, 1.0) if red else (0.0, 1.0, 0.0, 1.0),
                          points=[tuple(p) for p in pts.tolist()]))
    return out


def parse_sets(sets) -> UrfParams:
    """LidarFilters.cfg defaults (and `channels`) with `name=value` overrides, checked by make_params."""
    over = {}
    for s in sets or ():
        name, sep, val = s.partition("=")
        if not sep or name not in DEFAULTS:
            raise ReplayError(f"--set {s!r}: expected name=value with name one of {', '.join(DEFAULTS)}")
        kind = type(DEFAULTS[name])
        try:
            over[name] = val if kind is bytes else kind(val)
        except ValueError:
            raise ReplayError(f"--set {s!r}: {name} takes a {kind.__name__}") from None
    return make_params(**over)


@dataclasses.dataclass
class Report:
    scans: dict                  # input topic -> scans classified
    published: dict              # input topic -> scans that wrote their outputs (not URF_TOO_FEW_POINTS)
    seconds: float               # wall time of the stream, from the first submit to the last write
    read_s: float                # producer: parsing the bag and its messages
    wait_s: float                # consumer: waiting for results from the queue
    pack_s: float                # consumer: packing the clouds and building the markers
    write_s: float               # consumer: serialising and writing the output bag
    devices: tuple

    @property
    def total(self) -> int:
        return sum(self.scans.values())

    def __str__(self) -> str:
        rate = self.total / self.seconds if self.seconds > 0 else 0.0
        lines = [f"replayed {self.total} scans in {self.seconds:.3f} s ({rate:.1f} scans/s) on devices {list(self.devices)}"]
        lines += [f"  {t}: {n} scans, {self.published[t]} published" for t, n in self.scans.items()]
        lines.append(f"  reading {self.read_s:.3f} s, waiting on the queue {self.wait_s:.3f} s, packing {self.pack_s:.3f} s, "
                     f"writing {self.write_s:.3f} s")
        return "\n".join(lines)


def replay(in_path: str, out_path: str | None, topics=None, devices=(0,), slots: int = 16, batch: int = 8,
           params: UrfParams | None = None, reference_tie_order: bool = False, compression: str = "none",
           limit: int | None = None, process_fn=None) -> Report:
    """Replays the PointCloud2 topics `topics` (None: every PointCloud2 topic) of the bag at in_path through one formats
    MultiGpuQueue over `devices` and writes the outputs to out_path (None: built, then discarded). params: one parameter set
    for every scan (default: LidarFilters.cfg). limit: the first `limit` scans in bag time order. process_fn: stand-in
    devices (MultiGpuQueue's test hook) instead of GPUs. Raises ReplayError for a failed scan or a refused input."""
    prm = params if params is not None else make_params()
    frame_id = bytes(prm.fixed_frame).decode()
    with BagReader(in_path) as reader:
        available = {t: ty for t, ty in reader.topics().items() if ty == POINTCLOUD2.name}
        if topics is None:
            topics = sorted(available)
        for t in topics:
            if t not in available:
                raise ReplayError(f"{t}: no sensor_msgs/PointCloud2 topic of that name in {in_path}")
        if not topics:
            raise ReplayError(f"{in_path} has no sensor_msgs/PointCloud2 topic")
        try:
            fmts, largest, _ = rosbag.topic_formats(reader, set(topics), limit)
        except rosbag.BagError as e:
            raise ReplayError(str(e)) from None
        table = sorted(set(fmts.values()))
        fmt_index = {t: table.index(f) for t, f in fmts.items()}
        mq = MultiGpuQueue(list(devices), max(largest, 1), slots_per_device=slots, max_batch=batch, params=prm,
                           process_fn=process_fn, label8=True, order=True, formats=table)
        try:
            if reference_tie_order:
                mq.set_tie_order("reference")
            return _stream(reader, mq, set(fmts), fmts, fmt_index, prm, frame_id, out_path, compression, limit,
                           slots * len(devices), tuple(devices))
        finally:
            mq.close()
            mq.destroy()


def _stream(reader, mq, topics, fmts, fmt_index, prm, frame_id, out_path, compression, limit, cap, devices) -> Report:
    pending = {}                          # tag -> (topic, time, input header, records)
    errors = []                           # exceptions of either thread
    failed = []                           # (topic, time, error code) of a failed scan
    scans = collections.Counter()
    published = collections.Counter()
    ghost = collections.Counter()         # per input topic: lidar_segmentation.cpp:23's ghostcount
    times = dict(read=0.0, wait=0.0, pack=0.0, write=0.0)
    names = {t: output_topics(t) for t in topics}
    writer = BagWriter(out_path, compression) if out_path is not None else None

    def produce():
        try:
            it = reader.messages(topics)
            tag = 0
            while limit is None or tag < limit:
                t0 = time.perf_counter()
                item = next(it, None)
                if item is None:
                    break
                topic, _, t, data = item
                msg = rosbag.decode_cloud2(data, topic)
                n = msg.width * msg.height
                raw = np.frombuffer(msg.data, np.uint8, count=n * fmts[topic].point_step)
                pending[tag] = (topic, t, msg.header, raw)
                times["read"] += time.perf_counter() - t0
                if mq.submit_records(raw, n, tag=tag, fmt=fmt_index[topic]) == URF_ERR_CLOSED:
                    break
                tag += 1
        except BaseException as e:        # noqa: BLE001 — handed to the caller
            errors.append(e)
        finally:
            mq.close()

    def consume():
        try:
            while True:
                t0 = time.perf_counter()
                got = mq.next_batch(cap)
                times["wait"] += time.perf_counter() - t0
                if not got:
                    return
                for tag, r in got:
                    topic, t, header, raw = pending.pop(tag)
                    if r.status < 0:
                        failed.append((topic, t, r.status))
                        return
                    scans[topic] += 1
                    if r.status == URF_TOO_FEW_POINTS:
                        continue
                    published[topic] += 1
                    t0 = time.perf_counter()
                    clouds = pack_clouds(raw, fmts[topic], r)
                    markers = None
                    if r.n_vert > 2:                           # urf_glue_common.hpp build_marker_array
                        strips, ghost[topic] = build_markers(prm, r.vert, ghost[topic])
                        markers = marker_array(strips, frame_id)
                    t1 = time.perf_counter()
                    times["pack"] += t1 - t0
                    if writer is not None:
                        out = names[topic]
                        if markers is not None:
                            writer.write(out["road_marker"], MARKERARRAY, t, rosbag.encode_marker_array(markers))
                        for k in CLOUDS:
                            writer.write(out[k], POINTCLOUD2, t, rosbag.cloud2_parts(cloud_message(header, clouds[k])))
                        times["write"] += time.perf_counter() - t1
        except BaseException as e:        # noqa: BLE001 — handed to the caller
            errors.append(e)
        finally:
            mq.close()                    # a producer blocked in submit returns URF_ERR_CLOSED

    start = time.perf_counter()
    threads = [threading.Thread(target=produce, name="replay-producer"), threading.Thread(target=consume, name="replay-consumer")]
    for th in threads:
        th.start()
    for th in threads:
        th.join()
    t0 = time.perf_counter()
    if writer is not None:
        writer.close()
    times["write"] += time.perf_counter() - t0
    seconds = time.perf_counter() - start
    if errors:
        raise errors[0]
    if failed:
        topic, t, code = failed[0]
        detail = load_library().urf_strerror(code).decode()
        raise ReplayError(f"{topic}: the scan at {t.secs}.{t.nsecs:09d} failed with urf error {code} ({detail})")
    order = sorted(topics)
    return Report({t: scans[t] for t in order}, {t: published[t] for t in order}, seconds, times["read"], times["wait"],
                  times["pack"], times["write"], devices)


def main(argv=None) -> int:
    ap = argparse.ArgumentParser(prog="python -m urban_road_filter_b200.replay", description=__doc__.split("\n\n")[0])
    ap.add_argument("input", help="ROS1 bag (format 2.0, indexed; uncompressed or bz2 chunks)")
    ap.add_argument("output", help="bag to write")
    ap.add_argument("--topics", help="comma-separated PointCloud2 topics (default: every PointCloud2 topic)")
    ap.add_argument("--devices", default="0", help="comma-separated CUDA devices (default: 0)")
    ap.add_argument("--slots", type=int, default=16, help="queue slots per device")
    ap.add_argument("--batch", type=int, default=8, help="largest batch a device runs at once")
    ap.add_argument("--set", action="append", default=[], metavar="NAME=VALUE",
                    help="a LidarFilters.cfg parameter or channels (repeatable)")
    ap.add_argument("--reference-tie-order", action="store_true",
                    help="equal azimuths in the order the reference's quicksort leaves them")
    ap.add_argument("--bz2", action="store_true", help="bz2-compress the output chunks")
    ap.add_argument("--limit", type=int, help="replay the first N scans only")
    a = ap.parse_args(argv)
    try:
        report = replay(a.input, a.output, topics=a.topics.split(",") if a.topics else None,
                        devices=tuple(int(d) for d in a.devices.split(",")), slots=a.slots, batch=a.batch,
                        params=parse_sets(a.set), reference_tie_order=a.reference_tie_order,
                        compression="bz2" if a.bz2 else "none", limit=a.limit)
    except (ReplayError, rosbag.BagError, UrfError, KeyError) as e:
        print(f"replay: {e}", file=sys.stderr)
        return 1
    print(report)
    return 0


if __name__ == "__main__":
    sys.exit(main())

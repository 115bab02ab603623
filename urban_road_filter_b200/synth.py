"""Seeded synthetic LiDAR scans (SURVEY.md §8d): a ray-cast street scene with the ring x column shapes of the
BASELINE.json configs. Used by tests/ and bench.py; there is no dataset in this offline environment, and the
reference itself ships none (its only fixture is an external rosbag, README.md:36-46).

Scene: sensor at the origin, road plane z = -1.80 m, straight road along x with half-width 4 m, curbs (0.12 m high,
0.05 m wide sloped face) at y = +-4 m, side-walk plateau out to vertical walls at y = +-12 m and x = +-60 m so that
upward beams return too. Range noise is applied ALONG the beam only (keeps per-ring elevation constant, which the
reference's `interval` clustering of elevation angles needs, lidar_segmentation.cpp:170-196).
"""
from __future__ import annotations

import dataclasses

import numpy as np

GROUND_Z = -1.80
ROAD_HALF = 4.0
CURB_H = 0.12
CURB_W = 0.05
WALL_Y = 12.0
WALL_X = 60.0


@dataclasses.dataclass(frozen=True)
class SensorShape:
    name: str
    rings: int
    cols: int
    elev_lo: float
    elev_hi: float
    channels: int      # urf_params.channels needed
    interval: float    # urf_params.interval that separates this sensor's rings


# BASELINE.json configs 1..5 (SURVEY.md §8d)
SHAPES = {
    "C1": SensorShape("VLP-16 16x1800", 16, 1800, -15.0, 15.0, 64, 0.18),
    "C2": SensorShape("OS1-64 64x2048", 64, 2048, -16.6, 16.6, 64, 0.18),
    "C3": SensorShape("HDL-64E 64x2083", 64, 2083, -24.8, 2.0, 64, 0.18),
    "C4": SensorShape("OS2-128 128x2048", 128, 2048, -11.25, 11.25, 128, 0.07),
    "C5": SensorShape("synthetic 256x4096", 256, 4096, -25.0, 20.0, 256, 0.07),
}


def _cast(dx: np.ndarray, dy: np.ndarray, dz: np.ndarray, curb_offset: np.ndarray | float = 0.0) -> np.ndarray:
    """Range t along unit directions (float64) to the first surface of the scene. curb_offset shifts the curb lines
    in y per ray (lets scenes have a gently curving road edge)."""
    with np.errstate(divide="ignore", invalid="ignore"):
        ady = np.abs(dy)
        t_wall = np.minimum(np.where(ady > 1e-12, WALL_Y / ady, np.inf),
                            np.where(np.abs(dx) > 1e-12, WALL_X / np.abs(dx), np.inf))
        half = ROAD_HALF + curb_offset
        down = dz < 0
        t_road = np.where(down, GROUND_Z / dz, np.inf)
        on_road = down & (np.abs(t_road * dy) <= half)
        plateau_z = GROUND_Z + CURB_H
        t_plat = np.where(down, plateau_z / dz, np.inf)
        on_plat = down & (np.abs(t_plat * dy) >= half + CURB_W)
        slope = CURB_H / CURB_W
        # curb face: z = GROUND_Z + (|y| - half) * slope
        denom = dz - slope * ady
        t_face = np.where(down, (GROUND_Z - half * slope) / denom, np.inf)
        t_ground = np.where(on_road, t_road, np.where(on_plat, t_plat, t_face))
        t = np.minimum(t_ground, t_wall)
    return t


def make_scan(shape: SensorShape | str, seed: int = 0, order: str = "column", noise: float = 0.01,
              drop: float = 0.005, curve: float = 0.0, cols: int | None = None) -> np.ndarray:
    """Returns an (N, 4) float32 array (x, y, z, intensity), N = rings * cols.

    order: "column" = all rings of one azimuth column together (Velodyne/HDL packet order);
           "ring"   = ring-major, organised H x W cloud (Ouster driver).
    """
    if isinstance(shape, str):
        shape = SHAPES[shape]
    rng = np.random.default_rng(seed)
    R = shape.rings
    W = cols if cols is not None else shape.cols
    elev = np.deg2rad(np.linspace(shape.elev_lo, shape.elev_hi, R))
    # half-column offset keeps beams off the coordinate axes; per-scan phase + small per-beam azimuth jitter
    phase = rng.uniform(0.0, 1.0)
    az = (np.arange(W) + 0.5 * phase + 0.25) * (2.0 * np.pi / W)
    if order == "column":
        azg, elg = np.meshgrid(az, elev, indexing="ij")      # (W, R)
    elif order == "ring":
        elg, azg = np.meshgrid(elev, az, indexing="ij")      # (R, W)
    else:
        raise ValueError(order)
    azg = azg.ravel() + rng.uniform(-0.05, 0.05, azg.size) * (2.0 * np.pi / W)
    elg = elg.ravel()
    ce = np.cos(elg)
    dx, dy, dz = ce * np.cos(azg), ce * np.sin(azg), np.sin(elg)
    off = curve * np.sin(azg * 2.0) if curve else 0.0
    t = _cast(dx, dy, dz, off)
    t = t + rng.normal(0.0, noise, t.shape)
    t = np.maximum(t, 0.3)
    pts = np.empty((t.size, 4), dtype=np.float32)
    pts[:, 0] = (t * dx).astype(np.float32)
    pts[:, 1] = (t * dy).astype(np.float32)
    pts[:, 2] = (t * dz).astype(np.float32)
    pts[:, 3] = rng.uniform(0.0, 255.0, t.size).astype(np.float32)
    _detie_radius(pts, seed)
    if drop > 0:
        dead = rng.random(t.size) < drop
        pts[dead, :3] = 0.0
    return pts


def _detie_radius(pts: np.ndarray, seed: int = 0) -> None:
    """Make the float32 planar radius sqrtf(x*x+y*y) unique across the scan, so that no star-shaped sector
    (star_shaped_search.cpp:109, std::sort by r) ever holds an exact tie (SURVEY.md §7.4 H3). Colliding points are
    pushed outwards by a random sub-millimetre amount (dense wall returns need more than a few ulps)."""
    rng = np.random.default_rng(1_000_003 + seed)
    for _ in range(32):
        x, y = pts[:, 0], pts[:, 1]
        r = np.sqrt(x * x + y * y)                       # float32 arithmetic, same ops as the reference
        o = np.argsort(r, kind="stable")
        rs = r[o]
        dup = np.zeros(r.size, dtype=bool)
        dup[o[1:]] = rs[1:] == rs[:-1]
        if not dup.any():
            return
        k = np.float32(1.0) + np.float32(2.0 ** -21) * rng.integers(1, 1024, int(dup.sum())).astype(np.float32)
        pts[dup, 0] *= k
        pts[dup, 1] *= k
    raise RuntimeError("could not de-tie radii")


def make_batch(shape: SensorShape | str, batch: int, seed0: int = 0, **kw) -> list[np.ndarray]:
    return [make_scan(shape, seed0 + b, **kw) for b in range(batch)]


def random_cloud(n: int, seed: int = 0, rings: int = 8, extent: float = 40.0) -> np.ndarray:
    """Unstructured adversarial cloud: random ranges/azimuths on a few elevation cones plus pure noise points.
    Exercises ragged rings, unregistered elevations and empty sectors."""
    rng = np.random.default_rng(seed)
    elev = np.deg2rad(rng.uniform(-25, 10, rings))
    k = rng.integers(0, rings, n)
    az = rng.uniform(0, 2 * np.pi, n)
    t = rng.uniform(1.0, extent, n)
    e = elev[k] + np.where(rng.random(n) < 0.02, rng.uniform(-0.3, 0.3, n), 0.0)
    pts = np.empty((n, 4), dtype=np.float32)
    pts[:, 0] = t * np.cos(e) * np.cos(az)
    pts[:, 1] = t * np.cos(e) * np.sin(az)
    pts[:, 2] = t * np.sin(e)
    pts[:, 3] = rng.uniform(0, 255, n)
    _detie_radius(pts, seed)
    return pts


# PointCloud2 layouts of drive_bag's sensors: (point_step, [(field, offset, datatype)]), datatype 7 = FLOAT32
CLOUD2_LAYOUTS = {
    "ouster": (48, [("x", 0, 7), ("y", 4, 7), ("z", 8, 7), ("intensity", 16, 7), ("t", 20, 6), ("reflectivity", 24, 4),
                    ("ring", 26, 4), ("ambient", 28, 4), ("range", 32, 6)]),
    "velodyne": (32, [("x", 0, 7), ("y", 4, 7), ("z", 8, 7), ("intensity", 16, 7), ("ring", 20, 4), ("time", 24, 7)]),
}


def drive_bag(path: str, sensors, scans_per_sensor: int, seed: int = 0, distinct: int = 4, compression: str = "none") -> int:
    """Writes a seeded synthetic recorded drive to `path` as a ROS1 bag: sensors = [(topic, shape, layout)] with layout a
    key of CLOUD2_LAYOUTS; each sensor publishes scans_per_sensor PointCloud2 messages 0.1 s apart (sensors offset by
    10 ms), cycling through `distinct` make_scan scans of its shape; the bytes outside x / y / z / intensity are seeded
    noise. Returns the number of messages."""
    from .rosbag import POINTCLOUD2, BagWriter, Header, PointCloud2, PointField, Time, cloud2_parts

    msgs = []
    for i, (topic, shape, layout) in enumerate(sensors):
        step, fields = CLOUD2_LAYOUTS[layout]
        offs = {name: off for name, off, _ in fields}
        recs = []
        for k in range(distinct):
            pts = make_scan(shape, seed + 97 * i + k)
            rec = np.random.default_rng(seed + 1000 * i + k).integers(0, 256, (pts.shape[0], step), dtype=np.uint8)
            for j, name in enumerate(("x", "y", "z", "intensity")):
                rec[:, offs[name]: offs[name] + 4] = pts[:, j: j + 1].copy().view(np.uint8)
            recs.append((pts.shape[0], rec.reshape(-1)))
        pf = [PointField(name, off, dt, 1) for name, off, dt in fields]
        for k in range(scans_per_sensor):
            t = 1_000_000_000_000 + k * 100_000_000 + i * 10_000_000
            stamp = Time(t // 1_000_000_000, t % 1_000_000_000)
            n, rec = recs[k % distinct]
            msgs.append((stamp, topic, PointCloud2(Header(k, stamp, topic.strip("/").split("/")[0]), 1, n, pf, False, step,
                                                   n * step, rec, True)))
    msgs.sort(key=lambda m: m[0])
    with BagWriter(path, compression) as w:
        for stamp, topic, msg in msgs:
            w.write(topic, POINTCLOUD2, stamp, cloud2_parts(msg))
    return len(msgs)

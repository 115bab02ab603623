"""The device's tie policy written out plainly, and seeded clouds whose rings hold equal azimuths or whose degree bins hold
equal farthest planar ranges.

`policy(pts, o)` takes the cloud and the oracle port's debug run, and uses from that run only the per-point stages the
device has to match bit for bit anyway (ring id, azimuth, label). From them it derives what k_sort_rings, the marker
search and the cloud packing must produce under DESIGN.md deviation 2:
  * order: per ring, azimuth bits ascending, every NaN azimuth after every finite one, ties in input order;
  * bit2 (F_TIE_AZIMUTH): some ring holds two points with bit-identical azimuth. The device computes one NaN pattern, so
    two NaN azimuths of one ring tie; a lone NaN does not;
  * vertices: lidar_segmentation.cpp:298-351 on that order (per degree bin [i, i + 1): the cut is the first non-road point
    in scan order, the vertex the strictly farthest road point before it, redPoints = a cut exists);
  * the road / curb / road_probably / roi clouds as input indices in that order.
It does not use urf_logic.cuh or the CPU model of the kernels, so it is an independent witness of their tie handling."""
from __future__ import annotations

import dataclasses

import numpy as np

from urban_road_filter_b200 import FULL_ROI, make_params
from urban_road_filter_b200.synth import make_scan

from util import _ulps

# k_sort_rings (urf_kernels.cuh): counting sort up to kRingFast points with at most kBinCap points per bin, else a
# bitonic sort in shared memory up to kRingSmemKeys padded keys, else in global memory (sortbuf)
RING_FAST, RING_BINS, BIN_CAP, RING_SMEM_KEYS = 4096, 4096, 48, 6144
NAN_KEY = np.uint32(0x7fc00000)          # every NaN azimuth sorts as this: after +inf, equal to every other NaN


@dataclasses.dataclass
class Policy:
    order: np.ndarray         # input indices, ring by ring
    ring_start: np.ndarray    # [n_rings + 1]
    tie: bool                 # expected flags bit2
    vert: np.ndarray          # [n_vert, 4] float32: x, y, z, redPoints
    shared_max: int           # degree bins whose farthest candidate range is reached by two or more candidates
    winners: np.ndarray       # input index of each vertex
    clouds: dict              # "road" / "curb" / "road_probably" / "roi" -> input indices in emission order


def azimuth_keys(az: np.ndarray) -> np.ndarray:
    az = np.asarray(az, np.float32)
    fin = az[~np.isnan(az)]
    assert not np.any(np.signbit(fin)), "azimuths are >= +0, so their bits order them"
    return np.where(np.isnan(az), NAN_KEY, az.view(np.uint32)).astype(np.uint32)


def planar_range(pts: np.ndarray) -> np.ndarray:
    """float32(sqrt(double(x)^2 + double(y)^2)): the marker distance of lidar_segmentation.cpp:327."""
    x = pts[:, 0].astype(np.float64)
    y = pts[:, 1].astype(np.float64)
    return np.sqrt(x * x + y * y).astype(np.float32)


def policy(pts: np.ndarray, o) -> Policy:
    ring = np.asarray(o.ring, np.int64)
    label = np.asarray(o.label, np.int64)
    R = int(o.n_rings)
    idx = np.flatnonzero(ring >= 0)
    key = azimuth_keys(np.asarray(o.az, np.float32)[idx])
    perm = np.lexsort((idx, key, ring[idx]))
    order = idx[perm].astype(np.int32)
    okey, oring = key[perm], ring[order]
    ring_start = np.concatenate([[0], np.cumsum(np.bincount(oring, minlength=R))]).astype(np.int32)
    tie = bool(np.any((oring[1:] == oring[:-1]) & (okey[1:] == okey[:-1])))

    # markers: scan positions in emission order, 361 degree bins
    az = np.asarray(o.az, np.float32)[order]
    lab = label[order]
    d = planar_range(pts)[order]
    fin = ~np.isnan(az)
    b = np.full(order.size, -1, np.int64)
    b[fin] = np.floor(az[fin]).astype(np.int64)        # az >= i && az < i + 1
    inb = (b >= 0) & (b <= 360)
    pos = np.arange(order.size)
    big = order.size
    cut = np.full(361, big, np.int64)
    nonroad = inb & (lab != 1)
    np.minimum.at(cut, b[nonroad], pos[nonroad])
    cand = inb & (lab == 1) & (d > 0)
    cand[cand] &= pos[cand] < cut[b[cand]]
    dmax = np.zeros(361, np.float32)
    np.maximum.at(dmax, b[cand], d[cand])
    win = cand.copy()
    win[win] &= d[win] == dmax[b[win]]
    first = np.full(361, big, np.int64)
    np.minimum.at(first, b[win], pos[win])
    shared = np.bincount(b[win], minlength=361)
    bins = np.flatnonzero(first < big)
    p = order[first[bins]]
    vert = np.zeros((bins.size, 4), np.float32)
    vert[:, :3] = pts[p, :3]
    vert[:, 3] = (cut[bins] < big).astype(np.float32)

    clouds = {"road": order[lab == 1], "curb": order[lab == 2], "roi": np.flatnonzero(label >= 0).astype(np.int32),
              "road_probably": order[ring_start[10]: ring_start[11]] if R > 10 else order[:0]}
    return Policy(order, ring_start, tie, vert, int((shared >= 2).sum()), p.astype(np.int64), clouds)


def ring_regime(az_ring: np.ndarray) -> str:
    """The k_sort_rings path a ring with these azimuths takes: "fast" (counting sort, insertion sort inside a bin),
    "smem" (bitonic sort in shared memory) or "global" (bitonic sort in sortbuf). The bin map restates bin_of."""
    n = az_ring.size
    if n > RING_FAST:
        return "smem" if 1 << (n - 1).bit_length() <= RING_SMEM_KEYS else "global"
    return "fast" if max_bin_count(az_ring) <= BIN_CAP else "smem"


def max_bin_count(az_ring: np.ndarray) -> int:
    a = np.asarray(az_ring, np.float32)
    fin = a[~np.isnan(a)]
    lo, hi = (fin.min(), fin.max()) if fin.size else (np.float32(0), np.float32(0))
    scale = np.float32(RING_BINS - 2) / np.float32(hi - lo) if hi > lo else np.float32(0)
    with np.errstate(invalid="ignore"):
        v = np.trunc(np.float32(a - lo) * scale)
    bins = np.where(np.isnan(a), RING_BINS - 1, np.clip(np.nan_to_num(v, nan=0), 0, RING_BINS - 2)).astype(np.int64)
    return int(np.bincount(bins, minlength=RING_BINS).max())


# ---------------------------------------------------------------------------------------------------------------------
# Tie clouds. Every builder takes the oracle port, returns (pts, params) and asserts that the cloud reaches its target.

def _rings_of(o):
    ring, az = np.asarray(o.ring), np.asarray(o.az, np.float32)
    return [az[ring == k] for k in range(o.n_rings)]


def dual_return(port, seed: int, interleave: bool, n2: int = 3000):
    """A VLP-16 scan with a second return for n2 of its points at 2x or 0.5x the range along the same beam. A power-of-two
    scale keeps the azimuth and elevation bits, so the second return ties its first in azimuth and ring while its planar
    range differs. interleave: each second return right after its first, else all appended after the scan."""
    pts = make_scan("C1", seed)
    rng = np.random.default_rng(seed)
    pick = np.sort(rng.choice(np.flatnonzero(np.any(pts[:, :3] != 0, axis=1)), n2, replace=False))
    sec = pts[pick].copy()
    sec[:, :3] *= np.where(rng.random(n2) < 0.5, np.float32(2.0), np.float32(0.5))[:, None]
    out = np.insert(pts, pick + 1, sec, axis=0) if interleave else np.concatenate([pts, sec])
    prm = make_params(**FULL_ROI)
    o = port.run(out, prm, debug=True)
    first = pick + np.arange(n2) if interleave else pick
    second = first + 1 if interleave else pts.shape[0] + np.arange(n2)
    ok = (o.ring[first] >= 0) & (o.label[first] >= 0)
    assert ok.sum() > n2 * 0.9
    assert np.array_equal(o.ring[first][ok], o.ring[second][ok]), "a second return left its first's ring"
    assert np.array_equal(o.az[first][ok].view(np.uint32), o.az[second][ok].view(np.uint32)), "azimuth bits changed"
    return out, prm


def duplicates(port, seed: int):
    """A VLP-16 scan with exact copies of 500 of its points, half right after the original, half appended: equal azimuth,
    planar range and star-sector radius (flags bit1 as well as bit2)."""
    pts = make_scan("C1", seed)
    rng = np.random.default_rng(seed)
    pick = np.sort(rng.choice(np.flatnonzero(np.any(pts[:, :3] != 0, axis=1)), 500, replace=False))
    out = np.concatenate([np.insert(pts, pick[:250] + 1, pts[pick[:250]], axis=0), pts[pick[250:]]])
    prm = make_params(**FULL_ROI)
    assert port.run(out, prm).flags & 6 == 6
    return out, prm


def _ring(az_deg, planar, z, rng):
    az = np.deg2rad(np.asarray(az_deg, np.float64))
    n = az.size
    pts = np.zeros((n, 4), np.float32)
    pts[:, 0] = planar * np.cos(az)
    pts[:, 1] = planar * np.sin(az)
    pts[:, 2] = z
    pts[:, 3] = rng.uniform(0, 255, n)
    return pts


def same_xy_ring(port, m: int, regime: str, seed: int):
    """A ring of m points that share one (x, y), so one azimuth, with z varied inside `interval`, shuffled into a filler
    ring of 600 distinct azimuths at another elevation. Asserts the k_sort_rings path (`regime`) of the tied ring."""
    rng = np.random.default_rng(seed)
    filler = _ring(rng.uniform(0.0, 359.9, 600), rng.uniform(3.0, 30.0, 600), 0.0, rng)
    filler[:, 2] = -np.tan(np.deg2rad(30.0)) * np.hypot(filler[:, 0], filler[:, 1])     # elevation -30 deg
    ring = _ring(np.full(m, 37.3), 10.0, 0.0, rng)
    ring[:, 2] = rng.uniform(-1.80, -1.70, m)                                           # elevation about -10 deg
    pts = np.concatenate([filler, ring])
    pts = pts[rng.permutation(pts.shape[0])]
    prm = make_params(interval=3.0, **FULL_ROI)
    rings = _rings_of(port.run(pts, prm, debug=True))
    assert sorted(r.size for r in rings) == sorted([600, m])
    tied = next(r for r in rings if r.size == m and np.unique(r.view(np.uint32)).size == 1)
    assert max_bin_count(tied) == m and ring_regime(tied) == regime, (m, ring_regime(tied))
    return pts, prm


def ring_with_pairs(port, seed: int, m: int = 2000, pairs: int = 12):
    """A ring of m distinct azimuths plus `pairs` second returns at 2x the range: tied pairs inside the counting sort,
    whose bins stay below the crowding cap."""
    rng = np.random.default_rng(seed)
    ring = _ring(rng.uniform(0.0, 359.9, m), rng.uniform(4.0, 20.0, m), 0.0, rng)
    ring[:, 2] = -np.tan(np.deg2rad(10.0)) * np.hypot(ring[:, 0], ring[:, 1]) * rng.uniform(0.99, 1.01, m)
    sec = ring[rng.choice(m, pairs, replace=False)].copy()
    sec[:, :3] *= np.float32(2.0)
    pts = np.concatenate([ring, sec])
    pts = pts[rng.permutation(pts.shape[0])]
    prm = make_params(interval=3.0, **FULL_ROI)
    (r,) = _rings_of(port.run(pts, prm, debug=True))
    assert r.size == m + pairs and np.unique(r.view(np.uint32)).size == m and ring_regime(r) == "fast"
    return pts, prm


def nan_azimuth(port, several: int, seed: int):
    """Two rings near the nadir and the zenith (planar range 4-5 cm at |z| = 1.7 m) and points with x == y == 0 inside
    them: one below the sensor (azimuth NaN, nadir ring) and `several` above it (zenith ring). blind_spots is off: with it
    on, the reference's prefix scans stop at a NaN azimuth (DESIGN.md deviation 3) and labels would differ by design."""
    rng = np.random.default_rng(seed)
    lo = _ring(rng.uniform(0.0, 359.9, 200), rng.uniform(0.04, 0.05, 200), -1.7, rng)
    hi = _ring(rng.uniform(0.0, 359.9, 200), rng.uniform(0.04, 0.05, 200), 1.7, rng)
    z = np.zeros((1 + several, 4), np.float32)
    z[0, 2] = -1.7
    z[1:, 2] = rng.uniform(1.6, 1.8, several)
    z[:, 3] = 7.0
    pts = np.concatenate([lo, hi, z])
    pts = pts[rng.permutation(pts.shape[0])]
    prm = make_params(interval=3.0, blind_spots=0, **FULL_ROI)
    o = port.run(pts, prm, debug=True)
    nan = np.isnan(o.az) & (o.ring >= 0)
    assert nan.sum() == 1 + several and np.unique(o.ring[nan]).size == (2 if several else 1)
    return pts, prm


def _match_range(x, y, target):
    """y' within 64 ulps of y, nearest first, such that planar_range(x, y') has the bits of `target`; None if none does."""
    ks = np.array(sorted(range(-64, 65), key=abs))
    yy = _ulps(np.full(ks.size, y, np.float32), ks)
    r = planar_range(np.stack([np.full(ks.size, x, np.float32), yy], 1))
    hit = np.flatnonzero(r == target)
    return yy[hit[0]] if hit.size else None


def equal_range(port, seed: int, across_rings: bool, want: int = 100):
    """Marker ties: copies of the winning vertex of degree bins, turned by a few hundredths of a degree inside the bin and
    moved by ulps to the winner's bit-identical planar range. In the same ring (same z) on a VLP-16 scan with every
    detector on; or, across_rings, in the neighbouring ring of the bin (its elevation), with the detectors off so the copy
    stays road. Asserts that at least `want` bins end up with a shared farthest range (policy(...).shared_max)."""
    rng = np.random.default_rng(seed)
    pts = make_scan("C1", seed)
    over = dict(x_zero_method=0, z_zero_method=0, star_shaped_method=0) if across_rings else {}
    prm = make_params(**over, **FULL_ROI)
    o = port.run(pts, prm, debug=True)
    pol = policy(pts, o)
    az = np.asarray(o.az, np.float32)
    ring = np.asarray(o.ring)
    d = planar_range(pts)
    add = []
    for p in pol.winners:
        a = float(az[p])
        for delta in (rng.uniform(0.01, 0.04), -rng.uniform(0.01, 0.04)):
            if np.floor(a + delta) != np.floor(a):
                continue
            th = np.arctan2(pts[p, 1], pts[p, 0]) + np.deg2rad(delta)
            x = np.float32(d[p] * np.cos(th))
            yy = _match_range(x, np.float32(d[p] * np.sin(th)), d[p])
            if yy is None:
                continue
            q = pts[p].copy()
            q[0], q[1] = x, yy
            if across_rings:
                others = np.flatnonzero((ring >= 0) & (ring != ring[p]) & (np.floor(az) == np.floor(a)) & (np.abs(ring - ring[p]) == 1))
                if others.size == 0:
                    break
                r2 = others[0]
                q[2] = np.float32(pts[r2, 2] * d[p] / d[r2])                      # the other ring's elevation
            add.append(q)
            break
    out = np.concatenate([pts, np.array(add, np.float32)])
    res = port.run(out, prm, debug=True)
    got = policy(out, res)
    assert not (res.flags & 4), "distinct azimuths: the port's order is the policy's"
    assert got.shared_max >= want, f"only {got.shared_max} degree bins share their farthest range"
    return out, prm



# name -> builder(port): the tie clouds of tests/test_ties.py and tests/test_gpu_ties.py (and of the reference's fixture
# tests/golden/ref/ties.npz, tests/golden/make_golden.py --ref-checks)
CASES = {
    "dual_appended": lambda port: dual_return(port, 5, False),
    "dual_interleaved": lambda port: dual_return(port, 6, True),
    "duplicates": lambda port: duplicates(port, 7),
    "xy2_fast": lambda port: same_xy_ring(port, 2, "fast", 2),
    "xy48_fast": lambda port: same_xy_ring(port, 48, "fast", 48),
    "xy49_smem": lambda port: same_xy_ring(port, 49, "smem", 49),
    "xy4096_smem": lambda port: same_xy_ring(port, 4096, "smem", 4096),
    "xy4097_global": lambda port: same_xy_ring(port, 4097, "global", 4097),
    "xy7000_global": lambda port: same_xy_ring(port, 7000, "global", 7000),
    "pairs_in_counting_sort": lambda port: ring_with_pairs(port, 11),
    "nan_lone": lambda port: nan_azimuth(port, 0, 20),
    "nan_several": lambda port: nan_azimuth(port, 3, 23),
    "equal_range_ring": lambda port: equal_range(port, 8, False),
    "equal_range_across": lambda port: equal_range(port, 7, True),
}
EQUAL_RANGE = ("equal_range_ring", "equal_range_across")

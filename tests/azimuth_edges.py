"""blindSpots windows, blind quarters and marker bins where azimuths lie exactly on their bounds.

The device replaces the reference's window loops (blind_spots.cpp:68-283) by per-(ring, degree) curb bins, a reach table
per window start and the threshold rows Tf / Tb; the argument that they agree rests on inclusive and exclusive float
comparisons at the window bounds. Scans with random azimuths almost never put a point exactly on such a bound. This
module builds clouds that do, and restates the bounds in numpy, bit for bit, from the oracle port's debug tables:

  * hi_k(i): ring 0 `f32(i) + f32(beamZone)` (:107), rings k >= 1 `f32(f64(i) + A[k])` (:142), 360 at the forward
    start i == 360 - beamZone (:136-139); lo_k(i) the same with `-`, 0 at the backward start i == beamZone (:245-248);
  * whether a start is accepted for ring k: inside the loop range, not blind (is_blind of q1..q4, :72-99 / :181-208) and
    reach[dir][i] > k;
  * Tf[k][j] = hi_k of the largest accepted forward start <= j (-inf if none), Tb[k][j] = lo_k of the smallest accepted
    backward start >= j (+inf if none): a point of ring k with azimuth a is road iff a <= Tf[k][floor a] or
    Tb[k][ceil a] <= a (urf_logic.cuh covered_T), and iff some accepted window contains it (checked both ways).

Points are placed with `exact_azimuth`: float (x, y) whose azimuth in the port's debug run has exactly the target's bits.
Azimuth convention (lidar_segmentation.cpp:254-269): 0 on -y, 90 on +x, 180 on +y, 270 on -x; exactly 360.0 comes from
x = -tiny, y < 0. Near the x axis the azimuth comes from asinf close to 1 and is coarse (steps of about 0.02 degrees at
90 and 270): some floats there are unreachable, so builders that aim at arbitrary thresholds keep the reachable ones.

Curb points are made by the star-shaped search (star_shaped_search.cpp:112-150): a target T of ring k at a planar range
below every point of the scan and a helper H at exactly half T's x and y (the same star sector), 1.5 m lower. H is the
first point of the sector by radius, T the second, and the slope from H to T exceeds the slope parameter, so T is
marked. H's elevation matches no ring and every channel is taken (channels = the sensor's ring count), so H joins no
ring. Road points sit at the ring's median planar range and its elevation, so they move neither maxDistance (A) nor
the curb bins. Every builder asserts its targets on the final port run: azimuth bits, ring, detector label, and what the
target is there for (a threshold value, a window blocked at exactly its ring, a blind start, a marker vertex)."""
from __future__ import annotations

import numpy as np

from urban_road_filter_b200 import FULL_ROI, make_params
from urban_road_filter_b200.synth import SHAPES, make_scan

from util import _ulps

f32 = np.float32
NDEG = 361


# ---------------------------------------------------------------------------------------------------------------------
# exact azimuths

def _probe(port, xy):
    """Port azimuths of float (x, y) points: one ring (z = -1.7, planar ranges alike), no detectors, no blind spots."""
    pts = np.zeros((max(xy.shape[0], 30), 4), np.float32)
    pts[:, 1] = -5.0
    pts[: xy.shape[0], :2] = xy
    pts[:, 2] = -1.7
    pts[:, 3] = 1.0
    o = port.run(pts, make_params(channels=1, interval=90.0, blind_spots=0, x_zero_method=0, z_zero_method=0,
                                  star_shaped_method=0, **FULL_ROI), debug=True)
    assert np.all(o.ring[: xy.shape[0]] == 0)
    return np.asarray(o.az, np.float32)[: xy.shape[0]]


def exact_azimuth(port, targets, radius, K: int = 48, strict: bool = True):
    """(xy [T, 2] float32, found [T] bool): for every target azimuth a float point at about `radius` whose port azimuth
    has the target's bits. Candidates: the float point nearest the target direction and its +-K-ulp neighbours along
    each coordinate, all evaluated in one port call; the candidate nearest the start wins. strict: assert all found."""
    t = np.asarray(targets, np.float32).reshape(-1)
    th = np.deg2rad(t.astype(np.float64))
    x0 = (radius * np.sin(th)).astype(np.float32)
    y0 = (-radius * np.cos(th)).astype(np.float32)
    x0 = np.where(t == f32(360.0), f32(-1e-30), x0)          # 360.0: x just below zero, y < 0
    x0 = np.where((t == f32(0.0)) | (t == f32(180.0)), f32(0.0), x0)   # on the axes
    y0 = np.where((t == f32(90.0)) | (t == f32(270.0)), f32(0.0), y0)
    ks = np.array(sorted(range(-K, K + 1), key=lambda v: (abs(v), v)))
    cand = []
    for k in ks:
        cand.append(np.stack([_ulps(x0, k), y0], 1))
        cand.append(np.stack([x0, _ulps(y0, k)], 1))
    for dx in range(-6, 7):                                   # both coordinates: where one ulp turns by more than
        for dy in range(-6, 7):                               # one ulp of the azimuth
            cand.append(np.stack([_ulps(x0, dx), _ulps(y0, dy)], 1))
    cand = np.stack(cand, 1).astype(np.float32)               # [T, C, 2], nearest first
    az = _probe(port, cand.reshape(-1, 2)).reshape(cand.shape[:2])
    hit = az.view(np.uint32) == t.view(np.uint32)[:, None]
    x, y = cand[..., 0], cand[..., 1]
    hit &= ~((x > 0) & (y < 0) & (-y < 1e-6 * x))            # atan2f in (-6.4e-8, 0): the reference's star search
                                                              # reads beamp[360] there (DESIGN.md deviation 1)
    found = hit.any(1)
    first = np.argmax(hit, 1)
    xy = cand[np.arange(t.size), first]
    if strict:
        assert found.all(), f"no float point with azimuth {t[~found][:8]}"
    return xy, found


# ---------------------------------------------------------------------------------------------------------------------
# window bounds, bit-exact

class Windows:
    """The blindSpots tables of one port debug run `o` under parameters `prm`, restated in numpy."""

    def __init__(self, prm, o):
        self.R = R = int(o.n_rings)
        bz = f32(prm.beamZone)
        self.bz = bz
        lim_f, lim_b = f32(f32(360.0) - bz), bz                  # blind_spots.cpp:68 / :177 (int vs float)
        i = np.arange(NDEG)
        fi = i.astype(np.float32)
        self.in_f, self.in_b = fi <= lim_f, fi >= lim_b
        self.sp_f = np.flatnonzero(fi == lim_f)                   # :136 `i == 360 - beamZone`
        self.sp_b = np.flatnonzero(fi == lim_b)                   # :245 `i == 0 + beamZone`
        self.q = q = np.asarray(o.q, np.float32)
        self.blind = blind_starts(prm, q)
        A = np.asarray(o.A, np.float64)
        hi = np.empty((R, NDEG), np.float32)
        lo = np.empty((R, NDEG), np.float32)
        hi[0], lo[0] = fi + bz, fi - bz
        for k in range(1, R):
            hi[k] = (i.astype(np.float64) + A[k]).astype(np.float32)
            lo[k] = (i.astype(np.float64) - A[k]).astype(np.float32)
            hi[k, self.sp_f] = f32(360.0)
            lo[k, self.sp_b] = f32(0.0)
        self.hi, self.lo = hi, lo
        reach = np.asarray(o.reach, np.int64).reshape(2, NDEG)
        skipped = np.stack([~self.in_f | self.blind, ~self.in_b | self.blind])
        assert np.array_equal(reach < 0, skipped), "the port skips other window starts than the restatement"
        self.reach = reach
        k = np.arange(R)[:, None]
        self.acc_f = self.in_f & ~self.blind & (reach[0] > k)
        self.acc_b = self.in_b & ~self.blind & (reach[1] > k)
        self.Tf = np.full((R, NDEG), -np.inf, np.float32)
        self.Tb = np.full((R, NDEG), np.inf, np.float32)
        for kk in range(R):
            last = np.maximum.accumulate(np.where(self.acc_f[kk], i, -1))
            nxt = np.minimum.accumulate(np.where(self.acc_b[kk], i, NDEG)[::-1])[::-1]
            self.Tf[kk] = np.where(last >= 0, hi[kk, np.maximum(last, 0)], -np.inf)
            self.Tb[kk] = np.where(nxt <= 360, lo[kk, np.minimum(nxt, 360)], np.inf)

    def covered(self, k, a):
        """a <= Tf[k][floor a] || Tb[k][ceil a] <= a (a in [0, 360])."""
        k, a = np.asarray(k), np.asarray(a, np.float32)
        j = np.minimum(np.floor(a), 360).astype(np.int64)
        jc = np.minimum(np.ceil(a), 360).astype(np.int64)
        return (a <= self.Tf[k, j]) | (self.Tb[k, jc] <= a)

    def covered_by_windows(self, k, a):
        """Some accepted window contains a: i <= a <= hi_k(i) forward, lo_k(i) <= a <= i backward."""
        k, a = np.asarray(k), np.asarray(a, np.float32)[:, None]
        fi = np.arange(NDEG, dtype=np.float32)[None]
        fwd = self.acc_f[k] & (fi <= a) & (a <= self.hi[k])
        bwd = self.acc_b[k] & (self.lo[k] <= a) & (a <= fi)
        return (fwd | bwd).any(1)


def blind_starts(prm, q):
    """is_blind (blind_spots.cpp:72-99, :181-208) for every window start 0..360."""
    i = np.arange(NDEG)
    fi = i.astype(np.float32)
    q1, q2, q3, q4 = (f32(v) for v in q)
    if not prm.blind_spots:
        return np.zeros(NDEG, bool)
    if prm.xDirection == 0:
        return ((q1 != 0) & (q4 != 360) & ((fi <= q1) | (fi >= q4))) | ((q2 != 180) & (q3 != 180) & (fi >= q2) & (fi <= q3))
    if prm.xDirection == 1:
        return ((q2 != 180) & (fi >= q2) & (i <= 270)) | ((q1 != 0) & ((fi <= q1) | (i >= 270)))
    return ((q4 != 360) & ((fi >= q4) | (i <= 90))) | ((q3 != 180) & (fi <= q3) & (i >= 90))


def check_labels(pts, o, prm):
    """Every ring point that no detector marked is road exactly where both formulations of the window test say so."""
    w = Windows(prm, o)
    ring, az = np.asarray(o.ring), np.asarray(o.az, np.float32)
    sel = np.flatnonzero((ring >= 0) & (np.asarray(o.det_label) != 2) & (az >= 0))
    cov = w.covered(ring[sel], az[sel])
    np.testing.assert_array_equal(cov, w.covered_by_windows(ring[sel], az[sel]))
    np.testing.assert_array_equal(np.asarray(o.label)[sel] == 1, cov)
    return w


# ---------------------------------------------------------------------------------------------------------------------
# builders

class Scene:
    """A base scan plus points appended at exact azimuths. channels = the sensor's ring count, so no new ring appears."""

    def __init__(self, port, shape, order, seed, **over):
        self.port, self.sh = port, SHAPES[shape]
        self.base = make_scan(shape, seed, order=order)
        self.prm = make_params(channels=self.sh.rings, interval=self.sh.interval, **{**FULL_ROI, **over})
        self.o0 = port.run(self.base, self.prm, debug=True)
        assert self.o0.status == 0 and self.o0.n_rings == self.sh.rings
        ring = np.asarray(self.o0.ring)
        pr = np.hypot(self.base[:, 0], self.base[:, 1])
        self.r_ground = np.array([np.median(pr[ring == k]) for k in range(self.sh.rings)])
        self.slope = np.array([np.median(self.base[ring == k, 2] / pr[ring == k]) for k in range(self.sh.rings)])
        self.r_curb = 0.4 * pr[ring >= 0].min()
        self.w0 = Windows(self.prm, self.o0)
        self.add, self.want = [], []                   # appended rows; (row, ring, target, curb) per target

    def road(self, k, targets, strict=True, radius=None):
        t = np.asarray(targets, np.float32)
        xy, found = exact_azimuth(self.port, t, self.r_ground[k] if radius is None else radius, strict=strict)
        for (x, y), a in zip(xy[found], t[found]):
            self._push(k, a, x, y, False)
        return t[found]

    def curb(self, k, targets):
        t = np.asarray(targets, np.float32)
        xy, _ = exact_azimuth(self.port, t, self.r_curb)
        for (x, y), a in zip(xy, t):
            self._push(k, a, x, y, True)
            h = np.array([x * f32(0.5), y * f32(0.5), 0.0, 3.0], np.float32)
            h[2] = f32(self.slope[k] * np.hypot(x, y)) - f32(1.5)
            self.add.append(h)
        return t

    def _push(self, k, a, x, y, curb):
        p = np.array([x, y, self.slope[k] * np.hypot(float(x), float(y)), 2.0 if curb else 1.0], np.float32)
        self.want.append((self.base.shape[0] + len(self.add), k, f32(a), curb))
        self.add.append(p)

    def finish(self):
        """(pts, prm, o): the final cloud, its parameters and port debug run; asserts every target's azimuth bits, ring
        and detector label and the labels against the numpy window tests. A road point the detectors take for a curb
        (the star search, when it lands just above a noisy neighbour of its sector) is dropped and the cloud rebuilt."""
        while True:
            pts = np.concatenate([self.base, np.array(self.add, np.float32).reshape(-1, 4)])
            o = self.port.run(pts, self.prm, debug=True)
            bad = [row for row, k, a, curb in self.want if not curb and o.det_label[row] == 2]
            if not bad:
                break
            keep = np.setdiff1d(np.arange(len(self.add)), np.array(bad) - self.base.shape[0])
            shift = np.cumsum(np.isin(np.arange(len(self.add)), np.array(bad) - self.base.shape[0]))
            self.add = [self.add[j] for j in keep]
            n0 = self.base.shape[0]
            self.want = [(row - int(shift[row - n0]), k, a, c) for row, k, a, c in self.want if row not in bad]
        assert o.status == 0 and o.n_rings == self.sh.rings
        assert np.all(o.ring[self.base.shape[0]:][np.asarray(self.add)[:, 3] == 3.0] == -1), "a helper joined a ring"
        for row, k, a, curb in self.want:
            assert o.ring[row] == k, (row, k, o.ring[row])
            assert o.az[row].view(np.uint32) == a.view(np.uint32), (row, a, o.az[row])
            assert (o.det_label[row] == 2) == curb, (row, k, a, curb, o.det_label[row])
        self.w = check_labels(pts, o, self.prm)
        return pts, self.prm, o

    def rows(self, curb=None, k=None):
        return [(r, kk, a) for r, kk, a, c in self.want if (curb is None or c == curb) and (k is None or kk == k)]


def _spaced(cands, gap, n):
    out = []
    for c in cands:
        if all(abs(c - d) >= gap for d in out):
            out.append(c)
        if len(out) == n:
            break
    return out


def integer_azimuths(port, shape, order, seed):
    """Curb and road points on integer degrees, 0.0, 90, 180, 270 and 360.0 among them, on ring 0, ring 1 and a higher
    ring. Road points at every reachable integer degree of those rings, and at 360.0 on four rings at the far end of the
    ring's range (the only points of marker bin 360); curbs at 0, 90, 180, 270 and a few integers between them on one
    ring each (one per star sector). A curb at integer i is the first non-road point of bin i in scan order."""
    s = Scene(port, shape, order, seed)
    hk = s.sh.rings // 2
    ints = np.arange(NDEG, dtype=np.float32)
    for k in (0, 1, hk):
        got = s.road(k, ints, strict=False)
        assert np.isin([0, 90, 180, 270, 360], got).all() and got.size >= 280, (k, got.size)
    for k in (1, 2, 3, hk):
        s.road(k, [360.0], radius=0.999 * float(s.o0.max_dist[k]))
    s.curb(0, [25.0, 137.0, 225.0])
    s.curb(1, [90.0, 181.0, 300.0])
    s.curb(hk, [12.0, 180.0, 270.0])
    pts, prm, o = s.finish()
    for k in (0, 1, hk):
        got = [a for _, _, a in s.rows(curb=False, k=k)]
        assert np.isin([0, 90, 180, 270, 360], got).sum() >= (3 if k == 1 else 5) and len(got) >= 180, (k, len(got))
    return pts, prm


def thresholds(port, shape, order, seed):
    """Road points exactly on Tf[k][j] / Tb[k][j] where a run of accepted starts ends, with +-1-ulp companions, on
    rings 0, 1 and three rings k >= 2 (at most ten run ends per ring). The star search is off: it would take some of
    the road points for curbs."""
    s = Scene(port, shape, order, seed, star_shaped_method=0)
    w = s.w0
    R = w.R
    rings = (0, 1, 2, R // 3, (2 * R) // 3)
    exact = []
    for k in rings:
        end_f = np.flatnonzero(w.acc_f[k] & ~np.append(w.acc_f[k, 1:], False))          # last start of a run
        end_b = np.flatnonzero(w.acc_b[k] & ~np.insert(w.acc_b[k, :-1], 0, False))     # first start of a run
        tv = [w.hi[k, i] for i in end_f if w.hi[k, i] <= 360] + [w.lo[k, i] for i in end_b if w.lo[k, i] >= 0]
        tv = _spaced(tv, 3.0, 10)
        t3 = np.array([[_ulps(v, -1), v, _ulps(v, 1)] for v in tv], np.float32).reshape(-1)
        got = s.road(k, t3, strict=False)
        exact += [(k, v) for v in tv if np.isin(v, got)]
    assert len(exact) >= 10, len(exact)
    pts, prm, o = s.finish()
    w1 = s.w
    on = 0
    for k, v in exact:
        j, jc = int(min(np.floor(v), 360)), int(min(np.ceil(v), 360))
        on += int(w1.Tf[k, j] == v or w1.Tb[k, jc] == v)
    assert on == len(exact), f"only {on} of {len(exact)} threshold points still sit on a threshold"
    return pts, prm


def curb_bounds(port, shape, order, seed):
    """Curb points of a ring exactly at a window's hi_k(i) (forward, the last bin of CurbView::fwd), at lo_k(i)
    (backward, `mx(k, lb) >= lo`) and at an integer start i (backward, `azimuth == i`), each in a window that rings
    0..k accept in the base scan and spaced apart: on the final run window i is blocked at exactly ring k, by this curb
    alone. Blind spots off: the curbs made here may take the star mark of a ring-1 point and move q1..q4."""
    base = Scene(port, shape, order, seed, blind_spots=0)
    w = base.w0
    R = w.R
    plan = []                                    # (dir, i, k, azimuth, kind)
    for k in (0, 1, R // 4, R // 2):
        for dir_, kind in ((0, "hi"), (1, "lo"), (1, "int")):
            acc = (w.acc_f if dir_ == 0 else w.acc_b)[k]
            for i in np.flatnonzero(acc):
                a = w.hi[k, i] if kind == "hi" else w.lo[k, i] if kind == "lo" else f32(i)
                if not (0 < a < 360) or (kind == "int" and i in w.sp_b) or (kind != "int" and a == np.floor(a)):
                    continue
                if all(abs(float(a) - float(p[3])) >= 2 * float(w.bz) + 20 for p in plan):
                    if exact_azimuth(port, [a], base.r_curb, strict=False)[1][0]:
                        plan.append((dir_, int(i), k, f32(a), kind))
                        break
    for _ in range(3):                           # a new curb can change the ring's x-/z-zero marks next to it: drop
        s = Scene(port, shape, order, seed, blind_spots=0)          # the windows that then hold another curb
        for p in plan:
            s.curb(p[2], [p[3]])
        pts, prm, o = s.finish()
        ring, az, det = np.asarray(o.ring), np.asarray(o.az, np.float32), np.asarray(o.det_label)
        ok = []
        for dir_, i, k, a, kind in plan:
            lo, hi = (f32(i), s.w.hi[k, i]) if dir_ == 0 else (s.w.lo[k, i], f32(i))
            inside = (ring == k) & (det == 2) & (az >= lo) & (az <= hi)
            alone = inside.sum() == 1 and az[inside][0] == a
            ok.append(bool(alone and s.w.reach[dir_, i] == k))
        if all(ok):
            break
        plan = [p for p, g in zip(plan, ok) if g]
    assert all(ok) and len(plan) >= 2 and len({p[4] for p in plan}) >= 2, plan
    return pts, prm


def blind_quarters(port, shape, order, seed, xdir):
    """Ring-1 curbs at exactly 0, 90, 180, 270 and integer q1 = 20, q3 = 200 (the largest of their quarters): q2 = 90,
    q4 = 270, and window starts 20, 90, 200 and 270 are blind by an inclusive comparison."""
    s = Scene(port, shape, order, seed, xDirection=xdir)
    s.curb(1, [0.0, 20.0, 90.0, 180.0, 200.0, 270.0])
    pts, prm, o = s.finish()
    assert np.array_equal(np.asarray(o.q, np.float32), np.array([20.0, 90.0, 200.0, 270.0], np.float32)), o.q
    assert s.w.blind.sum() > 0
    return pts, prm


def blind_360(port, shape, order, seed, xdir):
    """A ring-1 curb at exactly 360.0 is quarter 4's smallest: q4 = 360 stays at its default; q1 = 75."""
    s = Scene(port, shape, order, seed, xDirection=xdir)
    s.curb(1, [360.0])
    s.curb(1, [75.0])
    pts, prm, o = s.finish()
    assert o.q[3] == f32(360.0) and o.q[0] == f32(75.0)
    return pts, prm


def special_windows(port, shape, order, seed, beam, which):
    """Points at 0.0 and 360.0 on rings >= 1 with an integer beamZone (the windows of start 360 - beamZone and of
    start beamZone reach 360 and 0) or a non-integer one (no such start). which = 0: curbs at 0.0 on rings 1 and 2 (one
    star sector: ring 1 only) and road points at 360.0; which = 360: the reverse."""
    s = Scene(port, shape, order, seed, beamZone=beam)
    R = s.w0.R
    cur, road = (f32(0.0), f32(360.0)) if which == 0 else (f32(360.0), f32(0.0))
    s.curb(1, [cur])
    for k in (1, 2, 3, R // 2, R - 1):
        s.road(k, [road, cur])
    pts, prm, o = s.finish()
    assert (len(s.w.sp_f) == 1) == (beam == int(beam))
    return pts, prm


# name -> builder(port) -> (pts, params): the clouds of tests/test_azimuth_edges.py and tests/test_gpu_azimuth_edges.py
# (and of the reference's fixture tests/golden/ref/azimuth_edges.npz, tests/golden/make_golden.py --ref-checks).
# BASE[name] = (shape, seed, order) of the scan the cloud starts with; the fixture stores the rows appended to it.
CASES, BASE = {}, {}
for _sh, _seed in (("C1", 31), ("C2", 32)):
    for _o in ("column", "ring"):
        _t = f"{_sh}_{_o}"
        CASES[f"integer_{_t}"] = (lambda sh, o, sd: lambda port: integer_azimuths(port, sh, o, sd))(_sh, _o, _seed)
        CASES[f"thresholds_{_t}"] = (lambda sh, o, sd: lambda port: thresholds(port, sh, o, sd + 1))(_sh, _o, _seed)
        CASES[f"curb_bounds_{_t}"] = (lambda sh, o, sd: lambda port: curb_bounds(port, sh, o, sd + 2))(_sh, _o, _seed)
        BASE[f"integer_{_t}"], BASE[f"thresholds_{_t}"], BASE[f"curb_bounds_{_t}"] = \
            (_sh, _seed, _o), (_sh, _seed + 1, _o), (_sh, _seed + 2, _o)
for _x in (0, 1, 2):
    CASES[f"blind_xdir{_x}"] = (lambda x: lambda port: blind_quarters(port, "C1", "column", 40 + x, x))(_x)
    CASES[f"blind360_xdir{_x}"] = (lambda x: lambda port: blind_360(port, "C1", "ring", 43 + x, x))(_x)
    BASE[f"blind_xdir{_x}"], BASE[f"blind360_xdir{_x}"] = ("C1", 40 + _x, "column"), ("C1", 43 + _x, "ring")
for _b in (30.0, 45.5):
    for _w in (0, 360):
        CASES[f"special_bz{_b:g}_at{_w}"] = (lambda b, w: lambda port: special_windows(port, "C1", "column", 50, b, w))(_b, _w)
        BASE[f"special_bz{_b:g}_at{_w}"] = ("C1", 50, "column")


def base_scan(name):
    shape, seed, order = BASE[name]
    return make_scan(shape, seed, order=order)

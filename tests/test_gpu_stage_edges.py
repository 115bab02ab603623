"""Device stages at the edges where kernels go wrong, each compared with the CPU oracle stage by stage (util.stage_diffs:
star sector of every point, ring angles, maxDistance, q1..q4, ring widths, window reach, then labels, order, vertices):
star sectors on knife edges, the blindSpots tables across the detector toggles, device-resident batches with odd
strides, scan lengths at tile edges and on both sides of the marker-kernel switch, and a scan of 2^24 points."""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle.pyoracle import PortOracle
from urban_road_filter_b200 import FULL_ROI, UrfResult, api, make_params
from urban_road_filter_b200.synth import SHAPES, make_scan, random_cloud

from util import HUGE_ROI, SECTOR_RADII, GpuDebug, sector_boundary_cloud, stage_diffs

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def port():
    return PortOracle()


@pytest.fixture(scope="module")
def det():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    d = api.Detector(max_points=300_032, max_batch=2)
    yield d
    d.close()


def run_stages(det, port, pts, prm):
    """One host-buffer call; every stage against the oracle's debug run. Returns (device result, oracle result)."""
    det.set_params(prm)
    r = det.filtered(pts)
    o = port.run(pts, prm, debug=True)
    if o.status == 0 and r.status == 0:
        g = GpuDebug(det, r, pts.shape[0])
        bad = stage_diffs(o, g, pts.shape[0])
        if "sector" in bad:
            i = np.flatnonzero(o.sector != g.sector)[:8]
            bad.append(f"sector at {list(zip(pts[i, 0].tolist(), pts[i, 1].tolist(), o.sector[i].tolist(), g.sector[i].tolist()))}")
    else:
        bad = [] if o.status == r.status else ["status"]
    assert bad == [], f"stages differing from the oracle: {bad}"
    return r, o


@pytest.mark.parametrize("starbeam", [0, 1])
@pytest.mark.parametrize("r", SECTOR_RADII)
def test_gpu_star_sector_boundaries(det, port, r, starbeam):
    """k_points' star sector (fast path with __fdividef, exact fallback) on points within ulps of every integer-degree
    boundary and of the fast path's margin, on the axes with +-0.0, at the 0/360 wrap, subnormal, and beyond 2^126 where
    __fdividef returns 0: the oracle's sector for every point, with and without the rectangular beam filter."""
    for huge in (False, True):
        pts = sector_boundary_cloud(r, seed=int(r * 10), huge=huge)
        _, o = run_stages(det, port, pts, make_params(starbeam_filter=starbeam, **(HUGE_ROI if huge else FULL_ROI)))
        assert o.status == 0 and (o.sector >= 0).sum() > pts.shape[0] // 3


@pytest.mark.parametrize("mask", range(16))
def test_gpu_ring_and_blind_spot_tables(det, port, mask):
    """k_ring_detect / k_tab1 / k_reach tables (maxDistance, q1..q4, ring widths, window reach) one by one, for every
    detector toggle, xDirection 0/1/2 and beamZone at both ends of its range. The OS1-64 scene puts curbs into ring 1 in
    all four quarters, so q1..q4 all move off their defaults; the curved VLP-16 scene has few rings and wide windows."""
    toggles = dict(x_zero_method=mask & 1, z_zero_method=(mask >> 1) & 1, star_shaped_method=(mask >> 2) & 1, blind_spots=(mask >> 3) & 1)
    clouds = ((make_scan("C2", 3), SHAPES["C2"]), (make_scan("C1", 3, order="ring", curve=1.0), SHAPES["C1"]))
    for pts, sh in clouds:
        for xdir in (0, 1, 2):
            for bz in (10.0, 45.5, 359.5, 360.0):
                run_stages(det, port, pts, make_params(xDirection=xdir, beamZone=bz, channels=sh.channels, interval=sh.interval,
                                                       **toggles, **FULL_ROI))


def _device_batch(d, clouds, S, groups):
    """urf_enqueue_batch_device_ex with the emission order into [B][S] buffers followed by 64 guard entries."""
    B = len(clouds)
    x = torch.zeros((B * S + 64, 4), dtype=torch.float32, device="cuda")
    for b, c in enumerate(clouds):
        x[b * S: b * S + c.shape[0]] = torch.from_numpy(c).cuda()
    lab = torch.full((B * S + 64,), -7, dtype=torch.int32, device="cuda")
    order = torch.full((B * S + 64,), -7, dtype=torch.int32, device="cuda")
    n = (C.c_int * B)(*[c.shape[0] for c in clouds])
    outs = (UrfResult * B)()
    torch.cuda.synchronize()
    d.set_option(2, groups)
    assert d.lib.urf_enqueue_batch_device_ex(d._ctx, x.data_ptr(), S, n, B, lab.data_ptr(), order.data_ptr()) == 0
    assert d.lib.urf_finish_batch_device(d._ctx, outs) == 0
    return lab.cpu().numpy(), order.cpu().numpy(), outs


@pytest.mark.parametrize("stride", ["max_n+1", 7681, 4097])
def test_gpu_odd_strides_device_resident(port, stride):
    """Device-resident batches whose stride is not a multiple of four points: every scan's slice of the sector arrays
    starts off 16-byte alignment (k_star_sort's head and tail copies). Ragged scans, one and three stream groups. Each
    scan equals the host single-scan result byte for byte and the oracle stage by stage; nothing is written past n[b]."""
    d = api.Detector(max_points=30_000, max_batch=8)
    try:
        prm = make_params(**FULL_ROI)
        d.set_params(prm)
        cap = 28_800 if stride == "max_n+1" else stride
        clouds = [make_scan("C1", 70 + s, order=("column", "ring")[s % 2])[: cap - 1013 * s] for s in range(4)]
        clouds += [random_cloud(min(cap, 5000), 5), make_scan("C1", 75)[:29], np.zeros((0, 4), np.float32)]
        S = max(c.shape[0] for c in clouds) + 1 if stride == "max_n+1" else stride
        assert S % 4 != 0
        exp = [port.run(c, prm, debug=True) for c in clouds]
        single = [d.filtered(c) for c in clouds]
        for groups in (1, 3):
            lab, order, outs = _device_batch(d, clouds, S, groups)
            assert np.all(lab[len(clouds) * S:] == -7) and np.all(order[len(clouds) * S:] == -7), "written past the batch"
            for b, (c, o, h) in enumerate(zip(clouds, exp, single)):
                n = c.shape[0]
                lb, ob = lab[b * S: (b + 1) * S], order[b * S: (b + 1) * S]
                assert np.all(lb[n:] == -7) and np.all(ob[n:] == -7), f"scan {b}: written past n[b] (groups={groups})"
                r = api._scan_result(outs[b], lb[:n].copy(), None, ob)
                assert (r.status, r.n_roi, r.n_rings, r.n_order, r.n_road, r.n_curb, r.n_vert, r.flags) == \
                       (h.status, h.n_roi, h.n_rings, h.n_order, h.n_road, h.n_curb, h.n_vert, h.flags), (groups, b)
                assert r.label.tobytes() == h.label.tobytes() and r.vert.tobytes() == h.vert.tobytes(), (groups, b)
                if h.status == 0:
                    assert r.order.tobytes() == h.order.tobytes(), (groups, b)
                    assert stage_diffs(o, GpuDebug(d, r, n, b), n) == [], (groups, b)
                else:
                    assert o.status == h.status
    finally:
        d.close()


@pytest.mark.parametrize("lengths", [(30, 31), (255, 256, 257), (511, 512, 513), (1023, 1024, 1025), (4095, 4096, 4097),
                                     (16383, 16384, 16385)])
def test_gpu_scan_lengths_at_tile_edges(det, port, lengths):
    """Prefixes of one scan one point either side of the 256-point rounding, the 512-point partition chunk and the
    1024-point pack tile: every stage against the oracle."""
    for order in ("column", "ring"):
        pts = make_scan("C2", 41, order=order)
        for n in lengths:
            run_stages(det, port, pts[:n].copy(), make_params(**FULL_ROI))


def test_gpu_marker_kernel_switch(det, port):
    """A scan padded from S = 299,776 to S = 300,032 points (256 points outside the ROI) crosses kMarkSingleMax: the same
    ROI points go through k_markers1 and then k_markers_grid. Labels, order and vertices are identical between the two
    and equal the oracle's."""
    sh = SHAPES["C4"]
    base = make_scan("C4", 42, cols=2343)[:299_776].copy()
    pad = np.tile(np.array([[1000.0, 0.0, 0.0, 1.0]], np.float32), (256, 1))
    prm = make_params(channels=sh.channels, interval=sh.interval, **FULL_ROI)
    a, _ = run_stages(det, port, base, prm)
    b, _ = run_stages(det, port, np.concatenate([base, pad]), prm)
    assert a.status == b.status == 0 and a.n_vert > 0
    assert b.label[:base.shape[0]].tobytes() == a.label.tobytes() and np.all(b.label[base.shape[0]:] == -1)
    assert a.order.tobytes() == b.order.tobytes() and a.vert.tobytes() == b.vert.tobytes()


def test_gpu_index_width_2_24(port):
    """One scan of exactly 2^24 points (urf_create's limit) whose last 51,200 points are the only ones inside the ROI:
    every marker winner has an input index >= 2^23, which the 24-bit index field of the marker keys must carry, and the
    packed clouds span 16,384 pack tiles (k_pack_scan's carry over more than 1024 tiles). Host float4 path and
    PointCloud2 packed path against the oracle."""
    N = 1 << 24
    tail = make_scan("C2", 43, cols=800)
    rng = np.random.default_rng(24)
    pts = np.empty((N, 4), np.float32)
    pts[:, 0] = rng.uniform(50.0, 150.0, N)                   # outside the ROI: x > max_x
    pts[:, 1] = rng.uniform(-10.0, 10.0, N)
    pts[:, 2] = -1.7
    pts[:, 3] = 1.0
    pts[N - tail.shape[0]:] = tail
    prm = make_params(min_x=-40.0, max_x=40.0, min_y=-15.0, max_y=15.0, min_z=-3.0, max_z=1.0)
    d = api.Detector(max_points=N, max_batch=1)
    try:
        d.set_params(prm)
        o = port.run(pts, prm, debug=True)
        assert o.status == 0 and o.n_vert > 0 and o.n_road > 0
        r = d.filtered(pts)
        assert stage_diffs(o, GpuDebug(d, r, N), N) == []
        r, cl = d.filtered_cloud2_packed(pts.view(np.uint8).reshape(-1), N, 16, 0, 4, 8, 12)
        assert r.status == 0 and r.vert.tobytes() == o.vert.tobytes()
        lab, order = np.asarray(o.label), np.asarray(o.order)
        exp = {"road": order[lab[order] == 1], "curb": order[lab[order] == 2], "roi": np.flatnonzero(lab >= 0),
               "road_probably": order[o.ring_start[10]: o.ring_start[11]] if o.n_rings > 10 else order[:0]}
        for key, ids in exp.items():
            e = np.zeros((len(ids), 8), np.float32)
            e[:, 0:3] = pts[ids, 0:3]
            e[:, 3] = 1.0
            e[:, 4] = pts[ids, 3]
            assert cl[key].shape == e.shape and cl[key].tobytes() == e.tobytes(), key
    finally:
        d.close()

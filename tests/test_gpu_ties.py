"""Ties on the device (DESIGN.md deviation 2): rings with bit-identical azimuths in every k_sort_rings regime, NaN
azimuths, and degree bins whose farthest road points share one planar range, through the graphed single scan, the chunked
host batch, the device-resident batch over one and two stream groups, and the packed PointCloud2 clouds. Labels, ring ids,
ring starts, counts and bit1 are the port's; order, vertices, packed clouds and bit2 the policy reference's
(tests/tie_policy.py); order, vertices and flags & 6 the CPU model's as a second witness."""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle.pyoracle import PortOracle
from urban_road_filter_b200 import FULL_ROI, UrfResult, api, make_params
from urban_road_filter_b200.synth import make_scan

import tie_policy as tp
from util import CpuModel, cloud2_records

pytestmark = pytest.mark.gpu

NAMES = list(tp.CASES)


@pytest.fixture(scope="module")
def port():
    return PortOracle()


@pytest.fixture(scope="module")
def model():
    return CpuModel()


@pytest.fixture(scope="module")
def det():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    d = api.Detector(max_points=300_032, max_batch=2)
    yield d
    d.close()


class Expect:
    def __init__(self, port, model, pts, prm):
        self.pts, self.prm = pts, prm
        self.o = port.run(pts, prm, debug=True)
        self.p = tp.policy(pts, self.o)
        self.m = model.run(pts, prm)
        self.nan = bool(np.any(np.isnan(self.o.az) & (self.o.ring >= 0)))


_EXP: dict = {}


def expect(port, model, name) -> Expect:
    if name not in _EXP:
        _EXP[name] = Expect(port, model, *tp.CASES[name](port))
    return _EXP[name]


def check(r, e: Expect, what, ring=True, order=True):
    o, p, m = e.o, e.p, e.m
    assert r.status == o.status == 0, what
    np.testing.assert_array_equal(r.label, o.label, err_msg=f"{what}: labels")
    if ring and r.ring is not None:
        np.testing.assert_array_equal(r.ring, o.ring, err_msg=f"{what}: ring ids")
    assert (r.n_roi, r.n_rings, r.n_order, r.n_road, r.n_curb) == (o.n_roi, o.n_rings, o.n_order, o.n_road, o.n_curb), what
    assert (r.flags & 2) == (o.flags & 2), f"{what}: bit1"
    assert bool(r.flags & 8) == e.nan, f"{what}: bit3"
    assert r.vert.tobytes() == p.vert.tobytes(), f"{what}: vertices differ from the policy's"
    assert r.vert.tobytes() == m.vert.tobytes(), f"{what}: vertices differ from the CPU model's"
    if order:
        np.testing.assert_array_equal(r.ring_start, o.ring_start, err_msg=f"{what}: ring_start")
        np.testing.assert_array_equal(r.order, p.order, err_msg=f"{what}: order differs from the policy's")
        np.testing.assert_array_equal(r.order, m.order, err_msg=f"{what}: order differs from the CPU model's")
        assert bool(r.flags & 4) == p.tie, f"{what}: bit2"
        assert (r.flags & 6) == (m.flags & 6), f"{what}: flags & 6 differ from the CPU model's"
    else:
        assert not (r.flags & 4), f"{what}: bit2 without the emission order"


@pytest.mark.parametrize("name", NAMES)
def test_gpu_ties_single_scan(det, port, model, name):
    """Graphed single-scan call, with the emission order and without it (then no azimuth tie is detected, bit2 stays
    clear, urf_device.cuh F_TIE_AZIMUTH)."""
    e = expect(port, model, name)
    det.set_params(e.prm)
    check(det.filtered(e.pts), e, name)
    check(det.filtered(e.pts, want_order=False), e, name + " without order", order=False)


def test_gpu_ties_chunked_host_batch(port, model):
    """Every tie cloud in one host batch of 21 scans with tie-free scans between them (the chunked copy / compute
    pipeline). Parameters are per context, so the clouds run in groups of equal parameters."""
    groups = {}
    for name in NAMES:
        e = expect(port, model, name)
        groups.setdefault(bytes(e.prm), []).append((name, e))
    d = api.Detector(max_points=32_768, max_batch=24)
    try:
        for items in groups.values():
            prm = items[0][1].prm
            d.set_params(prm)
            fill = [make_scan("C1", 90 + s, order=("column", "ring")[s % 2]) for s in range(21 - len(items))]
            clouds = [e.pts for _, e in items] + fill
            clouds = clouds[::2] + clouds[1::2]                    # tie and tie-free scans mixed
            rs = d.filtered_batch(clouds)
            by_id = {id(e.pts): (n, e) for n, e in items}
            for c, r in zip(clouds, rs):
                if id(c) in by_id:
                    n, e = by_id[id(c)]
                    check(r, e, n + " in a batch")
                else:
                    o = port.run(c, prm, debug=True)
                    p = tp.policy(c, o)
                    np.testing.assert_array_equal(r.label, o.label)
                    np.testing.assert_array_equal(r.order, p.order)
                    assert r.vert.tobytes() == p.vert.tobytes() and bool(r.flags & 4) == p.tie
    finally:
        d.close()


@pytest.mark.parametrize("groups", [1, 2])
def test_gpu_ties_device_resident_batch(port, model, groups):
    """urf_enqueue_batch_device_ex with the emission order, the tie clouds of one parameter set as one device batch."""
    by_prm = {}
    for name in NAMES:
        e = expect(port, model, name)
        by_prm.setdefault(bytes(e.prm), []).append((name, e))
    S = max(e.pts.shape[0] for name in NAMES for e in [expect(port, model, name)])
    d = api.Detector(max_points=S, max_batch=16)
    try:
        for items in by_prm.values():
            clouds = [e.pts for _, e in items]
            while len(clouds) < 4:
                clouds.append(clouds[len(clouds) % len(items)])          # at least two scans per stream group
            B = len(clouds)
            d.set_params(items[0][1].prm)
            x = torch.zeros((B, S, 4), dtype=torch.float32, device="cuda")
            for b, c in enumerate(clouds):
                x[b, : c.shape[0]] = torch.from_numpy(c).cuda()
            lab = torch.full((B, S), -7, dtype=torch.int32, device="cuda")
            order = torch.full((B, S), -7, dtype=torch.int32, device="cuda")
            n = (C.c_int * B)(*[c.shape[0] for c in clouds])
            outs = (UrfResult * B)()
            torch.cuda.synchronize()
            d.set_option(2, groups)
            assert d.lib.urf_enqueue_batch_device_ex(d._ctx, x.data_ptr(), S, n, B, lab.data_ptr(), order.data_ptr()) == 0
            assert d.lib.urf_finish_batch_device(d._ctx, outs) == 0
            lab, order = lab.cpu().numpy(), order.cpu().numpy()
            for b in range(B):
                name, e = items[b % len(items)]
                m = clouds[b].shape[0]
                r = api._scan_result(outs[b], lab[b, :m].copy(), None, order[b], None)
                r.ring_start = e.o.ring_start                      # not returned by this entry point
                check(r, e, f"{name} device batch, {groups} groups")
                assert np.all(lab[b, m:] == -7) and np.all(order[b, m:] == -7)
    finally:
        d.close()


@pytest.mark.parametrize("name", NAMES)
def test_gpu_ties_packed_clouds(det, port, model, name):
    """urf_process_cloud2_packed: the road / curb / road_probably clouds follow the device order, so under ties they are
    the policy's clouds, record for record."""
    e = expect(port, model, name)
    n = e.pts.shape[0]
    det.set_params(e.prm)
    raw = cloud2_records(e.pts, 48, 0, 4, 8, 16, seed=n)
    r, cl = det.filtered_cloud2_packed(raw, n, 48, 0, 4, 8, 16, want_labels=True)
    check(r, e, name + " packed", ring=False)
    for key, ids in e.p.clouds.items():
        ids = np.asarray(ids, np.int64)
        exp = np.zeros((ids.size, 8), np.float32)
        exp[:, 0:3] = e.pts[ids, 0:3]
        exp[:, 3] = 1.0
        exp[:, 4] = e.pts[ids, 3]
        assert cl[key].shape == exp.shape and cl[key].tobytes() == exp.tobytes(), f"{name}: packed {key} cloud"


@pytest.mark.parametrize("name", tp.EQUAL_RANGE)
def test_gpu_equal_range_both_marker_kernels(det, port, model, name):
    """Degree bins whose farthest road points share one planar range: k_markers1 (S <= 300,000) and, padded past 300,000
    points outside the ROI, k_markers_grid (CTAs merge through tab.dmax / tab.best). Both give the first of them in scan
    order, the port's vertex."""
    e = expect(port, model, name)
    assert e.p.shared_max >= 100 and not (e.o.flags & 4)
    det.set_params(e.prm)
    a = det.filtered(e.pts)
    check(a, e, name + " k_markers1")
    assert a.vert.tobytes() == e.o.vert.tobytes()
    pad = np.tile(np.array([[1000.0, 0.0, 0.0, 1.0]], np.float32), (300_032 - e.pts.shape[0], 1))
    b = det.filtered(np.concatenate([e.pts, pad]))
    assert b.vert.tobytes() == a.vert.tobytes(), "k_markers_grid picks another vertex than k_markers1"
    assert b.order.tobytes() == a.order.tobytes() and b.label[: e.pts.shape[0]].tobytes() == a.label.tobytes()

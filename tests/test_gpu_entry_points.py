"""The host-buffer entry points against each other: one scan through urf_process, urf_process_cloud2 (float4-sized and
wider records), urf_process_cloud2_packed and urf_process_cloud2_batch gives byte-identical results and the same kernel
launches; the record staging buffer that the single-scan and batched record calls share; and the argument checks and the
too-few-points result of the single-scan PointCloud2 calls."""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle.pyoracle import PortOracle
from urban_road_filter_b200 import FULL_ROI, UrfResult, api, make_params
from urban_road_filter_b200.ctypes_abi import URF_ERR_CAPACITY, URF_ERR_INVALID, URF_OK, URF_TOO_FEW_POINTS, UrfClouds
from urban_road_filter_b200.synth import make_scan

from util import cloud2_records, stage_diffs

pytestmark = pytest.mark.gpu

# kernels a C1 scan with the emission order launches: k_reset .. k_scatter (6), k_ring_detect4, the star-shaped search
# (k_star_sort, k_star_sort_big, k_star_scan, k_star_refine), k_tab1, k_reach, k_tab2, k_label, k_markers1, k_sort_rings
C1_LAUNCHES = 17
PACK_LAUNCHES = 3          # k_pack_count, k_pack_scan, k_pack_write


@pytest.fixture(scope="module")
def port():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    return PortOracle()


def _same(a, b, what):
    for f in ("status", "n_in", "n_roi", "n_rings", "n_order", "n_road", "n_curb", "n_vert", "flags"):
        assert getattr(a, f) == getattr(b, f), f"{what}: {f}"
    assert a.label.tobytes() == b.label.tobytes(), f"{what}: labels"
    if a.ring is not None and b.ring is not None:
        assert a.ring.tobytes() == b.ring.tobytes(), f"{what}: ring ids"
    assert a.order.tobytes() == b.order.tobytes(), f"{what}: emission order"
    assert a.ring_start.tobytes() == b.ring_start.tobytes(), f"{what}: ring_start"
    assert a.vert.tobytes() == b.vert.tobytes(), f"{what}: vertices"


def test_gpu_one_scan_every_entry_point(port):
    d = api.Detector(max_points=30_000, max_batch=1)
    try:
        prm = make_params(**FULL_ROI)
        d.set_params(prm)
        pts = make_scan("C1", 9)
        n = pts.shape[0]
        ref = d.filtered(pts)                                             # urf_process
        assert d.last_launch_count() == C1_LAUNCHES
        assert ref.status == 0 and stage_diffs(port.run(pts, prm), ref, n) == []
        raw = {}
        for step, offs in ((16, (0, 4, 8, 12)), (48, (0, 4, 8, 16))):
            raw[step] = cloud2_records(pts, step, *offs, seed=step)
            r = d.filtered_cloud2(raw[step], n, step, *offs[:3])
            _same(ref, r, f"urf_process_cloud2, {step}-byte records")
            assert d.last_launch_count() == C1_LAUNCHES
        r, _ = d.filtered_cloud2_packed(raw[48], n, 48, 0, 4, 8, 16, want_labels=True)
        _same(ref, r, "urf_process_cloud2_packed")
        assert d.last_launch_count() == C1_LAUNCHES + PACK_LAUNCHES
        (r,) = d.filtered_batch_records([raw[48]], 48, 0, 4, 8, 16, want_order=True, label8=False)
        _same(ref, r, "urf_process_cloud2_batch, batch = 1")
        assert d.last_launch_count() == C1_LAUNCHES
    finally:
        d.close()


def test_gpu_record_staging_shared_by_single_and_batched_calls(port):
    """A single 64-byte-record scan, then a four-scan batch of 64-byte records (more than the staging buffer urf_create
    sized for one scan: it grows), then a single 22-byte-record scan again."""
    d = api.Detector(max_points=30_000, max_batch=4)
    try:
        prm = make_params(**FULL_ROI)
        d.set_params(prm)
        clouds = [make_scan("C1", 30 + s, order=("column", "ring")[s % 2])[: 28800 - 997 * s] for s in range(4)]
        exp = [port.run(c, prm) for c in clouds]
        r = d.filtered_cloud2(cloud2_records(clouds[0], 64, 40, 12, 28, -1, seed=1), clouds[0].shape[0], 64, 40, 12, 28)
        assert stage_diffs(exp[0], r, clouds[0].shape[0]) == []
        recs = [cloud2_records(c, 64, 40, 12, 28, -1, seed=2 + i) for i, c in enumerate(clouds)]
        for o, r, c in zip(exp, d.filtered_batch_records(recs, 64, 40, 12, 28, -1, want_order=True, label8=False), clouds):
            assert stage_diffs(o, r, c.shape[0]) == []
        r = d.filtered_cloud2(cloud2_records(clouds[3], 22, 0, 4, 8, 12, seed=3), clouds[3].shape[0], 22, 0, 4, 8)
        assert stage_diffs(exp[3], r, clouds[3].shape[0]) == []
    finally:
        d.close()


def test_gpu_single_scan_cloud2_failure_paths():
    d = api.Detector(max_points=30_000, max_batch=1)
    try:
        d.set_params(make_params(**FULL_ROI))
        pts = make_scan("C1", 9)[:17]                                     # fewer than 30 ROI points: nothing published
        raw = cloud2_records(pts, 16, 0, 4, 8, 12)
        ring = np.full(17, 7, np.int32)
        res = UrfResult()
        res.ring = ring.ctypes.data_as(C.POINTER(C.c_int32))
        assert d.lib.urf_process_cloud2(d._ctx, raw.ctypes.data, 17, 16, 0, 4, 8, C.byref(res)) == URF_OK
        assert res.status == URF_TOO_FEW_POINTS and np.all(ring == -1)

        big = np.zeros(40_000 * 16, np.uint8)
        cl = UrfClouds()
        cases = [  # (n, data, point_step, off_z, expected return code)
            (100, big.ctypes.data, 0, 8, URF_ERR_INVALID),
            (100, big.ctypes.data, 11, 8, URF_ERR_INVALID),
            (100, big.ctypes.data, 65, 8, URF_ERR_INVALID),
            (100, big.ctypes.data, 16, 13, URF_ERR_INVALID),                  # field ends past the record
            (40_000, big.ctypes.data, 16, 8, URF_ERR_CAPACITY),
            (100, None, 16, 8, URF_ERR_INVALID),
        ]
        for n, data, step, oz, want in cases:
            res = UrfResult()
            assert d.lib.urf_process_cloud2(d._ctx, data, n, step, 0, 4, oz, C.byref(res)) == want, (n, step, oz)
            assert d.lib.urf_process_cloud2_packed(d._ctx, data, n, step, 0, 4, oz, -1, C.byref(res), C.byref(cl)) == want, (n, step, oz)
    finally:
        d.close()

"""k_points' side outputs, which no label depends on directly: the first ROI input index per fine elevation bin (the
speculation input of the ring registration, debug item 13), the ROI count and the per-sector point counts. Each is
restated in numpy from the per-point outputs (item 0 alpha_v, item 3 sect), which the stage tests hold to the oracle.

A wrong bin entry changes no label: k_assign refutes the speculation and the exact registration repairs the scan, only
slower. So the bins are compared directly, and on the bench's scans the repair must not run at all.

Scan lengths are taken one below, at and one above the 512-point tile. A single scan of up to a few hundred tiles gets
one tile per CTA; a 2^20-point scan gets several tiles per CTA, with range boundaries inside the scan; a batch of more
scans than the device holds k_points CTAs at once gets one CTA per scan, which walks the whole scan."""
import ctypes as C

import numpy as np
import pytest
import torch

from urban_road_filter_b200 import FULL_ROI, UrfResult, api, make_params
from urban_road_filter_b200.synth import SHAPES, make_scan

from util import ScanTab

pytestmark = pytest.mark.gpu

ELEV_BINS = 4096
TILE = 512


def expected_bins(alpha: np.ndarray) -> np.ndarray:
    """Smallest input index per elev_bin(alpha) over the ROI points (alpha >= 0), 0xffffffff for empty bins."""
    roi = np.flatnonzero(alpha >= 0)
    scale = np.float32(ELEV_BINS) / np.float32(180.0)
    bins = np.clip((alpha[roi].astype(np.float32) * scale).astype(np.int64), 0, ELEV_BINS)
    exp = np.full(ELEV_BINS + 1, 0xFFFFFFFF, np.uint32)
    u, first = np.unique(bins, return_index=True)      # roi is ascending: the first occurrence is the smallest index
    exp[u] = roi[first]
    return exp


def check_scan(det, b: int, n: int, n_roi: int):
    alpha = det.debug_fetch(b, 0, np.float32, n)
    sect = det.debug_fetch(b, 3, np.int16, n)
    bins = det.debug_fetch(b, 13, np.uint32, ELEV_BINS + 1)
    exp = expected_bins(alpha)
    bad = np.flatnonzero(bins != exp)
    assert bad.size == 0, f"scan {b}, n={n}: firstidx differs in {bad.size} bins, e.g. {list(zip(bad[:4], bins[bad[:4]], exp[bad[:4]]))}"
    assert n_roi == int((alpha >= 0).sum()), (b, n)
    size = det.lib.urf_debug_sizeof_tab()
    tab = ScanTab.from_buffer_copy(det.debug_fetch(b, 8, np.uint8, size).tobytes())
    cnt = np.bincount(sect[sect >= 0].astype(np.int64), minlength=360)
    assert np.array_equal(np.array(tab.sect_cnt, np.int64), cnt), (b, n)
    if n_roi >= 30:                                     # k_scan_offsets turns the counts into sector starts
        starts = np.concatenate([[0], np.cumsum(cnt)])
        assert np.array_equal(np.array(tab.sect_start, np.int64), starts), (b, n)


def shape_params(shape: str):
    sh = SHAPES[shape]
    return make_params(channels=sh.channels, interval=sh.interval, **FULL_ROI)


@pytest.fixture(scope="module")
def det():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    d = api.Detector(max_points=1 << 20, max_batch=4)
    yield d
    d.close()


@pytest.mark.parametrize("order", ["column", "ring"])
@pytest.mark.parametrize("shape", ["C1", "C2", "C4", "C5"])
def test_gpu_points_bins_and_counts(det, shape, order):
    """Whole scans through the host-buffer path: C5 (2^20 points) spreads several tiles over each CTA."""
    det.set_params(shape_params(shape))
    pts = make_scan(shape, 11, order=order)
    r = det.filtered(pts)
    check_scan(det, 0, pts.shape[0], r.n_roi)


@pytest.mark.parametrize("order", ["column", "ring"])
def test_gpu_points_lengths_at_tile_edges(det, order):
    """Prefixes of a C2 scan around one, two and 256 tiles, and below 30 ROI points."""
    det.set_params(shape_params("C2"))
    pts = make_scan("C2", 12, order=order)
    for n in (1, 29, 30, TILE - 1, TILE, TILE + 1, 2 * TILE - 1, 2 * TILE, 2 * TILE + 1, 256 * TILE - 1, 256 * TILE):
        r = det.filtered(pts[:n].copy())
        check_scan(det, 0, n, r.n_roi)


def device_batch(d, clouds, S, groups):
    B = len(clouds)
    x = torch.zeros((B * S + 64, 4), dtype=torch.float32, device="cuda")
    for b, c in enumerate(clouds):
        x[b * S: b * S + c.shape[0]] = torch.from_numpy(c).cuda()
    lab = torch.empty((B * S + 64,), dtype=torch.int32, device="cuda")
    n = (C.c_int * B)(*[c.shape[0] for c in clouds])
    outs = (UrfResult * B)()
    torch.cuda.synchronize()
    d.set_option(2, groups)
    assert d.lib.urf_enqueue_batch_device(d._ctx, x.data_ptr(), S, n, B, lab.data_ptr()) == 0
    assert d.lib.urf_finish_batch_device(d._ctx, outs) == 0
    return outs


@pytest.mark.parametrize("groups", [1, 2])
def test_gpu_points_ragged_batch_odd_stride(det, groups):
    """Scans of different lengths (empty, below 30 ROI points, around a tile, a whole C4 scan) in one device-resident
    batch whose stride is odd, on one and two stream groups."""
    det.set_params(shape_params("C4"))
    full = make_scan("C4", 13, order="ring")
    S = full.shape[0] + 1
    clouds = [full, make_scan("C4", 14)[:TILE + 1], full[:29], np.zeros((0, 4), np.float32)]
    outs = device_batch(det, clouds, S, groups)
    for b, c in enumerate(clouds):
        assert outs[b].n_in == c.shape[0]
        check_scan(det, b, c.shape[0], outs[b].n_roi)
    det.set_option(2, 2)                                # the library default


def test_gpu_points_batch_wider_than_the_device():
    """2048 scans of up to 1025 points in one launch: more scans than resident k_points CTAs, so each CTA walks its whole
    scan. Lengths one below, at and one above one and two tiles, at an odd stride."""
    S = 2 * TILE + 1
    lengths = [TILE - 1, TILE, TILE + 1, 2 * TILE - 1, 2 * TILE, 2 * TILE + 1, 0, 29]
    base = make_scan("C1", 15)
    clouds = [base[(97 * b) % 20000:][:lengths[b % len(lengths)]].copy() for b in range(2048)]
    d = api.Detector(max_points=S, max_batch=len(clouds))
    try:
        d.set_params(shape_params("C1"))
        outs = device_batch(d, clouds, S, 1)
        for b, c in enumerate(clouds):
            check_scan(d, b, c.shape[0], outs[b].n_roi)
    finally:
        d.close()


def test_gpu_points_no_repairs_on_bench_scans(det):
    """The bench's C2 scans take the speculative ring registration: no exact registration (bit 0), which is also where a
    refuted speculation (internal bit 5) ends up."""
    det.set_params(shape_params("C2"))
    clouds = [make_scan("C2", seed) for seed in range(4)]
    outs = device_batch(det, clouds, clouds[0].shape[0], 2)
    for b, c in enumerate(clouds):
        assert outs[b].status == 0
        assert outs[b].flags & (1 | 32) == 0, (b, outs[b].flags)
        check_scan(det, b, c.shape[0], outs[b].n_roi)

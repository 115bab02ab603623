"""The star search's sector records: k_scatter writes radius, height and input index into three arrays (sr, sz, sidx),
every sort writes (r, z) pairs and, per sorted position, the sector slot or the flagged input index (ssrz, ssl), and the
edge search resolves the index of the point it marks from those. Each case below takes one of the paths that read or
write them, checks through the star sort's work-list counters (debug items 9 and 10) that it was taken, and compares the
labels with the CPU oracle. x-zero and z-zero are off, so every curb label comes from a point the star search marked."""
import ctypes

import numpy as np
import pytest
import torch

from oracle.pyoracle import PortOracle
from urban_road_filter_b200 import FULL_ROI, api, make_params
from urban_road_filter_b200.synth import SHAPES, _detie_radius, make_scan
from util import ScanTab

pytestmark = pytest.mark.gpu

F_TIE_SECTOR = 2
WARP_CAP = 1024                   # kWarpCap: larger refined sectors are sorted by the whole CTA


@pytest.fixture(scope="module")
def det():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    d = api.Detector(max_points=300_000, max_batch=1)
    yield d
    d.close()


@pytest.fixture(scope="module")
def det5():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    d = api.Detector(max_points=1_048_576, max_batch=1)
    yield d
    d.close()


def star_params(shape="C1"):
    sh = SHAPES[shape]
    return make_params(channels=sh.channels, interval=sh.interval, x_zero_method=0, z_zero_method=0, **FULL_ROI)


def run(det, pts, prm, pivot=17):
    """labels of the device and of the oracle, and the work-list counters (nbig, nslow, nrefine) of the device run"""
    det.set_params(prm)
    det.set_option(10, pivot)
    try:
        r = det.filtered(pts)
        nbig, nslow = (int(v) for v in det.debug_fetch(0, 9, np.int32, 2))
        nrefine = int(det.debug_fetch(0, 10, np.int32, 1)[0])
    finally:
        det.set_option(10, 17)
    o = PortOracle().run(pts, prm)
    assert r.status == o.status == 0
    assert r.n_curb > 0, "no curb point: the walk's hit index is not exercised"
    np.testing.assert_array_equal(r.label, o.label)
    assert (r.flags & F_TIE_SECTOR) == (o.flags & F_TIE_SECTOR)
    return r, nbig, nslow, nrefine


def scan_tab(det):
    """the per-scan tables of the detector's last call (debug item 8)"""
    size = det.lib.urf_debug_sizeof_tab()
    assert size == ctypes.sizeof(ScanTab)
    return ScanTab.from_buffer_copy(det.debug_fetch(0, 8, np.uint8, size).tobytes())


def refined_sectors(det, nrefine):
    """(sector, points) of every sector k_star_refine sorted in full"""
    tab = scan_tab(det)
    return [(s, tab.sect_start[s + 1] - tab.sect_start[s]) for s in tab.refine[:nrefine]]


def half_flat(shape, seed):
    """a scan of `shape` whose ground is flat where x < 0: walks there run off their prefix, and their resumed walks find
    the edges the other half finds in its prefix"""
    pts = make_scan(shape, seed).copy()
    pts[pts[:, 0] < 0, 2] = -1.8
    return pts


def tie_behind_the_prefix(pts, prm, pairs=4):
    """Give `pairs` points among the farthest 10 % of every sector of 256 points or more the exact (x, y) of their next
    farther neighbour. The near-first pivot sits at about 56 % of a sector, so these equal radii are met only by a sort of
    the whole sector: the device flags them only in the sectors it refines, the oracle in every sector (the flag is per
    scan, so the two agree when one refined sector holds a pair). Returns the oracle's sector id of every point."""
    sector = PortOracle().run(pts, prm, debug=True).sector
    r = np.hypot(pts[:, 0].astype(np.float64), pts[:, 1])
    for s in np.unique(sector[sector >= 0]):
        idx = np.flatnonzero(sector == s)
        if idx.size < 256:
            continue
        far = idx[np.argsort(r[idx], kind="stable")][-(idx.size // 10):]
        for j in range(pairs):
            pts[far[2 * j], :2] = pts[far[2 * j + 1], :2]
    return sector


def has_equal_xy(pts, sector, s):
    xy = pts[sector == s, :2]
    return np.unique(xy, axis=0).shape[0] < xy.shape[0]


def test_whole_sector_single_warp_sort(det):
    # pivot rank 28 leaves about 90 % of a sector below the pivot: too many for a prefix, so every sector is sorted whole
    # (k_star_sort's STAGED hand-out of whole sectors; sorted_len = the sector, nothing to refine)
    r, nbig, nslow, nrefine = run(det, make_scan("C2", 7), star_params("C2"), pivot=28)
    assert nslow == 0 and nrefine == 0, (nbig, nslow, nrefine)


def test_near_first_prefix_and_refine(det):
    # a flat world has no edge: every walk runs off its prefix and k_star_refine sorts the rest behind it
    pts = make_scan("C2", 31).copy()
    pts[:, 2] = -1.8
    prm = star_params("C2")
    det.set_params(prm)
    det.set_option(10, 17)
    det.filtered(pts)
    nrefine = int(det.debug_fetch(0, 10, np.int32, 1)[0])
    assert nrefine > 0
    # half of it flat: refined sectors whose resumed walk finds an edge, next to sectors whose prefix holds one
    pts = make_scan("C2", 31).copy()
    pts[pts[:, 0] < 0, 2] = -1.8
    r, nbig, nslow, nrefine = run(det, pts, prm)
    assert nrefine > 0 and nslow == 0, (nbig, nslow, nrefine)


def test_warp_refine_with_ties_behind_the_prefix(det):
    # equal radii only behind the near-first pivot: the first sort sees none (nothing on the slow list), the remainder sort
    # of k_star_refine's warp loop meets them and redoes the sector with the exact fallback
    prm = star_params("C2")
    pts = half_flat("C2", 31)
    sector = tie_behind_the_prefix(pts, prm)
    r, nbig, nslow, nrefine = run(det, pts, prm)
    assert nrefine > 0 and nslow == 0 and r.flags & F_TIE_SECTOR, (nbig, nslow, nrefine, r.flags)
    refined = refined_sectors(det, nrefine)
    assert all(n <= WARP_CAP for _, n in refined)
    assert any(has_equal_xy(pts, sector, s) for s, _ in refined)


def test_eight_warp_sort(det5):
    # C5 sectors hold about 2,900 points: k_star_sort_big's near-first network
    r, nbig, nslow, nrefine = run(det5, make_scan("C5", 0), star_params("C5"))
    assert nbig > 0 and nslow == 0, (nbig, nslow, nrefine)


def test_cta_refine(det5):
    # half of a C5 scan flat: refined sectors above kWarpCap points, sorted again by the whole CTA, walk resumed by one warp
    r, nbig, nslow, nrefine = run(det5, half_flat("C5", 3), star_params("C5"))
    assert nrefine > 0 and nslow == 0, (nbig, nslow, nrefine)
    assert any(n > WARP_CAP for _, n in refined_sectors(det5, nrefine))


def test_cta_refine_with_ties_behind_the_prefix(det5):
    # as the warp case above, on C5: the CTA network of k_star_refine meets the ties, the exact fallback redoes the sector
    prm = star_params("C5")
    pts = half_flat("C5", 3)
    sector = tie_behind_the_prefix(pts, prm)
    r, nbig, nslow, nrefine = run(det5, pts, prm)
    assert nrefine > 0 and nslow == 0 and r.flags & F_TIE_SECTOR, (nbig, nslow, nrefine, r.flags)
    refined = refined_sectors(det5, nrefine)
    assert any(n > WARP_CAP and has_equal_xy(pts, sector, s) for s, n in refined)


def test_exact_fallback_on_equal_radii(det):
    # 2 mm range quantisation: neighbouring columns of a flat ring return the same radius, the fallback sorts those
    # sectors by (radius, input index) and stores flagged input indices
    pts = make_scan("C2", 12).copy()
    rng = np.linalg.norm(pts[:, :3], axis=1, keepdims=True)
    q = np.round(rng * 500.0) / 500.0
    pts[:, :3] = (pts[:, :3] / np.maximum(rng, 1e-9) * q).astype(np.float32)
    r, nbig, nslow, nrefine = run(det, pts, star_params("C2"))
    assert nslow > 0 and r.flags & F_TIE_SECTOR, (nbig, nslow, nrefine, r.flags)


def test_sector_beyond_the_networks(det):
    # more than kCtaCap = 8192 points inside one degree (one ring): the exact fallback with its keys in global scratch
    g = np.random.default_rng(5)
    n = 12_000
    az = np.deg2rad(g.uniform(40.05, 40.95, n))
    t = g.uniform(2.0, 40.0, n)
    e = np.deg2rad(-12.0)
    pts = np.zeros((n, 4), np.float32)
    pts[:, 0] = t * np.cos(e) * np.cos(az); pts[:, 1] = t * np.cos(e) * np.sin(az)
    pts[:, 2] = t * np.sin(e) + g.normal(0, 0.02, n) + np.where(t > 20.0, 0.4, 0.0)   # a step: the walk has an edge to find
    _detie_radius(pts, 5)
    prm = make_params(interval=3.0, x_zero_method=0, z_zero_method=0, **FULL_ROI)
    r, nbig, nslow, nrefine = run(det, pts, prm)
    assert nslow > 0, (nbig, nslow, nrefine)

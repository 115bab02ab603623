"""k_star_sort takes a sector of up to 512 points that has no equal radii to its end itself, whether it sorts the
near-first prefix or the whole sector: such a sector must never reach the exact fallback (tab.slowlist), whose
64-bit sort is only there for equal radii and for sectors too large for the register networks."""
import numpy as np
import pytest
import torch

from oracle.pyoracle import PortOracle
from urban_road_filter_b200 import FULL_ROI, api, make_params
from urban_road_filter_b200.synth import SHAPES, make_scan

pytestmark = pytest.mark.gpu

F_TIE_SECTOR = 2


@pytest.fixture(scope="module")
def det():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    d = api.Detector(max_points=300_000, max_batch=1)
    yield d
    d.close()


# option 10 = pivot rank among 32 radius samples: 17 (default) sorts a prefix of about 56 % of a sector; 28 leaves about
# 90 % below the pivot, too many for a prefix sort, so every sector above 128 points is sorted whole after the selection
# has run; 3 sorts a prefix of about 12 %
@pytest.mark.parametrize("pivot", [17, 28, 3])
@pytest.mark.parametrize("shape", ["C2", "C4"])
def test_gpu_star_sort_keeps_tie_free_sectors_off_the_fallback(det, shape, pivot):
    sh = SHAPES[shape]
    pts = make_scan(shape, 7)                      # synthetic scans have no equal radii inside a sector
    prm = make_params(channels=sh.channels, interval=sh.interval, **FULL_ROI)
    det.set_params(prm)
    det.set_option(10, pivot)
    try:
        r = det.filtered(pts)
        nbig, nslow = det.debug_fetch(0, 9, np.int32, 2)
    finally:
        det.set_option(10, 17)
    assert r.flags & F_TIE_SECTOR == 0
    assert nslow == 0, f"{nslow} tie-free sectors went to the exact fallback ({nbig} to the eight-warp sort)"
    np.testing.assert_array_equal(r.label, PortOracle().run(pts, prm).label)

"""Device-resident batches spread over several compute streams, and the channel-wide chunk histograms of the ring
partition: every stream-group count gives the outputs of one stream, the launch count of a step stays the pipeline's, and
every scan matches the CPU oracle."""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle.pyoracle import PortOracle
from urban_road_filter_b200 import FULL_ROI, UrfResult, api, make_params
from urban_road_filter_b200.synth import SHAPES, make_scan, random_cloud

pytestmark = pytest.mark.gpu

# kernels of one pipeline with the default parameters (star-shaped search on, curb_points 5, one CTA per scan for the
# marker search), plus k_sort_rings when the emission order is produced
PIPELINE_KERNELS = 16


@pytest.fixture(scope="module")
def port():
    return PortOracle()


def run_device(d, clouds, S, groups):
    """One urf_enqueue_batch_device_ex call with the emission order: labels [B][S], order [B][S], per-scan results."""
    B = len(clouds)
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
    G = 1 if B < 2 * groups else groups
    assert d.last_launch_count() == G * (PIPELINE_KERNELS + 1), (B, groups)
    res = [(o.status, o.n_in, o.n_roi, o.n_rings, o.n_order, o.n_road, o.n_curb, o.n_vert, o.flags,
            np.ctypeslib.as_array(o.vert).reshape(-1, 4)[: o.n_vert].copy()) for o in outs]
    return lab.cpu().numpy(), order.cpu().numpy(), res


def assert_same(a, b, what):
    la, oa, ra = a
    lb, ob, rb = b
    assert np.array_equal(la, lb), f"{what}: labels"
    for s, (x, y) in enumerate(zip(ra, rb)):
        assert x[:-1] == y[:-1], f"{what}: counts of scan {s}"
        assert np.array_equal(x[-1], y[-1]), f"{what}: vertices of scan {s}"
        assert np.array_equal(oa[s, : x[4]], ob[s, : y[4]]), f"{what}: emission order of scan {s}"


def assert_oracle(port, prm, clouds, got, scans):
    lab, order, res = got
    for b in scans:
        c = clouds[b]
        o = port.run(c, prm)
        r = res[b]
        assert r[0] == o.status, b
        assert np.array_equal(lab[b, : c.shape[0]], o.label), b
        assert np.all(lab[b, c.shape[0]:] == -7), b                  # nothing written beyond the scan
        if o.status != 0:
            continue
        assert (r[3], r[4], r[5], r[6], r[7]) == (o.n_rings, o.n_order, o.n_road, o.n_curb, o.n_vert), b
        assert np.array_equal(order[b, : r[4]], o.order), b
        assert np.array_equal(r[9], o.vert), b


@pytest.mark.parametrize("batch", [2, 3, 5, 17, 128])
def test_gpu_groups_give_the_one_stream_result(port, batch):
    """Uneven splits included: scan lengths differ, and the stride is larger than any scan."""
    S = 7680
    d = api.Detector(max_points=S, max_batch=128)
    try:
        prm = make_params(**FULL_ROI)
        d.set_params(prm)
        clouds = [make_scan("C1", 200 + s, order=("column", "ring")[s % 2], cols=450)[: 7200 - 337 * (s % 5)] for s in range(batch)]
        one = run_device(d, clouds, S, 1)
        for groups in (2, 3, 4):
            assert_same(run_device(d, clouds, S, groups), one, f"{groups} groups")
        assert_oracle(port, prm, clouds, one, range(0, batch, max(1, batch // 6)))
    finally:
        d.close()


@pytest.mark.parametrize("shape,channels", [("C1", 16), ("C2", 64), ("C4", 128), ("C5", 256)])
def test_gpu_channel_wide_histogram_rows(port, shape, channels):
    """The chunk histograms hold `channels` counters per row; the scans register most of the rings a row can hold."""
    sh = SHAPES[shape]
    cols = max(64, 16384 // sh.rings)
    S = sh.rings * cols
    d = api.Detector(max_points=S, max_batch=6)
    try:
        prm = make_params(channels=channels, interval=sh.interval, **FULL_ROI)
        d.set_params(prm)
        clouds = [make_scan(shape, 300 + s, order=("column", "ring")[s % 2], cols=cols)[: S - 97 * s] for s in range(6)]
        one = run_device(d, clouds, S, 1)
        assert max(r[3] for r in one[2]) > channels // 2
        assert_same(run_device(d, clouds, S, 2), one, "2 groups")
        assert_oracle(port, prm, clouds, one, range(6))
    finally:
        d.close()


def test_gpu_repaired_scan_among_regular_scans(port):
    """A scan whose speculated ring registration is refuted (exact registration and re-assignment of the whole scan) in
    the same batch, and the same stream group, as scans that keep the speculation."""
    S = 7680
    d = api.Detector(max_points=S, max_batch=12)
    try:
        prm = make_params(**FULL_ROI)
        d.set_params(prm)
        clouds = [make_scan("C1", 400 + s, cols=450) for s in range(11)]
        clouds.insert(4, random_cloud(5000, 5))
        one = run_device(d, clouds, S, 1)
        assert one[2][4][8] & 1                                      # exact registration ran for the repaired scan
        for groups in (2, 3):
            assert_same(run_device(d, clouds, S, groups), one, f"{groups} groups")
        assert_oracle(port, prm, clouds, one, range(len(clouds)))
    finally:
        d.close()

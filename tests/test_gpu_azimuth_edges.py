"""blindSpots windows, blind quarters and marker bins with azimuths exactly on their bounds, on the device
(tests/azimuth_edges.py, clouds stored in tests/golden/ref/azimuth_edges.npz): every stage against the oracle port
(q1..q4, ring widths, window reach, labels, order, vertices), the threshold rows Tf / Tb k_tab2 leaves against the numpy
restatement bit for bit, a device-resident batch over two stream groups byte for byte against the single scan, and the
scan padded past kMarkSingleMax (k_markers_grid) against k_markers1."""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle.pyoracle import PortOracle
from urban_road_filter_b200 import UrfResult, api

import azimuth_edges as ae
from test_azimuth_edges import edge_cloud, stored_cloud
from util import GpuDebug, stage_diffs

pytestmark = pytest.mark.gpu

NAMES = list(ae.CASES)
MARK_SINGLE_MAX = 300_000          # urf_api.cu kMarkSingleMax


@pytest.fixture(scope="module")
def port():
    return PortOracle()


@pytest.fixture(scope="module")
def det():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    d = api.Detector(max_points=300_032, max_batch=2)
    yield d
    d.close()


def device_tables(det, prm, R):
    """Tf, Tb of scan 0 of the last call (debug items 11, 12), rows 0 .. R-1 as [R, 361]."""
    ch = prm.channels
    return [det.debug_fetch(0, what, np.float32, ae.NDEG * ch).reshape(ae.NDEG, ch).T[:R] for what in (11, 12)]


@pytest.mark.parametrize("name", NAMES)
def test_gpu_azimuth_edges(det, port, name):
    _, prm = edge_cloud(port, name)
    pts = stored_cloud(name)
    n = pts.shape[0]
    o = port.run(pts, prm, debug=True)
    w = ae.check_labels(pts, o, prm)
    det.set_params(prm)

    # graphed single scan: every stage, then the threshold rows
    r = det.filtered(pts)
    assert r.status == 0
    assert stage_diffs(o, GpuDebug(det, r, n), n) == []
    tf, tb = device_tables(det, prm, o.n_rings)
    for got, want, what in ((tf, w.Tf, "Tf"), (tb, w.Tb, "Tb")):
        bad = np.argwhere(got.view(np.uint32) != want.view(np.uint32))
        assert bad.size == 0, f"{what} differs at (ring, degree) {bad[:6].tolist()}: {got[tuple(bad[:6].T)]} vs {want[tuple(bad[:6].T)]}"

    # device-resident batch of two copies over two stream groups
    x = torch.from_numpy(np.concatenate([pts, pts])).cuda()
    lab = torch.full((2 * n,), -7, dtype=torch.int32, device="cuda")
    order = torch.full((2 * n,), -7, dtype=torch.int32, device="cuda")
    outs = (UrfResult * 2)()
    torch.cuda.synchronize()
    det.set_option(2, 2)                                   # one scan per stream group
    assert det.lib.urf_enqueue_batch_device_ex(det._ctx, x.data_ptr(), n, (C.c_int * 2)(n, n), 2, lab.data_ptr(),
                                               order.data_ptr()) == 0
    assert det.lib.urf_finish_batch_device(det._ctx, outs) == 0
    lab, order = lab.cpu().numpy(), order.cpu().numpy()
    for b in range(2):
        rb = api._scan_result(outs[b], lab[b * n: (b + 1) * n].copy(), None, order[b * n: (b + 1) * n])
        assert (rb.status, rb.n_road, rb.n_curb, rb.n_vert, rb.flags) == (r.status, r.n_road, r.n_curb, r.n_vert, r.flags)
        assert rb.label.tobytes() == r.label.tobytes() and rb.order.tobytes() == r.order.tobytes()
        assert rb.vert.tobytes() == r.vert.tobytes()

    # padded past kMarkSingleMax with points outside the ROI: k_markers_grid gives k_markers1's vertices
    pad = np.tile(np.array([[1000.0, 0.0, 0.0, 1.0]], np.float32), (MARK_SINGLE_MAX + 32 - n, 1))
    g = det.filtered(np.concatenate([pts, pad]))
    assert g.vert.tobytes() == r.vert.tobytes(), "k_markers_grid picks other vertices than k_markers1"
    assert g.label[:n].tobytes() == r.label.tobytes() and g.order.tobytes() == r.order.tobytes()

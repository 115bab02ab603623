"""Asynchronous host-buffer batches (urf_enqueue_batch / urf_enqueue_cloud2_batch / urf_finish_batch): two batches in
flight give, byte for byte, what the synchronous urf_process_batch / urf_process_cloud2_batch give on the same scans —
labels (int32 and int8), ring ids, emission order, ring_start, counts, flags and marker vertices, in both tie orders, on
the graph path (small batches) and the chunked path. The calls that would race with batches in flight are refused, and the
streaming queues, whose workers now keep two batches in flight, still match Detector.filtered."""
import ctypes as C
import threading

import numpy as np
import pytest
import torch

from urban_road_filter_b200 import FULL_ROI, api, make_params
from urban_road_filter_b200.ctypes_abi import URF_ERR_CAPACITY, URF_ERR_INVALID, URF_OK
from urban_road_filter_b200.synth import SHAPES, make_scan
from util import cloud2_records

pytestmark = pytest.mark.gpu

RECORDS = {"float4": None, "rec48": (48, (0, 4, 8, 16)), "rec22": (22, (0, 4, 8, 12))}

# (shape, input, int8 labels, ring + order wanted, (batch A, batch B)): 1 and 8 scans take the CUDA-graph path of slot 0,
# 24 scans the chunked pipeline
CASES = [
    ("C1", "float4", False, True, (1, 8)),
    ("C1", "rec22", False, True, (24, 8)),
    ("C2", "rec48", True, True, (8, 24)),
    ("C2", "float4", False, False, (1, 1)),
    ("C4", "rec22", True, False, (24, 1)),
    ("C4", "float4", True, True, (8, 24)),
]


def scans(shape, count, seed, cols_cut, cut0=0):
    """`count` scans of `shape`, each with its own point count (cols_cut columns fewer for every second one)."""
    W = SHAPES[shape].cols
    return [make_scan(shape, seed + k, order=("column", "ring")[k % 2], cols=W - cut0 - cols_cut * (k % 2) - k) for k in range(count)]


class Batch:
    """One batch of scans in one input format, run synchronously or enqueued on a detector."""

    def __init__(self, clouds, kind, label8, want):
        self.clouds, self.kind, self.label8, self.want = clouds, kind, label8, want
        if RECORDS[kind]:
            step, offs = RECORDS[kind]
            self.step, self.offs = step, offs
            self.raw = [cloud2_records(c, step, *offs, seed=k) for k, c in enumerate(clouds)]

    def sync(self, det):
        if not RECORDS[self.kind]:        # urf_process_batch has no int8 output: its int32 labels are the reference
            return det.filtered_batch(self.clouds, want_ring=self.want, want_order=self.want)
        return det.filtered_batch_records(self.raw, self.step, *self.offs, want_order=self.want, label8=self.label8, want_ring=self.want)

    def handle(self, pinned=True):
        """A handle to enqueue, built ahead: page-locked inputs and results, so the enqueued copies really run
        asynchronously (allocating page-locked memory between two enqueues could wait for the first batch)."""
        if not RECORDS[self.kind]:
            return api.BatchHandle.of_clouds(self.clouds, self.want, self.want, self.label8, pinned=pinned)
        return api.BatchHandle.of_records(self.raw, self.step, *self.offs, self.want, self.want, self.label8, pinned=pinned)


def assert_same(got, want, what):
    assert len(got) == len(want), what
    for b, (g, w) in enumerate(zip(got, want)):
        for f in ("status", "n_in", "n_roi", "n_rings", "n_order", "n_road", "n_curb", "n_vert", "flags"):
            assert getattr(g, f) == getattr(w, f), f"{what} scan {b}: {f}"
        for f in ("label", "ring", "order", "ring_start", "vert"):
            a, e = getattr(g, f), getattr(w, f)
            assert (a is None) == (e is None), f"{what} scan {b}: {f}"
            if a is not None:
                assert a.dtype == e.dtype and a.tobytes() == e.tobytes(), f"{what} scan {b}: {f} differs"


def refused(fn, code=URF_ERR_INVALID):
    with pytest.raises(api.UrfError) as e:
        fn()
    assert e.value.code == code


@pytest.mark.parametrize("tie", ["input", "reference"])
@pytest.mark.parametrize("shape,kind,label8,want,sizes", CASES)
def test_gpu_two_batches_in_flight_match_the_synchronous_call(shape, kind, label8, want, sizes, tie):
    assert torch.cuda.is_available()
    A = Batch(scans(shape, sizes[0], 100, 48), kind, label8, want)
    B = Batch(scans(shape, sizes[1], 300, 96, cut0=5), kind, label8, want)
    n = max(c.shape[0] for c in A.clouds + B.clouds)
    assert not {c.shape[0] for c in A.clouds} & {c.shape[0] for c in B.clouds}     # A and B differ in point counts
    det = api.Detector(max_points=n, max_batch=24, params=make_params(**FULL_ROI), tie_order=tie)
    want_a = A.sync(det)
    launches_a = det.last_launch_count()
    want_b = B.sync(det)
    launches_b = det.last_launch_count()

    ha, hb, hc = A.handle(), B.handle(), A.handle()
    stream = torch.cuda.ExternalStream(det.lib.urf_stream(det._ctx))
    det.enqueue(ha)                                                # slot 0
    det.enqueue(hb)                                                # slot 1: its copies overlap A's kernels
    if shape != "C1" and sum(sizes) >= 16:                         # both enqueues returned before the device was done
        assert not stream.query()                                  # (milliseconds of work; C1 batches can finish first)
    refused(lambda: det.enqueue(A.handle(pinned=False)), URF_ERR_CAPACITY)     # a third batch: no slot
    refused(lambda: A.sync(det))
    refused(lambda: det.set_params(det.params))
    refused(lambda: det.set_tie_order(tie))
    refused(lambda: det.set_option(3, 1))
    d_pts = torch.zeros((n, 4), dtype=torch.float32, device="cuda")
    d_lab = torch.zeros(n, dtype=torch.int32, device="cuda")
    cn = (C.c_int * 1)(n)
    assert det.lib.urf_enqueue_batch_device(det._ctx, d_pts.data_ptr(), n, cn, 1, d_lab.data_ptr()) == URF_ERR_INVALID
    assert det.lib.urf_finish_batch_device(det._ctx, None) == URF_ERR_INVALID

    assert det.finish_batch() is ha
    assert det.last_launch_count() == launches_a and det.last_device_ms() > 0
    det.enqueue(hc)                                                # slot 0 again, while B is in flight in slot 1
    assert det.finish_batch() is hb
    assert det.last_launch_count() == launches_b and det.last_device_ms() > 0
    assert det.finish_batch() is hc
    refused(det.finish_batch)                                      # nothing in flight
    assert_same(ha.results, want_a, f"{shape} {kind} A")
    assert_same(hb.results, want_b, f"{shape} {kind} B")
    assert_same(hc.results, want_a, f"{shape} {kind} C")

    # a handle is enqueued again once it is finished; the slot pair keeps alternating; Detector.enqueue_batch builds its
    # own pinned handle
    det.enqueue(hb)
    det.finish_batch()
    det.enqueue(ha)
    hd = B.handle()
    det.enqueue(hd)
    det.finish_batch()
    det.finish_batch()
    for h, w, what in ((hb, want_b, "B again"), (ha, want_a, "A again"), (hd, want_b, "D")):
        assert_same(h.results, w, f"{shape} {kind} {what}")
    if not RECORDS[kind]:
        he = det.enqueue_batch(A.clouds, want_ring=want, want_order=want, label8=label8)
        assert det.finish_batch() is he
        assert_same(he.results, want_a, f"{shape} {kind} enqueue_batch")
    assert_same(A.sync(det), want_a, f"{shape} {kind} A after the asynchronous calls")
    det.set_params(det.params)
    det.close()


def test_gpu_destroy_waits_for_batches_in_flight():
    clouds = scans("C2", 8, 7, 32)
    det = api.Detector(max_points=max(c.shape[0] for c in clouds), max_batch=8, params=make_params(**FULL_ROI))
    want = det.filtered_batch(clouds)
    det.enqueue_batch(clouds)
    det.enqueue_batch(clouds)
    det.close()                                                    # urf_destroy waits; nothing is left writing
    det = api.Detector(max_points=max(c.shape[0] for c in clouds), max_batch=8, params=make_params(**FULL_ROI))
    assert_same(det.filtered_batch(clouds), want, "after a destroy with batches in flight")
    det.close()


def expected(shape, clouds, prm):
    ref = api.Detector(max_points=max(c.shape[0] for c in clouds), max_batch=1, params=prm)
    out = [ref.filtered(c, want_ring=False, want_order=False) for c in clouds]
    ref.close()
    return out


def check_delivered(got, want):
    assert [t for t, _ in got] == list(range(len(want)))
    for t, r in got:
        w = want[t]
        assert (r.status, r.n_roi, r.n_road, r.n_curb, r.n_vert, r.flags) == (w.status, w.n_roi, w.n_road, w.n_curb, w.n_vert, w.flags)
        np.testing.assert_array_equal(r.label.astype(np.int32), w.label)
        np.testing.assert_array_equal(r.vert, w.vert)


@pytest.mark.parametrize("shape,count", [("C1", 40), ("C4", 16)])
@pytest.mark.parametrize("label8", [False, True])
def test_gpu_scan_queue_with_two_batches_in_flight(shape, count, label8):
    """One producer submits by reference, far faster than a batch of two scans runs, so the worker has the next run pending
    while a batch is in flight (the stats show two batches enqueued at once); every result equals Detector.filtered's, in
    order (next for int32 slots, next_batch views for int8 ones)."""
    prm = make_params(**FULL_ROI)
    clouds = scans(shape, count, 500, 64)
    want = expected(shape, clouds, prm)
    n = max(c.shape[0] for c in clouds)
    det = api.Detector(max_points=n, max_batch=2, params=prm)
    q = api.ScanQueue(det, max_points=n, slots=count, max_batch=2, label8=label8)
    got = []

    def consume():
        while len(got) < count:
            if label8:
                got.extend(q.next_batch(8, 60000, copy=True))
            else:
                got.append(q.next(60000))

    cons = threading.Thread(target=consume)
    cons.start()
    for k, c in enumerate(clouds):
        assert q.submit(c, tag=k, timeout_ms=60000, by_reference=True) == URF_OK
    cons.join(300)
    assert not cons.is_alive()
    check_delivered(got, want)
    st = q.stats()
    assert (st["submitted"], st["processed"], st["delivered"], st["dropped"]) == (count, count, count, 0)
    assert st["batches"] > 1 and st["most_in_flight"] == 2
    q.close()
    q.destroy()
    det.close()


@pytest.mark.parametrize("shape,count", [("C1", 30), ("C4", 12)])
def test_gpu_mq_with_two_batches_in_flight(shape, count):
    prm = make_params(**FULL_ROI)
    clouds = scans(shape, count, 700, 64)
    want = expected(shape, clouds, prm)
    n = max(c.shape[0] for c in clouds)
    mq = api.MultiGpuQueue([0, 0], max_points=n, slots_per_device=6, max_batch=2, params=prm)
    got = []
    cons = threading.Thread(target=lambda: [got.append(mq.next(120000)) for _ in range(count)])
    cons.start()
    for k, c in enumerate(clouds):
        assert mq.submit(c, tag=k, timeout_ms=120000, by_reference=bool(k % 2)) == URF_OK
    cons.join(300)
    assert not cons.is_alive() and all(g is not None for g in got)
    check_delivered(got, want)
    mq.set_params(prm)                                             # idle again: every batch was finished
    mq.close()
    mq.destroy()

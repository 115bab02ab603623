"""Batched delivery (urf_queue_next_batch, urf_mq_next_batch) and int8 label slots (URF_QUEUE_LABEL8) of the streaming
ingest: the host-side mechanics run here without a GPU around stand-in batch functions (urf_queue_create_with /
urf_mq_create_with); the real thing is checked against Detector.filtered on the GPU box."""
import ctypes as C
import os
import subprocess
import threading
import time

import numpy as np
import pytest
import torch

from urban_road_filter_b200 import api, make_params
from urban_road_filter_b200.ctypes_abi import (URF_ERR_CLOSED, URF_ERR_INVALID, URF_ERR_TIMEOUT, URF_OK,
                                               URF_QUEUE_DROP_OLDEST, UrfResult)
from util import ROOT


class Stepped:
    """urf_process_batch stand-in: label[i] = (x[i] + 1000 * first y) mod 4 - 1 (the URF_LABEL_* range, so int8 and int32
    slots carry the same values), n_vert = 1 with the scan's first y. `permits` = batches it may still run (None: no
    limit); `fail_on_batch`: that batch returns -3."""

    def __init__(self, permits=None, fail_on_batch=None, delay=None):
        self.sem = threading.Semaphore(permits) if permits is not None else None
        self.fail_on_batch = fail_on_batch
        self.delay = delay
        self.batches = []
        self.threads = []
        self.lock = threading.Lock()

    def allow(self, k=1):
        for _ in range(k):
            self.sem.release()

    def __call__(self, user, xyzi, n, batch, outs):
        if self.sem is not None:
            self.sem.acquire()
        with self.lock:
            me = threading.get_ident()
            if me not in self.threads:
                self.threads.append(me)
            dev = self.threads.index(me)
            self.batches.append(batch)
            nb = len(self.batches) - 1
        if self.delay is not None:
            time.sleep(self.delay(dev))
        if self.fail_on_batch is not None and nb == self.fail_on_batch:
            return -3
        for j in range(batch):
            m = max(n[j], 1)
            pts = np.ctypeslib.as_array(C.cast(xyzi[j], C.POINTER(C.c_float)), shape=(m, 4))
            lab = np.ctypeslib.as_array(outs[j].label, shape=(m,))
            if n[j]:
                lab[: n[j]] = expect_labels(int(pts[0, 1]), n[j])
            outs[j].status = 0
            outs[j].n_in = n[j]
            outs[j].n_vert = 1
            outs[j].vert[0][0] = float(pts[0, 1]) if n[j] else -1.0
        return 0


def scan(k, n=16):
    p = np.zeros((n, 4), np.float32)
    p[:, 0] = np.arange(n)
    p[:, 1] = k
    return p


def expect_labels(k, n=16):
    return ((np.arange(n) + 1000 * k) % 4 - 1).astype(np.int32)


def wait_processed(q, count, timeout=10.0):
    t0 = time.time()
    while q.stats()["processed"] < count:
        assert time.time() - t0 < timeout, q.stats()
        time.sleep(0.002)


def check(got, label8):
    for t, r in got:
        assert r.status == URF_OK and r.n_in == 16 and r.n_vert == 1 and r.vert.shape == (1, 4) and r.vert[0, 0] == t
        assert r.label.dtype == (np.int8 if label8 else np.int32)
        np.testing.assert_array_equal(r.label, expect_labels(t))


@pytest.mark.parametrize("label8", [False, True])
def test_batch_delivers_the_ready_run_in_submission_order(label8):
    fb = Stepped(permits=0)
    q = api.ScanQueue(None, max_points=32, slots=8, max_batch=3, process_fn=fb, label8=label8)
    for k in range(7):
        assert q.submit(scan(k), tag=k, timeout_ms=1000) == URF_OK
    assert q.next_batch(8, timeout_ms=50) == []                   # nothing finished: URF_ERR_TIMEOUT
    fb.allow(10)
    wait_processed(q, 7)
    got = q.next_batch(8, timeout_ms=1000)
    assert [t for t, _ in got] == list(range(7))
    check(got, label8)
    st = q.stats()
    assert (st["submitted"], st["processed"], st["delivered"], st["pending"]) == (7, 7, 7, 0)
    q.destroy()


def test_batch_run_stops_at_the_first_scan_that_is_not_done():
    fb = Stepped(permits=1)
    q = api.ScanQueue(None, max_points=32, slots=6, max_batch=1, process_fn=fb)
    for k in range(4):
        assert q.submit(scan(k), tag=k) == URF_OK
    wait_processed(q, 1)                                          # scan 0 done, scan 1 held inside the batch function
    got = q.next_batch(8, timeout_ms=1000)
    assert [t for t, _ in got] == [0]
    assert q.next_batch(8, timeout_ms=50) == []                   # the oldest live scan is not done: nothing behind it comes out
    fb.allow(3)
    wait_processed(q, 4)
    got = q.next_batch(8, timeout_ms=1000)
    assert [t for t, _ in got] == [1, 2, 3]
    check(got, False)
    q.destroy()


def test_batch_respects_max_results():
    fb = Stepped()
    q = api.ScanQueue(None, max_points=32, slots=8, max_batch=8, process_fn=fb)
    for k in range(7):
        assert q.submit(scan(k), tag=k) == URF_OK
    wait_processed(q, 7)
    assert [t for t, _ in q.next_batch(3)] == [0, 1, 2]
    assert [t for t, _ in q.next_batch(1)] == [3]
    got = q.next_batch(10)
    assert [t for t, _ in got] == [4, 5, 6]
    check(got, False)
    with pytest.raises(ValueError):
        q.next_batch(0)
    assert q.lib.urf_queue_next_batch(q._q, 0, None, None, (UrfResult * 1)(), None, 0) == URF_ERR_INVALID
    q.destroy()


def _next_view(q):
    res, tag, view = UrfResult(), C.c_uint64(), C.c_void_p()
    rc = q.lib.urf_queue_next_view(q._q, C.byref(tag), C.byref(res), C.byref(view), 1000)
    return rc, int(tag.value), res, view


def test_mixing_next_next_view_and_next_batch():
    fb = Stepped()
    q = api.ScanQueue(None, max_points=32, slots=5, max_batch=2, process_fn=fb)     # 3 in flight + up to 2 lent
    order = []
    k = 0
    for step in range(12):
        while k < 30 and q.stats()["pending"] + q.stats()["processed"] - q.stats()["delivered"] < 3:
            assert q.submit(scan(k), tag=k, timeout_ms=5000) == URF_OK
            k += 1
        wait_processed(q, q.stats()["submitted"])
        if step % 3 == 0:
            t, r = q.next(1000)
            np.testing.assert_array_equal(r.label, expect_labels(t))
            order.append(t)
        elif step % 3 == 1:
            rc, t, res, view = _next_view(q)
            assert rc == URF_OK
            np.testing.assert_array_equal(np.ctypeslib.as_array(C.cast(view, C.POINTER(C.c_int32)), shape=(16,)), expect_labels(t))
            order.append(t)
        else:
            got = q.next_batch(2, timeout_ms=1000)
            check(got, False)
            order += [t for t, _ in got]
    q.close()
    while True:
        got = q.next_batch(16, timeout_ms=1000)
        if not got:
            break
        order += [t for t, _ in got]
    assert order == list(range(k))
    q.destroy()


def test_views_stay_valid_until_the_next_call_then_slots_come_back():
    fb = Stepped()
    q = api.ScanQueue(None, max_points=32, slots=4, max_batch=4, process_fn=fb, label8=True)
    for k in range(4):
        assert q.submit(scan(k), tag=k) == URF_OK
    wait_processed(q, 4)
    got = q.next_batch(4)
    assert [t for t, _ in got] == [0, 1, 2, 3]
    assert q.submit(scan(9), tag=9, timeout_ms=100) == URF_ERR_TIMEOUT     # every slot is lent to the consumer
    check(got, True)                                                        # ... so the views still hold scans 0..3
    assert q.next_batch(4, timeout_ms=20) == []                             # the next call gives the slots back
    assert q.submit(scan(4), tag=4, timeout_ms=1000) == URF_OK
    got = q.next_batch(4, timeout_ms=1000, copy=True)
    q.release()                                                             # copies survive the release
    assert q.submit(scan(5), tag=5, timeout_ms=1000) == URF_OK
    assert [t for t, _ in got] == [4]
    check(got, True)
    q.destroy()


@pytest.mark.parametrize("label8", [False, True])
def test_streaming_with_slots_equal_to_max_results_does_not_deadlock(label8):
    fb = Stepped()
    q = api.ScanQueue(None, max_points=32, slots=4, max_batch=2, process_fn=fb, label8=label8)
    K = 60
    got = []

    def consume():
        while len(got) < K:
            out = q.next_batch(4, timeout_ms=10000)
            assert out
            check(out, label8)                   # the views are read before the next call gives the slots back
            got.extend(t for t, _ in out)

    cons = threading.Thread(target=consume)
    cons.start()
    for k in range(K):
        assert q.submit(scan(k), tag=k, timeout_ms=10000) == URF_OK
    cons.join(60)
    assert not cons.is_alive()
    assert got == list(range(K))
    q.destroy()


def test_failed_batch_gives_per_scan_error_codes():
    fb = Stepped(permits=1, fail_on_batch=0)
    q = api.ScanQueue(None, max_points=32, slots=4, max_batch=2, process_fn=fb)
    assert q.submit(scan(0), tag=0) == URF_OK
    wait_processed(q, 1)                                          # batch 0 = scan 0 alone: it failed
    for k in (1, 2):
        assert q.submit(scan(k), tag=k) == URF_OK
    fb.allow(4)
    wait_processed(q, 3)
    got = q.next_batch(8, timeout_ms=1000)
    assert [t for t, _ in got] == [0, 1, 2]
    assert got[0][1].status == -3 and got[0][1].label is None and not got[0][1].published
    check(got[1:], False)
    tags, rcs, views = (C.c_uint64 * 2)(), (C.c_int32 * 2)(), (C.c_void_p * 2)()
    assert q.submit(scan(3), tag=3) == URF_OK
    wait_processed(q, 4)
    assert q.lib.urf_queue_next_batch(q._q, 2, tags, rcs, (UrfResult * 2)(), views, 1000) == 1
    assert (tags[0], rcs[0]) == (3, URF_OK) and views[0]
    q.destroy()


def test_drop_oldest_scans_are_skipped():
    fb = Stepped(permits=1)
    q = api.ScanQueue(None, max_points=32, slots=3, max_batch=1, policy=URF_QUEUE_DROP_OLDEST, process_fn=fb, label8=True)
    assert q.submit(scan(0), tag=0) == URF_OK
    wait_processed(q, 1)                                          # scan 0 done; the worker waits inside the next batch
    for k in (1, 2, 3, 4):
        assert q.submit(scan(k), tag=k, timeout_ms=1000) == URF_OK
    st = q.stats()
    assert st["dropped"] >= 1
    fb.allow(10)
    wait_processed(q, 5 - st["dropped"])
    got = q.next_batch(8, timeout_ms=1000)
    tags = [t for t, _ in got]
    assert tags == sorted(tags) and tags[0] == 0 and tags[-1] == 4 and len(tags) == 5 - st["dropped"]
    check(got, True)
    q.destroy()


def test_timeout_close_and_drain_codes():
    fb = Stepped(permits=0)
    q = api.ScanQueue(None, max_points=32, slots=4, max_batch=4, process_fn=fb)
    outs = (UrfResult * 4)()
    t0 = time.perf_counter()
    assert q.lib.urf_queue_next_batch(q._q, 4, None, None, outs, None, 100) == URF_ERR_TIMEOUT
    assert time.perf_counter() - t0 >= 0.09
    assert q.lib.urf_queue_next_batch(q._q, 4, None, None, outs, None, 0) == URF_ERR_TIMEOUT
    for k in range(3):
        assert q.submit(scan(k), tag=k) == URF_OK
    q.close()
    assert q.submit(scan(9), tag=9, timeout_ms=100) == URF_ERR_CLOSED
    fb.allow(10)
    wait_processed(q, 3)
    got = q.next_batch(8, timeout_ms=1000)                        # what was accepted before the close is still delivered
    assert [t for t, _ in got] == [0, 1, 2]
    assert q.lib.urf_queue_next_batch(q._q, 4, None, None, outs, None, 1000) == URF_ERR_CLOSED
    assert q.next_batch(4, timeout_ms=1000) == []
    q.destroy()


def test_int8_slots_carry_the_int32_values():
    queues = {l8: api.ScanQueue(None, max_points=64, slots=6, max_batch=3, process_fn=Stepped(), label8=l8) for l8 in (False, True)}
    for q in queues.values():
        for k in range(5):
            assert q.submit(scan(k, 40 + k), tag=k) == URF_OK
        wait_processed(q, 5)
    a = queues[False].next_batch(8, copy=True)
    b = queues[True].next_batch(8, copy=True)
    assert [t for t, _ in a] == [t for t, _ in b] == list(range(5))
    for (_, ra), (_, rb) in zip(a, b):
        assert ra.label.dtype == np.int32 and rb.label.dtype == np.int8 and ra.n_in == rb.n_in
        np.testing.assert_array_equal(ra.label, rb.label.astype(np.int32))
        assert set(np.unique(ra.label)) <= {-1, 0, 1, 2}
    q8 = queues[True]
    assert q8.submit(scan(7, 20), tag=7) == URF_OK
    wait_processed(q8, 6)
    assert _next_view(q8)[0] == URF_ERR_INVALID                   # no int32 view of an int8 slot, and nothing is consumed
    t, r = q8.next(1000)                                          # urf_queue_next widens into the caller's int32 buffer
    assert t == 7 and r.label.dtype == np.int32
    np.testing.assert_array_equal(r.label, expect_labels(7, 20))
    for q in queues.values():
        q.destroy()


@pytest.mark.parametrize("label8", [False, True])
def test_mq_batch_keeps_the_global_order_across_uneven_devices(label8):
    """Three stand-in devices, the second one 3 ms per batch, the third 6 ms: a batch call takes finished scans from
    several devices while the global order holds, and a run stops at a slow device's unfinished scan."""
    fb = Stepped(delay=lambda dev: 0.003 * (dev % 3))
    mq = api.MultiGpuQueue([0, 1, 2], max_points=32, slots_per_device=3, max_batch=2, process_fn=fb, label8=label8)
    K = 60
    got, runs = [], []

    def consume():
        while len(got) < K:
            out = mq.next_batch(8, timeout_ms=20000)
            assert out
            check(out, label8)
            runs.append(len(out))
            got.extend(t for t, _ in out)

    cons = threading.Thread(target=consume)
    cons.start()
    for k in range(K):
        assert mq.submit(scan(k), tag=k, timeout_ms=20000, by_reference=bool(k & 1)) == URF_OK
    cons.join(60)
    assert not cons.is_alive()
    assert got == list(range(K))
    assert max(runs) > 1 and max(runs) <= 8
    st = mq.stats()
    assert sum(st["delivered"]) == K and min(st["delivered"]) > 0 and st["pending"] == 0
    mq.close()
    assert mq.next_batch(4, timeout_ms=1000) == []
    mq.destroy()


def test_mq_mixing_next_and_next_batch_and_int8_views():
    fb = Stepped()
    mq = api.MultiGpuQueue([0, 1], max_points=32, slots_per_device=3, max_batch=2, process_fn=fb, label8=True)
    for k in range(5):
        assert mq.submit(scan(k), tag=k, timeout_ms=5000) == URF_OK
    res, tag, view = UrfResult(), C.c_uint64(), C.c_void_p()
    assert mq.lib.urf_mq_next_view(mq._m, C.byref(tag), C.byref(res), C.byref(view), 1000) == URF_ERR_INVALID
    t, r = mq.next(5000)                                          # scan 0 was not consumed by the refused view call
    assert t == 0 and r.label.dtype == np.int32
    np.testing.assert_array_equal(r.label, expect_labels(0))
    out = []
    while len(out) < 4:
        b = mq.next_batch(2, timeout_ms=5000)
        check(b, True)
        out += [t for t, _ in b]
    assert out == [1, 2, 3, 4]
    for k in range(5, 11):                                        # slots lent by the last batch come back on the next call
        assert mq.submit(scan(k), tag=k, timeout_ms=5000) == URF_OK
        t, r = mq.next(5000)
        assert t == k
    mq.close()
    mq.destroy()


@pytest.mark.parametrize("args", [("queue", "4", "1500", "6", "4", "0", "6", "1"), ("queue", "4", "1500", "6", "4", "0", "6", "0"),
                                  ("queue", "3", "1500", "4", "3", "1", "4", "1"), ("queue", "2", "1000", "4", "2", "0", "4", "0"),
                                  ("mq", "4", "2", "800", "8", "1"), ("mq", "3", "1", "800", "6", "0"), ("mq", "8", "3", "400", "16", "1")])
def test_batch_thread_sanitizer_stress(args):
    """urf_queue.cpp + urf_mq.cpp built with -fsanitize=thread (tests/kat/queue_batch_stress.cpp). "queue": producers x
    scans x slots x max_batch x policy x max_results x label8, a consumer mixing next_batch with next / next_view and
    failing batches; "mq": devices (of uneven speed) x producers x scans x max_results x label8 through urf_mq_next_batch
    mixed with urf_mq_next. The binary checks that every scan is delivered once with its labels in per-producer order,
    TSAN that there is no data race."""
    out = subprocess.run([os.path.join(ROOT, "build", "queue_batch_stress"), *args], capture_output=True, text=True, timeout=600)
    print(out.stdout, out.stderr[-3000:])
    assert out.returncode == 0 and out.stdout.strip().endswith("OK") and "ThreadSanitizer" not in out.stderr


def _gpu_scans():
    from urban_road_filter_b200.synth import make_scan
    return {k: make_scan(("C1", "C4")[k % 2], 300 + k) for k in range(10)}


def _reference(clouds, prm):
    n = max(c.shape[0] for c in clouds.values())
    det = api.Detector(max_points=n, max_batch=1, params=prm)
    want = {t: det.filtered(c, want_ring=False, want_order=False) for t, c in clouds.items()}
    det.close()
    return n, want


def _same(r, w):
    assert (r.status, r.n_in, r.n_roi, r.n_rings, r.n_order, r.n_road, r.n_curb, r.n_vert, r.flags) == \
           (w.status, w.n_in, w.n_roi, w.n_rings, w.n_order, w.n_road, w.n_curb, w.n_vert, w.flags)
    assert r.label.tobytes() == w.label.astype(r.label.dtype).tobytes() and np.array_equal(r.label.astype(np.int32), w.label)
    assert r.vert.tobytes() == w.vert.tobytes()


@pytest.mark.gpu
def test_gpu_int8_queue_batches_equal_the_detector():
    """C1 and C4 scans through an int8 ScanQueue around a real context, collected with next_batch (and one with next): labels,
    counts and vertices equal Detector.filtered's for the same scans."""
    from urban_road_filter_b200 import FULL_ROI
    assert torch.cuda.is_available()
    prm = make_params(**FULL_ROI, channels=128)
    clouds = _gpu_scans()
    n, want = _reference(clouds, prm)
    det = api.Detector(max_points=n, max_batch=4, params=prm)
    q = api.ScanQueue(det, max_points=n, slots=6, max_batch=4, label8=True)
    got = []

    def consume():
        t, r = q.next(60000)                                      # int8 slot widened into int32
        _same(r, want[t])
        got.append(t)
        while len(got) < len(clouds):
            out = q.next_batch(4, timeout_ms=60000)
            assert out
            for t, r in out:
                assert r.label.dtype == np.int8
                _same(r, want[t])
                got.append(t)

    cons = threading.Thread(target=consume)
    cons.start()
    for t, c in clouds.items():
        assert q.submit(c, tag=t, timeout_ms=60000) == URF_OK
    cons.join(300)
    assert not cons.is_alive() and got == sorted(clouds)
    q.close()
    q.destroy()
    det.close()


@pytest.mark.gpu
@pytest.mark.parametrize("label8", [True, False])
def test_gpu_mq_next_batch_equals_the_detector_on_every_gpu(label8):
    """MultiGpuQueue over every visible GPU (one device when only one is visible), collected with next_batch: labels, counts
    and vertices equal Detector.filtered's, in submission order."""
    from urban_road_filter_b200 import FULL_ROI
    assert torch.cuda.is_available()
    prm = make_params(**FULL_ROI, channels=128)
    clouds = _gpu_scans()
    n, want = _reference(clouds, prm)
    mq = api.MultiGpuQueue(list(range(torch.cuda.device_count())), max_points=n, slots_per_device=4, max_batch=4, params=prm,
                           label8=label8)
    got = []

    def consume():
        while len(got) < len(clouds):
            out = mq.next_batch(8, timeout_ms=60000)
            assert out
            for t, r in out:
                assert r.label.dtype == (np.int8 if label8 else np.int32)
                _same(r, want[t])
                got.append(t)

    cons = threading.Thread(target=consume)
    cons.start()
    for t, c in clouds.items():
        assert mq.submit(c, tag=t, timeout_ms=60000, by_reference=bool(t % 3 == 0)) == URF_OK
    cons.join(300)
    assert not cons.is_alive() and got == sorted(clouds)
    mq.close()
    mq.destroy()

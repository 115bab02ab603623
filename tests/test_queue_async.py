"""The streaming queue's two-batches-in-flight worker (the schedule a urf_queue runs on a real context: enqueue what is
pending, enqueue the next pending run while a batch slot is free, finish the oldest) around an asynchronous stand-in
(urf_queue_create_with_async), without a GPU: delivery order, runs cut at a scan that is not finished, DROP_OLDEST once a
scan is enqueued, a batch that fails while another is in flight, close / drain / timeout, and the ThreadSanitizer stress."""
import collections
import ctypes as C
import os
import subprocess
import threading

import numpy as np
import pytest

from urban_road_filter_b200 import api
from urban_road_filter_b200.ctypes_abi import URF_ERR_CLOSED, URF_ERR_INVALID, URF_OK, URF_QUEUE_DROP_OLDEST
from util import ROOT

from test_queue import expect_labels, scan


class FakeDevice:
    """urf_enqueue_batch / urf_finish_batch stand-in. enqueue keeps the batch's pointers (valid until its finish, as for the
    real pair); finish computes the oldest batch — label[i] = int(x[i]) + 1000 * (scan's first y) — and returns its status.
    `enq_gate` holds enqueues back, `fin_permits` counts the finishes allowed to proceed (None: all)."""

    def __init__(self, fail_enqueue=(), fail_finish=(), fin_permits=None):
        self.enq_gate = threading.Event()
        self.enq_gate.set()
        self.entered = threading.Semaphore(0)        # released when an enqueue starts
        self.fin_permits = None if fin_permits is None else threading.Semaphore(fin_permits)
        self.flight = collections.deque()
        self.events = []                             # ("enq" | "fin", batch index, batch size)
        self.most = 0
        self.count = 0
        self.fail_enqueue, self.fail_finish = set(fail_enqueue), set(fail_finish)

    def allow(self, k=1):
        for _ in range(k):
            self.fin_permits.release()

    def enqueue(self, user, xyzi, n, batch, outs):
        self.entered.release()
        self.enq_gate.wait()
        i = self.count
        self.count += 1
        self.events.append(("enq", i, batch))
        if i in self.fail_enqueue:
            return -3
        self.flight.append((i, xyzi, n, batch, outs))
        self.most = max(self.most, len(self.flight))
        return 0

    def finish(self):
        if self.fin_permits is not None:
            self.fin_permits.acquire()
        i, xyzi, n, batch, outs = self.flight.popleft()
        self.events.append(("fin", i, batch))
        for j in range(batch):
            pts = np.ctypeslib.as_array(C.cast(xyzi[j], C.POINTER(C.c_float)), shape=(n[j], 4)) if n[j] else np.zeros((0, 4), np.float32)
            lab = np.ctypeslib.as_array(outs[j].label, shape=(max(n[j], 1),))
            if n[j]:
                lab[: n[j]] = pts[:, 0].astype(np.int32) + 1000 * int(pts[0, 1])
            outs[j].status = 0
            outs[j].n_in = n[j]
            outs[j].n_roi = n[j]
        return -3 if i in self.fail_finish else 0


def make_queue(fd, **kw):
    return api.ScanQueue(None, enqueue_fn=fd.enqueue, finish_fn=fd.finish, **kw)


def hold_first_enqueue(fd, q, tags):
    """Submits tags[0], waits until the worker is inside its enqueue (held at the gate), then submits the rest, which stay
    pending until open() lets the worker go on."""
    fd.enq_gate.clear()
    assert q.submit(scan(tags[0]), tag=tags[0], timeout_ms=5000) == URF_OK
    assert fd.entered.acquire(timeout=5)
    for t in tags[1:]:
        assert q.submit(scan(t), tag=t, timeout_ms=5000) == URF_OK


@pytest.mark.parametrize("label8", [False, True])
def test_async_queue_orders_and_keeps_two_batches_in_flight(label8):
    def want(t, n=16):                               # int8 slots keep the low byte of the stand-in's int32 labels
        return expect_labels(t, n).astype(np.int8).astype(np.int32) if label8 else expect_labels(t, n)

    fd = FakeDevice()
    q = make_queue(fd, max_points=64, slots=4, max_batch=2, label8=label8)
    hold_first_enqueue(fd, q, [0, 1, 2, 3])
    fd.enq_gate.set()
    got = [q.next(5000) for _ in range(4)]
    assert [t for t, _ in got] == [0, 1, 2, 3]
    for t, r in got:
        np.testing.assert_array_equal(r.label, want(t))
    # the next run is enqueued before the oldest batch is finished
    assert fd.events == [("enq", 0, 1), ("enq", 1, 2), ("fin", 0, 1), ("enq", 2, 1), ("fin", 1, 2), ("fin", 2, 1)]
    assert fd.most == 2 and q.stats()["most_in_flight"] == 2
    # a longer stream with a consumer thread: everything once, in order, never more than two batches enqueued
    got = []
    cons = threading.Thread(target=lambda: [got.append(q.next(5000)) for _ in range(60)])
    cons.start()
    for k in range(10, 70):
        assert q.submit(scan(k, 8 + k % 9), tag=k, timeout_ms=5000) == URF_OK
    cons.join(30)
    assert not cons.is_alive()
    assert [t for t, _ in got] == list(range(10, 70))
    for t, r in got:
        np.testing.assert_array_equal(r.label, want(t, 8 + t % 9))
    assert fd.most == 2 and not fd.flight
    st = q.stats()
    assert (st["submitted"], st["processed"], st["delivered"], st["dropped"], st["pending"]) == (64, 64, 64, 0, 0)
    q.destroy()


def test_async_queue_cuts_runs_at_a_scan_that_is_not_finished():
    fd = FakeDevice(fin_permits=0)
    q = make_queue(fd, max_points=64, slots=6, max_batch=2)
    hold_first_enqueue(fd, q, [0, 1, 2, 3])
    fd.enq_gate.set()
    assert q.next_batch(8, timeout_ms=100) == []                  # two batches enqueued, none finished
    fd.allow()
    assert [t for t, _ in q.next_batch(8, timeout_ms=5000, copy=True)] == [0]   # 1 and 2 are still in flight
    fd.allow()
    out = q.next_batch(8, timeout_ms=5000, copy=True)
    assert [t for t, _ in out] == [1, 2]
    for t, r in out:
        np.testing.assert_array_equal(r.label, expect_labels(t))
    fd.allow()
    assert [t for t, _ in q.next_batch(8, timeout_ms=5000)] == [3]
    q.destroy()


def test_async_queue_drop_oldest_spares_enqueued_scans():
    fd = FakeDevice(fin_permits=0)
    q = make_queue(fd, max_points=32, slots=3, max_batch=1, policy=URF_QUEUE_DROP_OLDEST)
    hold_first_enqueue(fd, q, [0, 1, 2])                          # 0 enqueueing, 1 and 2 pending: every slot taken
    assert q.submit(scan(3), tag=3, timeout_ms=1000) == URF_OK    # replaces 1
    assert q.stats()["dropped"] == 1
    fd.enq_gate.set()
    assert fd.entered.acquire(timeout=5)                          # 2 is being enqueued: it counts as started
    assert q.submit(scan(4), tag=4, timeout_ms=1000) == URF_OK    # replaces 3, the only scan still pending
    assert q.stats()["dropped"] == 2
    fd.allow(10)
    out = [q.next(5000) for _ in range(3)]
    assert [t for t, _ in out] == [0, 2, 4]
    for t, r in out:
        np.testing.assert_array_equal(r.label, expect_labels(t))
    st = q.stats()
    assert (st["submitted"], st["processed"], st["delivered"], st["dropped"]) == (5, 3, 3, 2)
    q.destroy()


def test_async_queue_reports_batches_that_fail_while_another_is_in_flight():
    # batch 0 ([0]) fails at its finish, batch 1 ([1, 2]) is refused at its enqueue while batch 0 is in flight
    fd = FakeDevice(fail_enqueue={1}, fail_finish={0})
    q = make_queue(fd, max_points=64, slots=6, max_batch=2)
    hold_first_enqueue(fd, q, [0, 1, 2, 3])
    fd.enq_gate.set()
    got = []
    while len(got) < 4:
        got += q.next_batch(8, timeout_ms=5000, copy=True)
    assert [t for t, _ in got] == [0, 1, 2, 3]
    assert [r.status for _, r in got[:3]] == [-3, -3, -3] and all(r.label is None for _, r in got[:3])
    assert got[3][1].status == URF_OK
    np.testing.assert_array_equal(got[3][1].label, expect_labels(3))
    assert fd.events == [("enq", 0, 1), ("enq", 1, 2), ("enq", 2, 1), ("fin", 0, 1), ("fin", 2, 1)]
    st = q.stats()
    assert (st["submitted"], st["processed"], st["delivered"]) == (4, 4, 4)
    assert q.submit(scan(5), tag=5, timeout_ms=1000) == URF_OK     # the queue keeps going
    t, r = q.next(5000)
    assert t == 5
    np.testing.assert_array_equal(r.label, expect_labels(5))
    q.destroy()


def test_async_queue_close_drains_and_times_out():
    fd = FakeDevice(fin_permits=0)
    q = make_queue(fd, max_points=32, slots=4, max_batch=2)
    for k in range(3):
        assert q.submit(scan(k), tag=k, timeout_ms=1000) == URF_OK
    q.close()
    assert q.submit(scan(9), tag=9, timeout_ms=100) == URF_ERR_CLOSED
    assert q.next(50) is None                                      # nothing finished yet: URF_ERR_TIMEOUT
    fd.allow(10)
    assert [q.next(5000)[0] for _ in range(3)] == [0, 1, 2]        # accepted before the close: still delivered
    assert q.next(1000) is None                                    # drained: URF_ERR_CLOSED
    assert fd.most <= 2 and not fd.flight
    q.destroy()


def test_async_entry_points_refuse_without_a_context():
    lib = api.load_library()
    assert lib.urf_finish_batch(None) == URF_ERR_INVALID
    res = (api.UrfResult * 1)()
    assert lib.urf_enqueue_batch(None, None, None, 1, res, None) == URF_ERR_INVALID
    q = C.c_void_p()
    fd = FakeDevice()
    enq = api.QUEUE_PROCESS_FN(fd.enqueue)
    assert lib.urf_queue_create_with_async(C.byref(q), enq, C.cast(None, api.QUEUE_FINISH_FN), None, 8, 2, 1, 0) == URF_ERR_INVALID
    assert not q.value


@pytest.mark.parametrize("args", [("4", "1500", "6", "4", "0"), ("8", "600", "3", "2", "0"), ("4", "1500", "4", "3", "1"),
                                  ("3", "1200", "5", "2", "2"), ("1", "3000", "2", "1", "0")])
def test_async_queue_thread_sanitizer_stress(args):
    """urf_queue.cpp built with -fsanitize=thread around a stand-in device thread (tests/kat/queue_async_stress.cpp):
    producers x scans x slots x max_batch x policy bits (1 DROP_OLDEST, 2 int8 labels); some batches fail at enqueue and
    some at finish. The binary checks delivery, payloads, per-producer order and at most (and at some point exactly) two
    batches enqueued; TSAN that there is no data race."""
    out = subprocess.run([os.path.join(ROOT, "build", "queue_async_stress"), *args], capture_output=True, text=True, timeout=600)
    print(out.stdout, out.stderr[-3000:])
    assert out.returncode == 0 and out.stdout.strip().endswith("OK") and "ThreadSanitizer" not in out.stderr

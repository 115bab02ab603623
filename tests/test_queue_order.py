"""Emission order through the streaming queues (URF_QUEUE_ORDER), without a GPU: the queues run around stand-in batch
functions that write, for each scan, an order and ring offsets derived from the scan (a seeded permutation and cuts), and
every delivery path must hand back exactly what was written for that tag: urf_queue_next into the caller's buffers,
urf_queue_next_view, urf_queue_next_batch views (valid until the next call, and their slots given back after it), the
two-batches-in-flight worker, DROP_OLDEST, int8 label slots, a parameter update in mid-stream, a failed batch, and urf_mq
over three stand-in devices. Without the bit the stand-in is handed NULL and delivery returns NULL. The ThreadSanitizer
program tests/kat/queue_order_stress.cpp runs several producers, random updates and one batched consumer."""
import ctypes as C
import os
import subprocess
import threading
import time

import numpy as np
import pytest

from urban_road_filter_b200 import api, make_params
from urban_road_filter_b200.ctypes_abi import (URF_ERR_INVALID, URF_ERR_TIMEOUT, URF_MAX_CHANNELS, URF_OK, URF_QUEUE_BLOCK,
                                               URF_QUEUE_DROP_OLDEST, URF_QUEUE_LABEL8, URF_QUEUE_ORDER, QUEUE_FINISH_FN,
                                               QUEUE_PROCESS_FN, UrfResult)
from util import ROOT

from test_queue import expect_labels, scan
from test_queue_async import FakeDevice


def expect_order(k, n=16, gen=0):
    """The order and ring_start the stand-ins write for scan k (first y == k) of n points run with generation gen: a
    seeded permutation of all but k % 3 points, cut into 1 + k % 13 rings."""
    rng = np.random.default_rng(1000 * gen + k)
    n_order = max(n - k % 3, 0)
    order = rng.permutation(n)[:n_order].astype(np.int32)
    cuts = np.sort(rng.integers(0, n_order + 1, k % 13))
    return order, np.concatenate([[0], cuts, [n_order]]).astype(np.int32)


def write_scan(xyzi, n, j, out, gen=0):
    """What every stand-in here does for scan j: labels as test_queue.FakeBatch, and the order and ring_start of
    expect_order when the queue handed it buffers for them. Returns whether it was handed them."""
    pts = np.ctypeslib.as_array(C.cast(xyzi[j], C.POINTER(C.c_float)), shape=(n[j], 4)) if n[j] else np.zeros((0, 4), np.float32)
    k = int(pts[0, 1]) if n[j] else 0
    if n[j]:
        np.ctypeslib.as_array(out.label, shape=(n[j],))[:] = pts[:, 0].astype(np.int32) + 1000 * k
    out.status, out.n_in, out.n_roi, out.n_vert = 0, n[j], n[j], 0
    given = bool(out.order) and bool(out.ring_start)
    if given:
        order, rs = expect_order(k, n[j], gen)
        out.n_order, out.n_rings = order.size, rs.size - 1
        if order.size:
            np.ctypeslib.as_array(out.order, shape=(order.size,))[:] = order
        np.ctypeslib.as_array(out.ring_start, shape=(rs.size,))[:] = rs
    assert bool(out.order) == bool(out.ring_start)
    return given


class OrderBatch:
    """Synchronous stand-in (urf_process_batch's signature); records per batch whether it got order buffers. `gate` holds
    it back, `fail_on_batch` fails that batch (0-based) with -3. A batch's generation is the last one the parameter hook
    named on the calling worker thread (each device of an mq has its own)."""

    def __init__(self, fail_on_batch=None):
        self.gate = threading.Event()
        self.gate.set()
        self.started = threading.Semaphore(0)
        self.given = []
        self.fail_on_batch = fail_on_batch
        self.gen = {}                                    # worker thread -> generation
        self.lock = threading.Lock()

    def hook(self, user, prm, gen):
        self.gen[threading.get_ident()] = gen
        return URF_OK

    def __call__(self, user, xyzi, n, batch, outs):
        self.started.release()
        self.gate.wait()
        with self.lock:
            i = len(self.given)
            self.given.append(None)
        if i == self.fail_on_batch:
            return -3
        gen = self.gen.get(threading.get_ident(), 0)
        self.given[i] = all([write_scan(xyzi, n, j, outs[j], gen) for j in range(batch)])
        return 0


class OrderDevice(FakeDevice):
    """FakeDevice whose finish also writes the order and ring_start of its oldest batch."""

    def finish(self):
        _, xyzi, n, batch, outs = self.flight[0]
        rc = super().finish()
        for j in range(batch):
            assert write_scan(xyzi, n, j, outs[j])
        return rc


def check(tag, r, n=16, gen=0, label8=False):
    want = expect_labels(tag, n)
    np.testing.assert_array_equal(r.label, want.astype(np.int8) if label8 else want)
    order, rs = expect_order(tag, n, gen)
    assert r.order is not None and r.ring_start is not None, tag
    assert r.n_order == order.size and r.n_rings == rs.size - 1, tag
    np.testing.assert_array_equal(r.order, order)
    np.testing.assert_array_equal(r.ring_start, rs)
    assert r.order.dtype == np.int32 and r.ring_start.dtype == np.int32


def drain(q, count, max_results=8):
    got = []
    while len(got) < count:
        out = q.next_batch(max_results, timeout_ms=5000, copy=True)
        assert out, "timed out"
        got += out
    return got


@pytest.mark.parametrize("label8", [False, True])
def test_next_fills_the_callers_buffers(label8):
    fb = OrderBatch()
    q = api.ScanQueue(None, max_points=32, slots=6, max_batch=4, process_fn=fb, label8=label8, order=True)
    got = []
    cons = threading.Thread(target=lambda: [got.append(q.next(5000)) for _ in range(30)])
    cons.start()
    for k in range(30):
        assert q.submit(scan(k, 8 + k % 9), tag=k, timeout_ms=5000) == URF_OK
    cons.join(20)
    assert not cons.is_alive() and all(fb.given)
    assert [t for t, _ in got] == list(range(30))
    for t, r in got:
        check(t, r, 8 + t % 9, label8=label8)            # next widens the low byte an int8 slot keeps
    q.destroy()


def test_next_keeps_the_callers_pointers_and_copies_only_what_exists():
    """urf_queue_next: out->label / order / ring_start are the caller's on return; n_order and n_rings + 1 entries are
    written, nothing beyond them."""
    lib = api.load_library()
    q = api.ScanQueue(None, max_points=32, slots=4, max_batch=2, process_fn=OrderBatch(), order=True)
    assert q.submit(scan(4, 20), tag=4, timeout_ms=1000) == URF_OK
    lab, order, rs = np.full(32, -5, np.int32), np.full(32, -5, np.int32), np.full(URF_MAX_CHANNELS + 1, -5, np.int32)
    res = UrfResult()
    ptrs = [a.ctypes.data_as(C.POINTER(C.c_int32)) for a in (lab, order, rs)]
    res.label, res.order, res.ring_start = ptrs
    tag = C.c_uint64()
    assert lib.urf_queue_next(q._q, C.byref(tag), C.byref(res), 5000) == URF_OK
    for f, a in zip(("label", "order", "ring_start"), (lab, order, rs)):
        assert C.addressof(getattr(res, f).contents) == a.ctypes.data, f
    want_order, want_rs = expect_order(4, 20)
    np.testing.assert_array_equal(lab[:20], expect_labels(4, 20))
    np.testing.assert_array_equal(order[: want_order.size], want_order)
    np.testing.assert_array_equal(rs[: want_rs.size], want_rs)
    assert (order[want_order.size:] == -5).all() and (rs[want_rs.size:] == -5).all() and (lab[20:] == -5).all()
    q.destroy()


def test_next_view_points_into_the_slot():
    lib = api.load_library()
    q = api.ScanQueue(None, max_points=32, slots=2, max_batch=1, process_fn=OrderBatch(), order=True)
    for k in (7, 8):
        assert q.submit(scan(k), tag=k, timeout_ms=1000) == URF_OK
    res, tag, view = UrfResult(), C.c_uint64(), C.c_void_p()
    assert lib.urf_queue_next_view(q._q, C.byref(tag), C.byref(res), C.byref(view), 5000) == URF_OK
    r = api._scan_result(res, np.ctypeslib.as_array(C.cast(view, C.POINTER(C.c_int32)), shape=(res.n_in,)),
                         order=np.ctypeslib.as_array(res.order, shape=(32,)), ring_start=np.ctypeslib.as_array(res.ring_start, shape=(URF_MAX_CHANNELS + 1,)))
    check(7, r)
    assert q.submit(scan(9), tag=9, timeout_ms=100) == URF_ERR_TIMEOUT      # slot 7 is lent, slot 8 waits to be collected
    assert lib.urf_queue_next_view(q._q, C.byref(tag), C.byref(res), C.byref(view), 5000) == URF_OK
    assert tag.value == 8
    assert q.submit(scan(9), tag=9, timeout_ms=1000) == URF_OK              # the first view's slot came back
    q.destroy()


def test_next_batch_views_stay_until_the_next_call_then_their_slots_come_back():
    fb = OrderBatch()
    q = api.ScanQueue(None, max_points=32, slots=4, max_batch=4, process_fn=fb, order=True)
    fb.gate.clear()
    for k in range(4):
        assert q.submit(scan(k), tag=k, timeout_ms=1000) == URF_OK
    fb.gate.set()
    deadline = time.time() + 5
    while q.stats()["processed"] < 4 and time.time() < deadline:
        time.sleep(0.01)
    got = q.next_batch(4, timeout_ms=5000)               # one call lends all four
    assert [t for t, _ in got] == [0, 1, 2, 3]
    assert q.submit(scan(10), tag=10, timeout_ms=100) == URF_ERR_TIMEOUT    # every slot is lent
    for t, r in got:
        check(t, r)
        assert not r.order.flags.owndata and not r.ring_start.flags.owndata   # views of the lent slots
    q.release()                                                             # the next call would give them back too
    for k in range(10, 14):
        assert q.submit(scan(k), tag=k, timeout_ms=1000) == URF_OK
    for t, r in drain(q, 4):
        check(t, r)
    q.destroy()


@pytest.mark.parametrize("label8", [False, True])
def test_two_batches_in_flight(label8):
    fd = OrderDevice()
    q = api.ScanQueue(None, enqueue_fn=fd.enqueue, finish_fn=fd.finish, max_points=64, slots=6, max_batch=3, label8=label8, order=True)
    got = []
    cons = threading.Thread(target=lambda: got.extend(drain(q, 60)))
    cons.start()
    for k in range(60):
        assert q.submit(scan(k, 8 + k % 9), tag=k, timeout_ms=5000, by_reference=bool(k % 2)) == URF_OK
    cons.join(30)
    assert not cons.is_alive()
    assert [t for t, _ in got] == list(range(60))
    for t, r in got:
        check(t, r, 8 + t % 9, label8=label8)
    assert fd.most <= 2
    q.destroy()


def test_drop_oldest():
    fb = OrderBatch()
    fb.gate.clear()
    q = api.ScanQueue(None, max_points=16, slots=3, max_batch=1, policy=URF_QUEUE_DROP_OLDEST | URF_QUEUE_ORDER, process_fn=fb)
    assert q.order
    assert q.submit(scan(0), tag=0) == URF_OK
    assert fb.started.acquire(timeout=5)
    for k in range(1, 6):                                # 1..3 are dropped in turn
        assert q.submit(scan(k), tag=k, timeout_ms=1000) == URF_OK
    assert q.stats()["dropped"] == 3
    fb.gate.set()
    got = drain(q, 3)
    assert [t for t, _ in got] == [0, 4, 5]
    for t, r in got:
        check(t, r)
    q.destroy()


def test_generation_update_in_mid_stream():
    """The stand-in writes an order that depends on the generation its batch ran with: each delivered scan carries the one
    of its own generation."""
    fb = OrderBatch()
    q = api.ScanQueue(None, max_points=16, slots=16, max_batch=4, process_fn=fb, label8=True, order=True)
    q.set_params_hook(fb.hook)
    fb.gate.clear()
    assert q.submit(scan(0), tag=0, timeout_ms=1000) == URF_OK
    assert fb.started.acquire(timeout=5)
    gen_of = {0: 0}
    for k in range(1, 15):
        if k in (5, 10):
            assert q.update_params(make_params(curb_points=3 + k)) == k // 5
        assert q.submit(scan(k), tag=k, timeout_ms=1000) == URF_OK
        gen_of[k] = k // 5
    fb.gate.set()
    got = drain(q, 15)
    assert [t for t, _ in got] == list(range(15))
    for t, r in got:
        assert r.params_gen == gen_of[t]
        check(t, r, gen=gen_of[t], label8=True)
    q.destroy()


def test_failed_batch_delivers_no_views():
    fb = OrderBatch(fail_on_batch=1)
    q = api.ScanQueue(None, max_points=16, slots=8, max_batch=2, process_fn=fb, order=True)
    fb.gate.clear()
    assert q.submit(scan(0), tag=0, timeout_ms=1000) == URF_OK
    assert fb.started.acquire(timeout=5)
    for k in (1, 2, 3):                                  # 1 and 2 are the second batch, which fails
        assert q.submit(scan(k), tag=k, timeout_ms=1000) == URF_OK
    fb.gate.set()
    got = drain(q, 4)
    assert [(t, r.status) for t, r in got] == [(0, URF_OK), (1, -3), (2, -3), (3, URF_OK)]
    for t, r in got:
        if r.status == URF_OK:
            check(t, r)
        else:
            assert r.label is None and r.order is None and r.ring_start is None
    # the raw call: outs[j].order / ring_start are NULL for the failed scans
    for k in (4, 5):
        fb.fail_on_batch = len(fb.given)
        assert q.submit(scan(k), tag=k, timeout_ms=1000) == URF_OK
        outs, rcs = (UrfResult * 1)(), (C.c_int32 * 1)()
        assert api.load_library().urf_queue_next_batch(q._q, 1, None, rcs, outs, None, 5000) == 1
        assert rcs[0] == -3 and not outs[0].order and not outs[0].ring_start
    q.destroy()


def test_without_the_bit_nothing_is_passed_or_delivered():
    lib = api.load_library()
    fb = OrderBatch()
    q = api.ScanQueue(None, max_points=16, slots=4, max_batch=2, process_fn=fb)
    for k in range(3):
        assert q.submit(scan(k), tag=k, timeout_ms=1000) == URF_OK
    t, r = q.next(5000)
    assert r.order is None and r.ring_start is None
    with pytest.raises(ValueError):
        r.cloud_indices("road")
    # the caller's order / ring_start pointers come back NULL, as before the bit existed
    res = UrfResult()
    order, rs = np.zeros(16, np.int32), np.zeros(URF_MAX_CHANNELS + 1, np.int32)
    res.order, res.ring_start = order.ctypes.data_as(C.POINTER(C.c_int32)), rs.ctypes.data_as(C.POINTER(C.c_int32))
    assert lib.urf_queue_next(q._q, None, C.byref(res), 5000) == URF_OK
    assert not res.order and not res.ring_start and not order.any() and not rs.any()
    outs = (UrfResult * 2)()
    assert lib.urf_queue_next_batch(q._q, 2, None, None, outs, None, 5000) == 1
    assert not outs[0].order and not outs[0].ring_start
    assert fb.given and not any(fb.given)                # the stand-in was never handed order buffers
    q.destroy()


@pytest.mark.parametrize("label8", [False, True])
def test_cloud_indices_on_queue_results(label8):
    fb = OrderBatch()
    q = api.ScanQueue(None, max_points=32, slots=4, max_batch=2, process_fn=fb, order=True, label8=label8)
    pts = scan(0, 24)
    pts[:, 0] = np.arange(24) % 3                        # labels 0, 1, 2 (scan 0: label = int(x))
    assert q.submit(pts, tag=0, timeout_ms=1000) == URF_OK
    assert q.submit(scan(11, 24), tag=11, timeout_ms=1000) == URF_OK      # 12 rings
    got = drain(q, 2)
    r = got[0][1]
    order, rs = expect_order(0, 24)
    lab = np.arange(24) % 3
    assert r.cloud_indices("road").size and r.cloud_indices("curb").size
    np.testing.assert_array_equal(r.cloud_indices("road"), order[lab[order] == 1])
    np.testing.assert_array_equal(r.cloud_indices("curb"), order[lab[order] == 2])
    np.testing.assert_array_equal(r.cloud_indices("roi"), np.arange(24))
    assert r.cloud_indices("road_probably").size == 0   # one ring
    order, rs = expect_order(11, 24)
    assert rs.size == 13
    np.testing.assert_array_equal(got[1][1].cloud_indices("road_probably"), order[rs[10]: rs[11]])
    q.destroy()


def test_policy_bits_are_checked():
    lib = api.load_library()
    fn = QUEUE_PROCESS_FN(OrderBatch())
    fin = QUEUE_FINISH_FN(lambda user: 0)
    h = C.c_void_p()
    for bad in (8, 16, URF_QUEUE_ORDER | 8, 1 << 30, -1):
        assert lib.urf_queue_create_with(C.byref(h), fn, None, 16, 2, 1, bad) == URF_ERR_INVALID, bad
        assert lib.urf_queue_create_with_async(C.byref(h), fn, fin, None, 16, 2, 1, bad) == URF_ERR_INVALID, bad
        assert lib.urf_mq_create_with_policy(C.byref(h), fn, None, 2, 16, 2, 1, bad) == URF_ERR_INVALID, bad
    dv = (C.c_int * 1)(0)
    for bad in (URF_QUEUE_DROP_OLDEST, URF_QUEUE_DROP_OLDEST | URF_QUEUE_ORDER, URF_QUEUE_DROP_OLDEST | URF_QUEUE_LABEL8, 8):
        assert lib.urf_mq_create_with_policy(C.byref(h), fn, None, 2, 16, 2, 1, bad) == URF_ERR_INVALID, bad
        assert lib.urf_mq_create_policy(C.byref(h), dv, 1, 16, 2, 1, None, bad) == URF_ERR_INVALID, bad   # before any device
    for good in (URF_QUEUE_BLOCK, URF_QUEUE_ORDER, URF_QUEUE_LABEL8 | URF_QUEUE_ORDER):
        assert lib.urf_queue_create_with(C.byref(h), fn, None, 16, 2, 1, good) == URF_OK
        lib.urf_queue_destroy(h)
        assert lib.urf_queue_create_with(C.byref(h), fn, None, 16, 2, 1, good | URF_QUEUE_DROP_OLDEST) == URF_OK
        lib.urf_queue_destroy(h)
        assert lib.urf_mq_create_with_policy(C.byref(h), fn, None, 2, 16, 2, 1, good) == URF_OK
        lib.urf_mq_destroy(h)
    assert lib.urf_queue_create(C.byref(h), None, 16, 2, 1, URF_QUEUE_ORDER) == URF_ERR_INVALID    # still needs a ctx


@pytest.mark.parametrize("label8", [False, True])
def test_mq_one_producer(label8):
    fb = OrderBatch()
    mq = api.MultiGpuQueue([0, 1, 2], max_points=32, slots_per_device=3, max_batch=2, process_fn=fb, label8=label8, order=True)
    mq.set_params_hook(fb.hook)
    got = []
    cons = threading.Thread(target=lambda: got.extend(drain(mq, 40, 5)))
    cons.start()
    for k in range(40):
        if k == 20:
            assert mq.update_params(make_params(curb_points=9)) == 1
        assert mq.submit(scan(k, 8 + k % 9), tag=k, timeout_ms=5000) == URF_OK
    cons.join(30)
    assert not cons.is_alive()
    assert [t for t, _ in got] == list(range(40))
    for t, r in got:
        assert r.params_gen == (t >= 20)
        check(t, r, 8 + t % 9, gen=r.params_gen, label8=label8)
    # next: the caller's buffers, copies
    for k in (50, 51):
        assert mq.submit(scan(k), tag=k, timeout_ms=5000) == URF_OK
        t, r = mq.next(5000)
        assert t == k
        check(k, r, gen=1, label8=label8)
        assert r.order.flags.owndata
    mq.destroy()


def test_mq_several_producers():
    fb = OrderBatch()
    mq = api.MultiGpuQueue([0, 1, 2], max_points=32, slots_per_device=4, max_batch=3, process_fn=fb, order=True)
    P, K = 3, 40
    got = []

    def consume():
        while len(got) < P * K:
            out = mq.next_batch(6, timeout_ms=5000)            # views, checked before the next call gives them back
            assert out
            for t, r in out:
                check(t % 100, r, 8 + t % 9)
            got.extend(t for t, _ in out)

    cons = threading.Thread(target=consume)
    cons.start()

    def produce(p):
        for k in range(K):
            tag = 1000 * p + k
            assert mq.submit(scan(tag % 100, 8 + tag % 9), tag=tag, timeout_ms=5000) == URF_OK

    prods = [threading.Thread(target=produce, args=(p,)) for p in range(P)]
    for t in prods:
        t.start()
    for t in prods:
        t.join(30)
    cons.join(30)
    assert not cons.is_alive() and sorted(got) == sorted(1000 * p + k for p in range(P) for k in range(K))
    for p in range(P):                                   # one producer's scans come back in its order
        mine = [t for t in got if t // 1000 == p]
        assert mine == sorted(mine)
    mq.destroy()


@pytest.mark.parametrize("args", [("4", "1500", "6", "4", "4"), ("3", "1200", "5", "2", "5"), ("2", "1500", "4", "3", "6"),
                                  ("1", "3000", "2", "1", "4")])
def test_queue_order_thread_sanitizer_stress(args):
    """urf_queue.cpp built with -fsanitize=thread (tests/kat/queue_order_stress.cpp): producers x scans x slots x max_batch
    x policy bits (URF_QUEUE_ORDER, with 1 DROP_OLDEST, 2 int8 labels), random parameter updates, one next_batch consumer.
    The binary checks every order and ring_start payload against its tag and generation; TSAN that there is no data race."""
    out = subprocess.run([os.path.join(ROOT, "build", "queue_order_stress"), *args], capture_output=True, text=True, timeout=600)
    print(out.stdout, out.stderr[-3000:])
    assert out.returncode == 0 and out.stdout.strip().endswith("OK") and "ThreadSanitizer" not in out.stderr

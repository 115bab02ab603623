"""PointCloud2 record scans through urf_mq and urf_queue without a GPU (urf_mq_create_cloud2_with,
urf_queue_create_cloud2_with): the queues run around a stand-in batch function that is handed the raw records and the record
format (a urf_cloud2_user as its `user`), decodes x / y / z at the format's offsets and writes labels, an order and ring
offsets derived from the scan, as tests/test_queue_order.py's stand-ins do for float4 scans. Covered: the bytes the stand-in
gets are the submitted records (with the by-reference submits, the caller's own buffer), global delivery order over three
stand-in devices with one producer and with several, next / next_view / next_batch with int8 slots and URF_QUEUE_ORDER, a
mid-stream parameter update (generations and batch cuts through the parameter hook), a failed batch, and every refusal. The
ThreadSanitizer program tests/kat/mq_records_stress.cpp mixes copying and by-reference record submits from several producers
with an updater and one consumer."""
import ctypes as C
import os
import subprocess
import threading

import numpy as np
import pytest

from urban_road_filter_b200 import api, make_params
from urban_road_filter_b200.ctypes_abi import (URF_ERR_CAPACITY, URF_ERR_INVALID, URF_OK, URF_QUEUE_BLOCK,
                                               URF_QUEUE_DROP_OLDEST, URF_QUEUE_LABEL8, URF_QUEUE_ORDER, QUEUE_PROCESS_FN,
                                               UrfCloud2User, UrfResult)
from util import ROOT, cloud2_records

from test_queue import scan
from test_queue_order import check, drain, expect_order

FMT48 = (48, 0, 4, 8, 16)             # Ouster: x, y, z at 0, 4, 8, intensity at 16
FMT22 = (22, 0, 4, 8, 12)             # Velodyne: x, y, z, intensity, then ring and time: records are not 4-byte aligned
FORMATS = [FMT48, FMT22]


def records(k, n, fmt, seed=None):
    """Record bytes of test_queue.scan(k, n) (x = point index, y = k, intensity = 0.5 * index) with seeded garbage in the
    bytes the format does not use."""
    pts = scan(k, n)
    pts[:, 3] = 0.5 * np.arange(n)
    return cloud2_records(pts, *fmt, seed=k if seed is None else seed)


def _fmt(u: UrfCloud2User):
    return (u.point_step, u.off_x, u.off_y, u.off_z, u.off_intensity)


class RecordBatch:
    """Synchronous record stand-in (urf_process_batch's signature; `user` is the queue's urf_cloud2_user). For scan j it
    decodes the records at the format's offsets and writes what test_queue_order.check expects for scan k = int(y), with the
    generation the parameter hook last named on the calling worker thread. Records, per batch, its generation and scans, and
    per scan k the address and a copy of the bytes it was handed. `gate` holds it back; `fail_on_batch` fails that batch."""

    def __init__(self, fail_on_batch=None):
        self.gate = threading.Event()
        self.gate.set()
        self.started = threading.Semaphore(0)
        self.fail_on_batch = fail_on_batch
        self.lock = threading.Lock()
        self.batches = []                                # (generation, [k of each scan]), None for a failed batch
        self.seen = {}                                   # k -> (address, bytes) of the last scan k handed in
        self.formats = set()                             # (format, user pointer) of every call
        self.gen = {}                                    # worker thread -> generation
        self.hook_sets = {}                              # generation -> curb_points of the set the hook got

    def hook(self, user, prm, gen):
        u = C.cast(user, C.POINTER(UrfCloud2User)).contents
        with self.lock:
            self.formats.add((_fmt(u), u.user))
            self.gen[threading.get_ident()] = gen
            self.hook_sets[gen] = prm.contents.curb_points
        return URF_OK

    def __call__(self, user, xyzi, n, batch, outs):
        self.started.release()
        self.gate.wait()
        u = C.cast(user, C.POINTER(UrfCloud2User)).contents
        fmt = _fmt(u)
        step, ox, oy, oz, _ = fmt
        with self.lock:
            i = len(self.batches)
            self.batches.append(None)
            self.formats.add((fmt, u.user))
        if i == self.fail_on_batch:
            return -3
        gen = self.gen.get(threading.get_ident(), 0)
        ks = []
        for j in range(batch):
            nj = n[j]
            raw = (np.ctypeslib.as_array(C.cast(xyzi[j], C.POINTER(C.c_uint8)), shape=(nj * step,)).copy() if nj
                   else np.zeros(0, np.uint8))
            rec = raw.reshape(nj, step)
            x, y = (rec[:, o: o + 4].copy().view(np.float32).ravel() for o in (ox, oy))
            k = int(y[0]) if nj else 0
            with self.lock:
                self.seen[k] = (xyzi[j], raw)
            out = outs[j]
            if nj:
                np.ctypeslib.as_array(out.label, shape=(nj,))[:] = x.astype(np.int32) + 1000 * k
            out.status, out.n_in, out.n_roi, out.n_vert = 0, nj, nj, 0
            if out.order:
                order, rs = expect_order(k, nj, gen)
                out.n_order, out.n_rings = order.size, rs.size - 1
                if order.size:
                    np.ctypeslib.as_array(out.order, shape=(order.size,))[:] = order
                np.ctypeslib.as_array(out.ring_start, shape=(rs.size,))[:] = rs
            ks.append(k)
        self.batches[i] = (gen, ks)
        return 0


def record_mq(fb, devices=3, fmt=FMT48, slots=4, max_batch=3, label8=False, order=True):
    return api.MultiGpuQueue(list(range(devices)), max_points=64, slots_per_device=slots, max_batch=max_batch, process_fn=fb,
                             label8=label8, order=order, records=fmt)


@pytest.mark.parametrize("fmt", FORMATS)
@pytest.mark.parametrize("kind", ["queue", "mq"])
def test_the_stand_in_gets_the_submitted_records(kind, fmt):
    """Byte for byte; by reference the very buffer the caller passed (nothing copied), otherwise a slot of the queue. The
    stand-in's urf_cloud2_user carries the format and the creator's user (NULL here)."""
    fb = RecordBatch()
    q = (api.ScanQueue(None, max_points=64, slots=4, max_batch=2, process_fn=fb, records=fmt) if kind == "queue"
         else record_mq(fb, fmt=fmt))
    raws = {}
    for k in range(12):
        raws[k] = records(k, 5 + k, fmt)
        assert q.submit_records(raws[k], 5 + k, tag=k, timeout_ms=5000, by_reference=bool(k % 2)) == URF_OK
        t, r = q.next(5000)
        assert t == k and r.n_in == 5 + k
        np.testing.assert_array_equal(r.label, np.arange(5 + k) + 1000 * k)
        addr, got = fb.seen[k]
        assert got.tobytes() == raws[k].tobytes(), k
        if k % 2:
            assert addr == raws[k].ctypes.data, k                    # the caller's buffer, used in place
        else:
            assert addr != raws[k].ctypes.data, k                    # a copy in the queue's slot
    assert fb.formats == {(fmt, None)}
    q.destroy()


def test_by_reference_records_are_read_when_the_batch_runs_and_kept_until_delivered():
    """urf_queue_submit_cloud2_ref on a single record queue: the worker reads the caller's bytes when it runs the batch (a
    change made before that is what it sees), and the wrapper keeps the array until its result has come back."""
    fb = RecordBatch()
    fb.gate.clear()
    q = api.ScanQueue(None, max_points=32, slots=4, max_batch=1, process_fn=fb, records=FMT48)
    first = records(0, 8, FMT48)
    assert q.submit_records(first, 8, tag=0, timeout_ms=1000) == URF_OK
    assert fb.started.acquire(timeout=5)                             # scan 0 is running; scan 1 waits behind it
    raw = records(1, 8, FMT48)
    assert q.submit_records(raw, 8, tag=1, timeout_ms=1000, by_reference=True) == URF_OK
    assert q._keep[1].ctypes.data == raw.ctypes.data                # a view of the caller's array is kept
    raw.reshape(8, 48)[:, 0:4] = np.full((8, 1), 7.0, np.float32).view(np.uint8)   # every x = 7, after the submit
    fb.gate.set()
    got = drain(q, 2)
    assert [t for t, _ in got] == [0, 1]
    np.testing.assert_array_equal(got[1][1].label, np.full(8, 7 + 1000, np.int32))
    assert fb.seen[1][0] == raw.ctypes.data and 1 not in q._keep
    # bytes objects (a message's `data`) are accepted too, and kept by reference
    msg = records(2, 8, FMT48).tobytes()
    assert q.submit_records(msg, 8, tag=2, timeout_ms=1000, by_reference=True) == URF_OK
    t, r = q.next(5000)
    assert t == 2 and fb.seen[2][1].tobytes() == msg
    q.destroy()


@pytest.mark.parametrize("label8", [False, True])
def test_mq_one_producer_every_delivery(label8):
    """Three stand-in devices, one producer mixing copying and by-reference record submits: the global order is the
    submission order, and next (copies), next_view (int32 slots) and next_batch views deliver the stand-in's payload."""
    fb = RecordBatch()
    mq = record_mq(fb, label8=label8)
    got = []
    cons = threading.Thread(target=lambda: got.extend(drain(mq, 45, 5)))
    cons.start()
    keep = []
    for k in range(45):
        raw = records(k, 8 + k % 9, FMT48)
        keep.append(raw)
        assert mq.submit_records(raw, 8 + k % 9, tag=k, timeout_ms=5000, by_reference=bool(k % 3 == 1)) == URF_OK
    cons.join(30)
    assert not cons.is_alive()
    assert [t for t, _ in got] == list(range(45))
    for t, r in got:
        check(t, r, 8 + t % 9, label8=label8)
    st = mq.stats()
    assert sum(st["delivered"]) == 45 and all(d > 0 for d in st["delivered"]), st
    for k in (50, 51):                                   # next: copies into the wrapper's buffers
        assert mq.submit_records(records(k, 12, FMT48), 12, tag=k, timeout_ms=5000) == URF_OK
        t, r = mq.next(5000)
        assert t == k
        check(k, r, 12, label8=label8)
        assert r.order.flags.owndata
    if not label8:                                       # next_view: labels, order and ring_start in the slot
        lib = api.load_library()
        assert mq.submit_records(records(52, 12, FMT48), 12, tag=52, timeout_ms=5000) == URF_OK
        res, tag, view = UrfResult(), C.c_uint64(), C.c_void_p()
        assert lib.urf_mq_next_view(mq._m, C.byref(tag), C.byref(res), C.byref(view), 5000) == URF_OK
        r = api._scan_result(res, np.ctypeslib.as_array(C.cast(view, C.POINTER(C.c_int32)), shape=(res.n_in,)),
                             order=np.ctypeslib.as_array(res.order, shape=(res.n_order,)),
                             ring_start=np.ctypeslib.as_array(res.ring_start, shape=(res.n_rings + 1,)))
        assert tag.value == 52
        check(52, r, 12)
    mq.destroy()


def test_mq_several_producers():
    fb = RecordBatch()
    mq = record_mq(fb, fmt=FMT22, slots=4, max_batch=3, label8=True)
    P, K = 3, 40
    got, err = [], []

    def consume():
        try:
            while len(got) < P * K:
                out = mq.next_batch(6, timeout_ms=5000)        # views, checked before the next call gives them back
                assert out
                for t, r in out:
                    check(t % 100, r, 8 + t % 9, label8=True)
                got.extend(t for t, _ in out)
        except BaseException as e:                         # noqa: BLE001 — re-raised below
            err.append(e)

    cons = threading.Thread(target=consume)
    cons.start()

    def produce(p):
        mine = []                                          # by-reference arrays stay alive until the end
        for k in range(K):
            tag = 1000 * p + k
            raw = records(tag % 100, 8 + tag % 9, FMT22)
            mine.append(raw)
            assert mq.submit_records(raw, 8 + tag % 9, tag=tag, timeout_ms=5000, by_reference=bool((k + p) % 2)) == URF_OK

    prods = [threading.Thread(target=produce, args=(p,)) for p in range(P)]
    for t in prods:
        t.start()
    for t in prods:
        t.join(30)
    cons.join(30)
    assert not cons.is_alive() and not err, err
    assert sorted(got) == sorted(1000 * p + k for p in range(P) for k in range(K))
    for p in range(P):                                     # one producer's scans come back in its order
        mine = [t for t in got if t // 1000 == p]
        assert mine == sorted(mine)
    assert fb.formats == {(FMT22, None)}
    mq.destroy()


def test_mq_update_in_mid_stream_cuts_batches_at_generations():
    """Two urf_mq_update_params while scans wait: every scan reports the generation in force when it was accepted, its
    payload is that generation's, no batch mixes generations, and the hook got each generation's set and the format."""
    fb = RecordBatch()
    mq = record_mq(fb, slots=12, max_batch=4, label8=True)
    mq.set_params_hook(fb.hook)
    fb.gate.clear()
    assert mq.submit_records(records(0, 16, FMT48), 16, tag=0, timeout_ms=1000) == URF_OK
    assert fb.started.acquire(timeout=5)
    gen_of = {0: 0}
    for k in range(1, 30):
        if k in (10, 20):
            assert mq.update_params(make_params(curb_points=k // 10 + 3)) == k // 10
        assert mq.submit_records(records(k, 16, FMT48), 16, tag=k, timeout_ms=1000, by_reference=bool(k % 2)) == URF_OK
        gen_of[k] = k // 10
    fb.gate.set()
    got = drain(mq, 30)
    assert [t for t, _ in got] == list(range(30))
    for t, r in got:
        assert r.params_gen == gen_of[t], t
        check(t, r, gen=gen_of[t], label8=True)
    runs = [b for b in fb.batches if b is not None]
    assert sum(len(ks) for _, ks in runs) == 30
    for gen, ks in runs:
        assert all(gen_of[k] == gen for k in ks), (gen, ks)
    assert any(len(ks) > 1 for _, ks in runs)                      # the waiting scans did run as batches
    assert fb.hook_sets == {1: 4, 2: 5}
    assert fb.formats == {(FMT48, None)}
    mq.destroy()


@pytest.mark.parametrize("kind", ["queue", "mq"])
def test_failed_batch(kind):
    fb = RecordBatch(fail_on_batch=1)
    q = (api.ScanQueue(None, max_points=16, slots=8, max_batch=2, process_fn=fb, records=FMT48, order=True) if kind == "queue"
         else record_mq(fb, devices=1, slots=8, max_batch=2))
    fb.gate.clear()
    assert q.submit_records(records(0, 16, FMT48), 16, tag=0, timeout_ms=1000) == URF_OK
    assert fb.started.acquire(timeout=5)
    for k in (1, 2, 3):                                  # 1 and 2 are the second batch, which fails
        assert q.submit_records(records(k, 16, FMT48), 16, tag=k, timeout_ms=1000, by_reference=k == 2) == URF_OK
    fb.gate.set()
    got = drain(q, 4)
    assert [(t, r.status) for t, r in got] == [(0, URF_OK), (1, -3), (2, -3), (3, URF_OK)]
    for t, r in got:
        if r.status == URF_OK:
            check(t, r)
        else:
            assert r.label is None and r.order is None and r.ring_start is None
    q.destroy()


def test_refusals():
    lib = api.load_library()
    fn = QUEUE_PROCESS_FN(RecordBatch())
    h = C.c_void_p()
    raw = records(0, 8, FMT48)
    pts = scan(0, 8)
    # float4 submits on a record mq / queue, and record submits on a float4 one
    for q in (record_mq(RecordBatch()), api.ScanQueue(None, max_points=64, slots=2, max_batch=1, process_fn=RecordBatch(), records=FMT48)):
        for by_ref in (False, True):
            with pytest.raises(api.UrfError) as e:
                q.submit(pts, tag=1, timeout_ms=1000, by_reference=by_ref)
            assert e.value.code == URF_ERR_INVALID
        with pytest.raises(api.UrfError) as e:                     # n_points > max_points
            q.submit_records(records(0, 65, FMT48), 65, tag=2, timeout_ms=1000)
        assert e.value.code == URF_ERR_CAPACITY
        with pytest.raises(ValueError):                              # fewer bytes than n_points records
            q.submit_records(raw, 9, tag=3)
        assert q.submit_records(raw, 8, tag=4, timeout_ms=1000) == URF_OK      # nothing refused was counted
        t, _ = q.next(5000)
        assert t == 4 and q.next(0) is None
        q.destroy()
    for q in (api.MultiGpuQueue([0, 1], max_points=64, process_fn=RecordBatch()),
              api.ScanQueue(None, max_points=64, slots=2, max_batch=1, process_fn=RecordBatch())):
        for by_ref in (False, True):
            with pytest.raises(api.UrfError) as e:
                q.submit_records(raw, 8, tag=1, timeout_ms=1000, by_reference=by_ref)
            assert e.value.code == URF_ERR_INVALID
        q.destroy()
    mq = record_mq(RecordBatch())
    assert mq.stats()["submitted"] == [0, 0, 0]
    for f in (lib.urf_mq_submit, lib.urf_mq_submit_ref):
        assert f(mq._m, pts.ctypes.data, 8, 0, 1000) == URF_ERR_INVALID
    assert mq.stats()["submitted"] == [0, 0, 0] and mq.stats()["pending"] == 0
    mq.destroy()
    # record formats (urf_queue_create_cloud2's checks) and policies
    bad_formats = [(11, 0, 4, 8, -1), (65, 0, 4, 8, -1), (48, -1, 4, 8, 16), (48, 0, 45, 8, 16), (48, 0, 4, 8, 45),
                   (22, 0, 4, 19, -1), (12, 0, 4, 8, 9)]
    dv = (C.c_int * 1)(0)
    for fmt in bad_formats:
        assert lib.urf_queue_create_cloud2_with(C.byref(h), fn, None, 16, 2, 1, URF_QUEUE_BLOCK, *fmt) == URF_ERR_INVALID, fmt
        assert lib.urf_mq_create_cloud2_with(C.byref(h), fn, None, 2, 16, 2, 1, URF_QUEUE_BLOCK, *fmt) == URF_ERR_INVALID, fmt
        assert lib.urf_mq_create_cloud2(C.byref(h), dv, 1, 16, 2, 1, None, URF_QUEUE_BLOCK, *fmt) == URF_ERR_INVALID, fmt
        assert lib.urf_queue_create_cloud2(C.byref(h), None, 16, 2, 1, URF_QUEUE_BLOCK, *fmt) == URF_ERR_INVALID, fmt
    for bad in (URF_QUEUE_DROP_OLDEST, URF_QUEUE_DROP_OLDEST | URF_QUEUE_ORDER, URF_QUEUE_DROP_OLDEST | URF_QUEUE_LABEL8, 8, -1):
        assert lib.urf_mq_create_cloud2_with(C.byref(h), fn, None, 2, 16, 2, 1, bad, *FMT48) == URF_ERR_INVALID, bad
        assert lib.urf_mq_create_cloud2(C.byref(h), dv, 1, 16, 2, 1, None, bad, *FMT48) == URF_ERR_INVALID, bad   # before any device
    assert lib.urf_queue_create_cloud2_with(C.byref(h), QUEUE_PROCESS_FN(), None, 16, 2, 1, URF_QUEUE_BLOCK, *FMT48) == URF_ERR_INVALID
    for good in ((12, 0, 4, 8, -1), (64, 52, 56, 60, 0), FMT22):
        for policy in (URF_QUEUE_BLOCK, URF_QUEUE_LABEL8 | URF_QUEUE_ORDER):
            assert lib.urf_mq_create_cloud2_with(C.byref(h), fn, None, 2, 16, 2, 1, policy, *good) == URF_OK
            lib.urf_mq_destroy(h)
        assert lib.urf_queue_create_cloud2_with(C.byref(h), fn, None, 16, 2, 1, URF_QUEUE_DROP_OLDEST, *good) == URF_OK
        lib.urf_queue_destroy(h)
    with pytest.raises(ValueError):
        api.ScanQueue(None, max_points=16, records=FMT48, enqueue_fn=lambda *a: 0, finish_fn=lambda: 0)


def test_record_queue_drop_oldest():
    """A single record queue keeps urf_queue's policies: DROP_OLDEST drops waiting scans, by reference or not."""
    fb = RecordBatch()
    fb.gate.clear()
    q = api.ScanQueue(None, max_points=16, slots=3, max_batch=1, policy=URF_QUEUE_DROP_OLDEST, process_fn=fb, records=FMT22,
                      order=True)
    assert q.submit_records(records(0, 16, FMT22), 16, tag=0) == URF_OK
    assert fb.started.acquire(timeout=5)
    for k in range(1, 6):                                # 1..3 are dropped in turn
        assert q.submit_records(records(k, 16, FMT22), 16, tag=k, timeout_ms=1000, by_reference=bool(k % 2)) == URF_OK
    assert q.stats()["dropped"] == 3
    fb.gate.set()
    got = drain(q, 3)
    assert [t for t, _ in got] == [0, 4, 5]
    for t, r in got:
        check(t, r)
    q.destroy()


@pytest.mark.parametrize("args", [("4", "1500", "4", "3", "2", "48"), ("3", "1200", "3", "4", "6", "22"), ("2", "2000", "2", "2", "0", "32")])
def test_mq_records_thread_sanitizer_stress(args):
    """urf_queue.cpp and urf_mq.cpp built with -fsanitize=thread (tests/kat/mq_records_stress.cpp): producers x scans x
    devices x slots per device x policy bits x point_step; producers mix copying and by-reference record submits, one thread
    updates the parameters, one consumer takes batches. The binary checks every payload against its tag and generation;
    TSAN that there is no data race."""
    out = subprocess.run([os.path.join(ROOT, "build", "mq_records_stress"), *args], capture_output=True, text=True, timeout=600)
    print(out.stdout, out.stderr[-3000:])
    assert out.returncode == 0 and out.stdout.strip().endswith("OK") and "ThreadSanitizer" not in out.stderr

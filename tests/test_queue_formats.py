"""PointCloud2 records of several sensor formats through one urf_queue / urf_mq, without a GPU (urf_queue_create_formats_with,
urf_mq_create_formats_with): the queues run around a stand-in batch function whose `user` is the queue's urf_formats_user
(the format table and, during the call, each scan's format index). The stand-in decodes every scan at its own format's
offsets and writes labels, an order and ring offsets derived from the scan, as tests/test_mq_records.py's stand-in does for
one format. Covered: the bytes and format index each scan arrives with (copying and by-reference submits), a scan of
max_points records of the largest format, global delivery order over three stand-in devices with one producer and with
several, next / next_view / next_batch with int8 slots and URF_QUEUE_ORDER, a mid-stream parameter update (batches cut at
the generation, never at a format change), DROP_OLDEST, a failed batch, and every refusal. The ThreadSanitizer program
tests/kat/queue_formats_stress.cpp mixes formats, copying and by-reference submits, an updater and one consumer."""
import ctypes as C
import os
import subprocess
import threading

import numpy as np
import pytest

from urban_road_filter_b200 import api, make_params
from urban_road_filter_b200.ctypes_abi import (URF_ERR_CAPACITY, URF_ERR_INVALID, URF_MAX_FORMATS, URF_OK, URF_QUEUE_BLOCK,
                                               URF_QUEUE_DROP_OLDEST, URF_QUEUE_LABEL8, URF_QUEUE_ORDER, QUEUE_PROCESS_FN,
                                               UrfFormatsUser, UrfResult)
from util import ROOT

from test_mq_records import records
from test_queue import scan
from test_queue_order import check, drain, expect_order

OUSTER = api.CloudFormat(48, 0, 4, 8, 16)         # x, y, z at 0, 4, 8, intensity at 16
VELO32 = api.CloudFormat(32, 0, 4, 8, 16)
VELO22 = api.CloudFormat(22, 0, 4, 8, 12)         # packed: records are not 4-byte aligned
TABLE = [OUSTER, VELO32, VELO22, api.FLOAT4_FORMAT]


def fmt_of(k):
    """The format index scan k is submitted with: the table's formats in turn, in an order that is not the tags'."""
    return (k * 3 + k // 4) % len(TABLE)


class FormatsBatch:
    """Synchronous formats stand-in (urf_process_batch's signature; `user` is the queue's urf_formats_user). For scan j it
    reads the format index the queue names, decodes the records at that format's offsets and writes what
    test_queue_order.check expects for scan k = int(y), with the generation the parameter hook last named on the calling
    worker thread. Records per batch its generation, scans and format indices, and per scan k the address, format index and
    a copy of the bytes it was handed. `gate` holds it back; `fail_on_batch` fails that batch."""

    def __init__(self, fail_on_batch=None):
        self.gate = threading.Event()
        self.gate.set()
        self.started = threading.Semaphore(0)
        self.fail_on_batch = fail_on_batch
        self.lock = threading.Lock()
        self.batches = []                                # (generation, [k], [format index]), None for a failed batch
        self.seen = {}                                   # k -> (address, format index, bytes)
        self.tables = set()                              # (format table, creator's user) of every call
        self.gen = {}                                    # worker thread -> generation
        self.hook_sets = {}                              # generation -> curb_points of the set the hook got

    @staticmethod
    def _table(u):
        return tuple(api.CloudFormat(f.point_step, f.off_x, f.off_y, f.off_z, f.off_intensity) for f in u.formats[: u.n_formats])

    def hook(self, user, prm, gen):
        u = C.cast(user, C.POINTER(UrfFormatsUser)).contents
        with self.lock:
            self.tables.add((self._table(u), u.user))
            self.gen[threading.get_ident()] = gen
            self.hook_sets[gen] = prm.contents.curb_points
        return URF_OK

    def __call__(self, user, xyzi, n, batch, outs):
        self.started.release()
        self.gate.wait()
        u = C.cast(user, C.POINTER(UrfFormatsUser)).contents
        table = self._table(u)
        with self.lock:
            i = len(self.batches)
            self.batches.append(None)
            self.tables.add((table, u.user))
        if i == self.fail_on_batch:
            return -3
        gen = self.gen.get(threading.get_ident(), 0)
        ks, fs = [], []
        for j in range(batch):
            f = u.fmt[j]
            step, ox, oy = table[f][:3]
            nj = n[j]
            raw = (np.ctypeslib.as_array(C.cast(xyzi[j], C.POINTER(C.c_uint8)), shape=(nj * step,)).copy() if nj
                   else np.zeros(0, np.uint8))
            rec = raw.reshape(nj, step)
            x, y = (rec[:, o: o + 4].copy().view(np.float32).ravel() for o in (ox, oy))
            k = int(y[0]) if nj else 0
            with self.lock:
                self.seen[k] = (xyzi[j], f, raw)
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
            fs.append(f)
        self.batches[i] = (gen, ks, fs)
        return 0


def formats_queue(fb, max_points=64, slots=4, max_batch=3, policy=URF_QUEUE_BLOCK, order=True, label8=False, table=TABLE):
    return api.ScanQueue(None, max_points=max_points, slots=slots, max_batch=max_batch, policy=policy, process_fn=fb, order=order,
                         label8=label8, formats=table)


def formats_mq(fb, devices=3, slots=4, max_batch=3, label8=False, order=True, table=TABLE):
    return api.MultiGpuQueue(list(range(devices)), max_points=64, slots_per_device=slots, max_batch=max_batch, process_fn=fb,
                             label8=label8, order=order, formats=table)


def submit(q, k, n, by_reference=False, timeout_ms=5000):
    f = fmt_of(k)
    raw = records(k, n, TABLE[f])
    assert q.submit_records(raw, n, tag=k, timeout_ms=timeout_ms, by_reference=by_reference, fmt=f) == URF_OK
    return raw


@pytest.mark.parametrize("kind", ["queue", "mq"])
def test_the_stand_in_gets_each_scans_bytes_and_format(kind):
    """Byte for byte, with the format index the scan was submitted with; by reference the very buffer the caller passed,
    otherwise a slot of the queue. The stand-in's urf_formats_user carries the table and the creator's user (NULL)."""
    fb = FormatsBatch()
    q = formats_queue(fb, max_batch=2) if kind == "queue" else formats_mq(fb)
    raws = {}
    for k in range(16):
        raws[k] = submit(q, k, 5 + k, by_reference=bool(k % 2))
        t, r = q.next(5000)
        assert t == k and r.n_in == 5 + k
        np.testing.assert_array_equal(r.label, np.arange(5 + k) + 1000 * k)
        addr, f, got = fb.seen[k]
        assert f == fmt_of(k) and got.tobytes() == raws[k].tobytes(), k
        if k % 2:
            assert addr == raws[k].ctypes.data, k
        else:
            assert addr != raws[k].ctypes.data, k
    assert {fmt_of(k) for k in range(16)} == set(range(len(TABLE)))
    assert fb.tables == {(tuple(TABLE), None)}
    q.destroy()


def test_a_full_scan_of_the_largest_format_fits_its_slot():
    """Slots hold max_points records of the table's largest point_step: a full scan of the 64-byte format is copied whole, and
    so is a full scan of the 12-byte one next to it."""
    big, small = api.CloudFormat(64, 52, 56, 60, 0), api.CloudFormat(12, 0, 4, 8, -1)
    fb = FormatsBatch()
    q = formats_queue(fb, max_points=40, slots=2, max_batch=2, table=[small, big])
    raw_big, raw_small = records(1, 40, big), records(2, 40, small)
    assert q.submit_records(raw_big, 40, tag=1, timeout_ms=5000, fmt=1) == URF_OK
    assert q.submit_records(raw_small, 40, tag=2, timeout_ms=5000, fmt=0) == URF_OK
    got = drain(q, 2)
    assert [t for t, _ in got] == [1, 2]
    for t, r in got:
        check(t, r, 40)
    assert fb.seen[1][1] == 1 and fb.seen[1][2].tobytes() == raw_big.tobytes()
    assert fb.seen[2][1] == 0 and fb.seen[2][2].tobytes() == raw_small.tobytes()
    q.destroy()


@pytest.mark.parametrize("label8", [False, True])
def test_mq_one_producer_every_delivery(label8):
    """Three stand-in devices, one producer mixing formats, copying and by-reference submits: the global order is the
    submission order, and next (copies), next_view (int32 slots) and next_batch views deliver the stand-in's payload."""
    fb = FormatsBatch()
    mq = formats_mq(fb, label8=label8)
    got = []
    cons = threading.Thread(target=lambda: got.extend(drain(mq, 48, 5)))
    cons.start()
    # while the stand-ins wait at the gate nothing is delivered, so scans 0..8 are dealt round-robin, three to a device, and
    # wait behind its first batch: each device runs its three in at most two batches, and one holds two of formats 0, 1, 3
    # (device 0: scans 0, 3, 6)
    fb.gate.clear()
    keep = [submit(mq, k, 8 + k % 9, by_reference=k % 3 == 1) for k in range(9)]
    fb.gate.set()
    keep += [submit(mq, k, 8 + k % 9, by_reference=k % 3 == 1) for k in range(9, 48)]
    cons.join(30)
    assert not cons.is_alive() and len(keep) == 48
    assert [t for t, _ in got] == list(range(48))
    for t, r in got:
        check(t, r, 8 + t % 9, label8=label8)
    st = mq.stats()
    assert sum(st["delivered"]) == 48 and all(d > 0 for d in st["delivered"]), st
    assert any(len(set(fs)) > 1 for _, _, fs in fb.batches), "no batch mixed formats"
    for k in (50, 51):                                   # next: copies into the wrapper's buffers
        submit(mq, k, 12)
        t, r = mq.next(5000)
        assert t == k
        check(k, r, 12, label8=label8)
        assert r.order.flags.owndata
    if not label8:                                       # next_view: labels, order and ring_start in the slot
        lib = api.load_library()
        submit(mq, 52, 12)
        res, tag, view = UrfResult(), C.c_uint64(), C.c_void_p()
        assert lib.urf_mq_next_view(mq._m, C.byref(tag), C.byref(res), C.byref(view), 5000) == URF_OK
        r = api._scan_result(res, np.ctypeslib.as_array(C.cast(view, C.POINTER(C.c_int32)), shape=(res.n_in,)),
                             order=np.ctypeslib.as_array(res.order, shape=(res.n_order,)),
                             ring_start=np.ctypeslib.as_array(res.ring_start, shape=(res.n_rings + 1,)))
        assert tag.value == 52
        check(52, r, 12)
    mq.destroy()


def test_mq_several_producers():
    """Three producers, each of its own format (as three LiDAR callbacks), on one mq: every scan once, each producer's in its
    order, and batches that mix the producers' formats."""
    fb = FormatsBatch()
    mq = formats_mq(fb, slots=4, max_batch=3, label8=True)
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
            raw = records(tag % 100, 8 + tag % 9, TABLE[p])
            mine.append(raw)
            assert mq.submit_records(raw, 8 + tag % 9, tag=tag, timeout_ms=5000, by_reference=bool((k + p) % 2), fmt=p) == URF_OK

    prods = [threading.Thread(target=produce, args=(p,)) for p in range(P)]
    for t in prods:
        t.start()
    for t in prods:
        t.join(30)
    cons.join(30)
    assert not cons.is_alive() and not err, err
    assert sorted(got) == sorted(1000 * p + k for p in range(P) for k in range(K))
    for p in range(P):
        mine = [t for t in got if t // 1000 == p]
        assert mine == sorted(mine)
    assert fb.tables == {(tuple(TABLE), None)}
    mq.destroy()


@pytest.mark.parametrize("kind", ["queue", "mq"])
def test_update_in_mid_stream_cuts_batches_at_generations_not_formats(kind):
    """Two updates while scans of every format wait: every scan reports the generation in force when it was accepted, no
    batch mixes generations, batches do mix formats, and the hook got each generation's set and the table."""
    fb = FormatsBatch()
    q = (formats_queue(fb, slots=32, max_batch=6, label8=True) if kind == "queue"
         else formats_mq(fb, devices=2, slots=16, max_batch=6, label8=True))
    q.set_params_hook(fb.hook)
    fb.gate.clear()
    submit(q, 0, 16)
    assert fb.started.acquire(timeout=5)
    gen_of = {0: 0}
    for k in range(1, 30):
        if k in (10, 20):
            assert q.update_params(make_params(curb_points=k // 10 + 3)) == k // 10
        submit(q, k, 16, by_reference=bool(k % 2))
        gen_of[k] = k // 10
    fb.gate.set()
    got = drain(q, 30)
    assert [t for t, _ in got] == list(range(30))
    for t, r in got:
        assert r.params_gen == gen_of[t], t
        check(t, r, gen=gen_of[t], label8=True)
    runs = [b for b in fb.batches if b is not None]
    assert sum(len(ks) for _, ks, _ in runs) == 30
    for gen, ks, fs in runs:
        assert all(gen_of[k] == gen for k in ks), (gen, ks)
        assert fs == [fmt_of(k) for k in ks], (ks, fs)
    assert any(len(set(fs)) > 1 for _, _, fs in runs)               # the cut is not at a format change
    assert fb.hook_sets == {1: 4, 2: 5}
    assert fb.tables == {(tuple(TABLE), None)}
    q.destroy()


@pytest.mark.parametrize("kind", ["queue", "mq"])
def test_failed_batch(kind):
    fb = FormatsBatch(fail_on_batch=1)
    q = formats_queue(fb, slots=8, max_batch=2) if kind == "queue" else formats_mq(fb, devices=1, slots=8, max_batch=2)
    fb.gate.clear()
    submit(q, 0, 16)
    assert fb.started.acquire(timeout=5)
    for k in (1, 2, 3):                                  # 1 and 2 are the second batch, which fails
        submit(q, k, 16, by_reference=k == 2)
    fb.gate.set()
    got = drain(q, 4)
    assert [(t, r.status) for t, r in got] == [(0, URF_OK), (1, -3), (2, -3), (3, URF_OK)]
    for t, r in got:
        if r.status == URF_OK:
            check(t, r)
        else:
            assert r.label is None and r.order is None and r.ring_start is None
    q.destroy()


def test_formats_queue_drop_oldest():
    """A single formats queue keeps urf_queue's policies: DROP_OLDEST drops waiting scans of any format, by reference or not."""
    fb = FormatsBatch()
    fb.gate.clear()
    q = formats_queue(fb, max_points=16, slots=3, max_batch=1, policy=URF_QUEUE_DROP_OLDEST)
    submit(q, 0, 16, timeout_ms=-1)
    assert fb.started.acquire(timeout=5)
    for k in range(1, 6):                                # 1..3 are dropped in turn
        submit(q, k, 16, by_reference=bool(k % 2), timeout_ms=1000)
    assert q.stats()["dropped"] == 3
    fb.gate.set()
    got = drain(q, 3)
    assert [t for t, _ in got] == [0, 4, 5]
    for t, r in got:
        check(t, r)
    assert [fs for _, _, fs in fb.batches] == [[fmt_of(0)], [fmt_of(4)], [fmt_of(5)]]
    q.destroy()


def test_refusals():
    lib = api.load_library()
    fn = QUEUE_PROCESS_FN(FormatsBatch())
    h = C.c_void_p()
    raw = records(0, 8, OUSTER)
    pts = scan(0, 8)
    fq = lambda: formats_queue(FormatsBatch(), slots=2, max_batch=1)      # noqa: E731
    for q in (formats_mq(FormatsBatch()), fq()):
        for by_ref in (False, True):
            with pytest.raises(api.UrfError) as e:                   # float4 submits
                q.submit(pts, tag=1, timeout_ms=1000, by_reference=by_ref)
            assert e.value.code == URF_ERR_INVALID
            with pytest.raises(api.UrfError) as e:                   # one-format record submits
                q.submit_records(raw, 8, tag=1, timeout_ms=1000, by_reference=by_ref)
            assert e.value.code == URF_ERR_INVALID
            for bad in (-1, len(TABLE), URF_MAX_FORMATS):            # a format index outside the table
                with pytest.raises(api.UrfError) as e:
                    q.submit_records(raw, 8, tag=1, timeout_ms=1000, by_reference=by_ref, fmt=bad)
                assert e.value.code == URF_ERR_INVALID
        with pytest.raises(api.UrfError) as e:                       # n_points > max_points
            q.submit_records(records(0, 65, OUSTER), 65, tag=2, timeout_ms=1000, fmt=0)
        assert e.value.code == URF_ERR_CAPACITY
        with pytest.raises(ValueError):                              # fewer bytes than n_points records of that format
            q.submit_records(raw, 9, tag=3, fmt=0)
        assert q.submit_records(raw, 8, tag=4, timeout_ms=1000, fmt=0) == URF_OK   # nothing refused was counted
        t, _ = q.next(5000)
        assert t == 4 and q.next(0) is None
        q.destroy()
    # the _format submits on every other kind of queue and mq
    for q in (api.MultiGpuQueue([0, 1], max_points=64, process_fn=FormatsBatch()),
              api.MultiGpuQueue([0, 1], max_points=64, process_fn=FormatsBatch(), records=OUSTER),
              api.ScanQueue(None, max_points=64, slots=2, max_batch=1, process_fn=FormatsBatch()),
              api.ScanQueue(None, max_points=64, slots=2, max_batch=1, process_fn=FormatsBatch(), records=OUSTER)):
        for by_ref in (False, True):
            with pytest.raises(api.UrfError) as e:
                q.submit_records(raw, 8, tag=1, timeout_ms=1000, by_reference=by_ref, fmt=0)
            assert e.value.code == URF_ERR_INVALID
        q.destroy()
    mq = formats_mq(FormatsBatch())
    for f in (lib.urf_mq_submit, lib.urf_mq_submit_ref, lib.urf_mq_submit_cloud2, lib.urf_mq_submit_cloud2_ref):
        assert f(mq._m, pts.ctypes.data, 8, 0, 1000) == URF_ERR_INVALID
    for f in (lib.urf_mq_submit_format, lib.urf_mq_submit_format_ref):
        assert f(mq._m, 0, None, 8, 0, 1000) == URF_ERR_INVALID      # NULL data
    assert mq.stats()["submitted"] == [0, 0, 0] and mq.stats()["pending"] == 0
    mq.destroy()
    for f in (lib.urf_queue_submit_format, lib.urf_mq_submit_format):
        assert f(None, 0, raw.ctypes.data, 8, 0, 1000) == URF_ERR_INVALID
    # tables: every entry passes urf_queue_create_cloud2's checks, 1..URF_MAX_FORMATS entries; policies as before
    bad_formats = [(11, 0, 4, 8, -1), (65, 0, 4, 8, -1), (48, -1, 4, 8, 16), (48, 0, 45, 8, 16), (48, 0, 4, 8, 45),
                   (22, 0, 4, 19, -1), (12, 0, 4, 8, 9)]
    dv = (C.c_int * 1)(0)
    tables = [[OUSTER, bad] for bad in bad_formats] + [[bad] for bad in bad_formats] + [[], [OUSTER] * (URF_MAX_FORMATS + 1)]
    for table in tables:
        t = api._format_array(table) if table else None
        for n in {len(table), 0}:
            assert lib.urf_queue_create_formats_with(C.byref(h), fn, None, 16, 2, 1, URF_QUEUE_BLOCK, t, n) == URF_ERR_INVALID, table
            assert lib.urf_mq_create_formats_with(C.byref(h), fn, None, 2, 16, 2, 1, URF_QUEUE_BLOCK, t, n) == URF_ERR_INVALID, table
            assert lib.urf_mq_create_formats(C.byref(h), dv, 1, 16, 2, 1, None, URF_QUEUE_BLOCK, t, n) == URF_ERR_INVALID, table
            assert lib.urf_queue_create_formats(C.byref(h), None, 16, 2, 1, URF_QUEUE_BLOCK, t, n) == URF_ERR_INVALID, table
    good = api._format_array(TABLE)
    for bad in (URF_QUEUE_DROP_OLDEST, URF_QUEUE_DROP_OLDEST | URF_QUEUE_ORDER, 8, -1):
        assert lib.urf_mq_create_formats_with(C.byref(h), fn, None, 2, 16, 2, 1, bad, good, len(TABLE)) == URF_ERR_INVALID, bad
        assert lib.urf_mq_create_formats(C.byref(h), dv, 1, 16, 2, 1, None, bad, good, len(TABLE)) == URF_ERR_INVALID, bad
    assert lib.urf_queue_create_formats_with(C.byref(h), QUEUE_PROCESS_FN(), None, 16, 2, 1, URF_QUEUE_BLOCK, good, 4) == URF_ERR_INVALID
    for table in ([OUSTER], [OUSTER] * URF_MAX_FORMATS, [(64, 52, 56, 60, 0), (12, 0, 4, 8, -1)]):
        t = api._format_array(table)
        for policy in (URF_QUEUE_BLOCK, URF_QUEUE_LABEL8 | URF_QUEUE_ORDER):
            assert lib.urf_mq_create_formats_with(C.byref(h), fn, None, 2, 16, 2, 1, policy, t, len(table)) == URF_OK
            lib.urf_mq_destroy(h)
        assert lib.urf_queue_create_formats_with(C.byref(h), fn, None, 16, 2, 1, URF_QUEUE_DROP_OLDEST, t, len(table)) == URF_OK
        lib.urf_queue_destroy(h)
    with pytest.raises(ValueError):
        api.ScanQueue(None, max_points=16, formats=TABLE, enqueue_fn=lambda *a: 0, finish_fn=lambda: 0)
    with pytest.raises(ValueError):
        api.ScanQueue(None, max_points=16, process_fn=FormatsBatch(), formats=TABLE, records=OUSTER)


@pytest.mark.parametrize("args", [("4", "1500", "3", "3", "6"), ("3", "1200", "1", "4", "2"), ("2", "2000", "2", "2", "0")])
def test_queue_formats_thread_sanitizer_stress(args):
    """urf_queue.cpp and urf_mq.cpp built with -fsanitize=thread (tests/kat/queue_formats_stress.cpp): producers x scans x
    devices x slots per device x policy bits. Every producer submits scans of the table's formats in turn, copying and by
    reference, one thread updates the parameters, one consumer takes batches; the binary checks every record the stand-in
    decoded, every payload against its tag and generation, and that batches mixed formats; TSAN that there is no data race."""
    out = subprocess.run([os.path.join(ROOT, "build", "queue_formats_stress"), *args], capture_output=True, text=True, timeout=600)
    print(out.stdout, out.stderr[-3000:])
    assert out.returncode == 0 and out.stdout.strip().endswith("OK") and "ThreadSanitizer" not in out.stderr

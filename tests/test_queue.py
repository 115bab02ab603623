"""Streaming ingest queue (include/urf.h urf_queue, SURVEY.md §8 f4): the host-side mechanics — ordering, batching,
back-pressure, the reference's drop-oldest subscriber policy (lidar_segmentation.cpp:53), close/drain, error propagation —
run here without a GPU around a stand-in batch function (urf_queue_create_with); the real thing, around urf_process_batch,
is checked against Detector.filtered on the GPU box."""
import ctypes as C
import threading
import time

import numpy as np
import pytest
import torch

from urban_road_filter_b200 import api, make_params
from urban_road_filter_b200.ctypes_abi import URF_ERR_CLOSED, URF_ERR_TIMEOUT, URF_OK, URF_QUEUE_BLOCK, URF_QUEUE_DROP_OLDEST


class FakeBatch:
    """urf_process_batch stand-in: label[i] = int(x[i]) + 1000 * (scan's first y); can be held back with `gate`."""

    def __init__(self, fail_on_batch=None):
        self.gate = threading.Event()
        self.gate.set()
        self.batches = []
        self.started = threading.Semaphore(0)
        self.fail_on_batch = fail_on_batch

    def __call__(self, user, xyzi, n, batch, outs):
        self.started.release()
        self.gate.wait()
        self.batches.append(batch)
        if self.fail_on_batch is not None and len(self.batches) - 1 == self.fail_on_batch:
            return -3
        for j in range(batch):
            pts = np.ctypeslib.as_array(C.cast(xyzi[j], C.POINTER(C.c_float)), shape=(n[j], 4)) if n[j] else np.zeros((0, 4), np.float32)
            lab = np.ctypeslib.as_array(outs[j].label, shape=(max(n[j], 1),))
            if n[j]:
                lab[: n[j]] = pts[:, 0].astype(np.int32) + 1000 * int(pts[0, 1])
            outs[j].status = 0
            outs[j].n_in = n[j]
            outs[j].n_roi = n[j]
            outs[j].n_vert = 0
        return 0


def scan(k, n=16):
    p = np.zeros((n, 4), np.float32)
    p[:, 0] = np.arange(n)
    p[:, 1] = k
    return p


def expect_labels(k, n=16):
    return np.arange(n, dtype=np.int32) + 1000 * k


def test_queue_orders_and_batches():
    fb = FakeBatch()
    q = api.ScanQueue(None, max_points=64, slots=6, max_batch=4, process_fn=fb)
    got = []
    consumer = threading.Thread(target=lambda: [got.append(q.next(5000)) for _ in range(50)])
    consumer.start()
    for k in range(50):
        assert q.submit(scan(k, 8 + k % 9), tag=k, timeout_ms=5000) == URF_OK
    consumer.join(20)
    assert not consumer.is_alive()
    assert [t for t, _ in got] == list(range(50))
    for t, r in got:
        np.testing.assert_array_equal(r.label, expect_labels(t, 8 + t % 9))
    st = q.stats()
    assert (st["submitted"], st["processed"], st["delivered"], st["dropped"], st["pending"]) == (50, 50, 50, 0, 0)
    assert 1 <= st["largest_batch"] <= 4 and sum(fb.batches) == 50 and max(fb.batches) <= 4
    assert st["most_in_flight"] == 1                              # a synchronous stand-in: one batch call at a time
    q.destroy()


def test_queue_blocks_when_full_then_resumes():
    fb = FakeBatch()
    fb.gate.clear()
    q = api.ScanQueue(None, max_points=32, slots=3, max_batch=2, policy=URF_QUEUE_BLOCK, process_fn=fb)
    for k in range(3):
        assert q.submit(scan(k), tag=k, timeout_ms=1000) == URF_OK
    t0 = time.perf_counter()
    assert q.submit(scan(3), tag=3, timeout_ms=100) == URF_ERR_TIMEOUT          # every slot taken, nothing consumed yet
    assert time.perf_counter() - t0 >= 0.09
    assert q.next(50) is None                                                    # nothing finished either
    fb.gate.set()
    assert q.next(5000)[0] == 0
    assert q.submit(scan(3), tag=3, timeout_ms=5000) == URF_OK                   # the consumed slot is free again
    assert [q.next(5000)[0] for _ in range(3)] == [1, 2, 3]
    assert q.stats()["dropped"] == 0
    q.destroy()


def test_queue_drop_oldest_like_the_reference_subscriber():
    fb = FakeBatch()
    fb.gate.clear()
    q = api.ScanQueue(None, max_points=32, slots=3, max_batch=1, policy=URF_QUEUE_DROP_OLDEST, process_fn=fb)
    assert q.submit(scan(0), tag=0) == URF_OK
    assert fb.started.acquire(timeout=5)              # scan 0 is being processed: it can no longer be dropped
    for k in (1, 2, 3, 4):                            # 1 and 2 wait; 3 replaces 1, 4 replaces 2
        assert q.submit(scan(k), tag=k, timeout_ms=1000) == URF_OK
    assert q.stats()["dropped"] == 2
    fb.gate.set()
    out = [q.next(5000) for _ in range(3)]
    assert [t for t, _ in out] == [0, 3, 4]
    for t, r in out:
        np.testing.assert_array_equal(r.label, expect_labels(t))
    st = q.stats()
    assert (st["submitted"], st["processed"], st["delivered"], st["dropped"]) == (5, 3, 3, 2)
    assert q.next(50) is None
    q.destroy()


def test_queue_many_producers_deliver_everything_once():
    fb = FakeBatch()
    q = api.ScanQueue(None, max_points=32, slots=5, max_batch=3, process_fn=fb)
    P, K = 4, 30
    got = []

    def consume():
        for _ in range(P * K):
            got.append(q.next(10000))

    def produce(p):
        for k in range(K):
            assert q.submit(scan(p * 100 + k), tag=p * 100 + k, timeout_ms=10000) == URF_OK

    threads = [threading.Thread(target=consume)] + [threading.Thread(target=produce, args=(p,)) for p in range(P)]
    for t in threads:
        t.start()
    for t in threads:
        t.join(30)
        assert not t.is_alive()
    tags = [t for t, _ in got]
    assert sorted(tags) == sorted(p * 100 + k for p in range(P) for k in range(K))
    for p in range(P):                                # per producer, results keep that producer's order
        mine = [t for t in tags if t // 100 == p]
        assert mine == sorted(mine)
    for t, r in got:
        np.testing.assert_array_equal(r.label, expect_labels(t))
    q.destroy()


def test_queue_close_drains_and_rejects():
    fb = FakeBatch()
    fb.gate.clear()
    q = api.ScanQueue(None, max_points=32, slots=4, max_batch=4, process_fn=fb)
    for k in range(3):
        assert q.submit(scan(k), tag=k) == URF_OK
    q.close()
    assert q.submit(scan(9), tag=9, timeout_ms=100) == URF_ERR_CLOSED
    fb.gate.set()
    assert [q.next(5000)[0] for _ in range(3)] == [0, 1, 2]      # what was accepted before the close is still delivered
    assert q.next(1000) is None                                   # drained: URF_ERR_CLOSED
    q.destroy()


def test_queue_reports_a_failed_batch():
    fb = FakeBatch(fail_on_batch=0)
    fb.gate.clear()
    q = api.ScanQueue(None, max_points=32, slots=4, max_batch=2, process_fn=fb)
    assert q.submit(scan(0), tag=0) == URF_OK
    assert fb.started.acquire(timeout=5)                          # batch 0 = scan 0 alone, held at the gate; it will fail
    for k in (1, 2):
        assert q.submit(scan(k), tag=k) == URF_OK
    fb.gate.set()
    with pytest.raises(api.UrfError) as e:                        # the scan of the failed batch carries its error code
        q.next(5000)
    assert e.value.code == -3
    for k in (1, 2):                                              # the queue keeps going
        t, r = q.next(5000)
        assert t == k
        np.testing.assert_array_equal(r.label, expect_labels(k))
    st = q.stats()
    assert (st["submitted"], st["processed"], st["delivered"]) == (3, 3, 3)
    q.destroy()


def test_queue_argument_checks():
    fb = FakeBatch()
    with pytest.raises(api.UrfError):
        api.ScanQueue(None, max_points=0, process_fn=fb)
    q = api.ScanQueue(None, max_points=8, slots=2, max_batch=1, process_fn=fb)
    with pytest.raises(api.UrfError) as e:
        q.submit(scan(0, 9))
    assert e.value.code == -5                                     # URF_ERR_CAPACITY
    q.destroy()


@pytest.mark.parametrize("args", [("4", "1500", "6", "4", "0"), ("8", "600", "3", "2", "0"), ("4", "1500", "4", "3", "1"),
                                  ("close", "40"), ("mq", "4", "3", "1500"), ("mq", "2", "1", "2000"), ("mq", "8", "6", "500")])
def test_queue_thread_sanitizer_stress(args):
    """urf_queue.cpp + urf_mq.cpp built with -fsanitize=thread. Plain arguments: producers x scans x slots x max_batch x
    policy; "close": the queue is closed while producers sit inside submit (nobody may hang); "mq": devices x producers x
    scans through the multi-GPU ingest around stand-in devices. The binary checks that every accepted scan is delivered
    once with its payload and per-producer order, TSAN that there is no data race."""
    import os
    import subprocess
    from util import ROOT
    out = subprocess.run([os.path.join(ROOT, "build", "queue_stress"), *args], capture_output=True, text=True, timeout=600)
    print(out.stdout, out.stderr[-3000:])
    assert out.returncode == 0 and out.stdout.strip().endswith("OK") and "ThreadSanitizer" not in out.stderr


@pytest.mark.gpu
def test_gpu_queue_streams_scans_through_the_detector():
    """Two producer threads (two LiDAR topics) stream distinct scans through urf_queue around a real context; every result
    equals what Detector.filtered gives for that scan, in per-producer order, and scans get batched while the GPU is busy."""
    from urban_road_filter_b200 import FULL_ROI
    from urban_road_filter_b200.synth import make_scan
    assert torch.cuda.is_available()
    clouds = {p * 100 + k: make_scan("C1", 40 + p * 20 + k) for p in range(2) for k in range(12)}
    n = max(c.shape[0] for c in clouds.values())
    prm = make_params(**FULL_ROI)
    ref_det = api.Detector(max_points=n, max_batch=1, params=prm)
    want = {t: ref_det.filtered(c, want_ring=False, want_order=False) for t, c in clouds.items()}
    ref_det.close()
    det = api.Detector(max_points=n, max_batch=8, params=prm)
    q = api.ScanQueue(det, max_points=n, slots=10, max_batch=8)
    got = []
    consumer = threading.Thread(target=lambda: [got.append(q.next(60000)) for _ in range(len(clouds))])
    consumer.start()

    def produce(p):
        for k in range(12):
            assert q.submit(clouds[p * 100 + k], tag=p * 100 + k, timeout_ms=60000) == URF_OK

    producers = [threading.Thread(target=produce, args=(p,)) for p in range(2)]
    for t in producers:
        t.start()
    for t in producers + [consumer]:
        t.join(120)
        assert not t.is_alive()
    tags = [t for t, _ in got]
    assert sorted(tags) == sorted(clouds)
    for p in range(2):
        mine = [t for t in tags if t // 100 == p]
        assert mine == sorted(mine)
    for t, r in got:
        w = want[t]
        assert (r.status, r.n_roi, r.n_road, r.n_curb, r.n_vert) == (w.status, w.n_roi, w.n_road, w.n_curb, w.n_vert)
        np.testing.assert_array_equal(r.label, w.label)
        np.testing.assert_array_equal(r.vert, w.vert)
    st = q.stats()
    assert (st["submitted"], st["processed"], st["delivered"], st["dropped"]) == (24, 24, 24, 0)
    q.close()
    q.destroy()
    det.close()


def test_mq_python_binding_with_stand_in_devices():
    """urf_mq through the Python binding around a Python batch function (no GPU): three stand-in devices, two producer
    threads, copying and by-reference submits; results in per-producer order, every device used."""
    seen = []

    def fake(user, xyzi, n, batch, outs):
        seen.append(batch)
        for j in range(batch):
            a = np.ctypeslib.as_array(C.cast(xyzi[j], C.POINTER(C.c_float)), shape=(max(n[j], 1) * 4,))
            lab = np.ctypeslib.as_array(outs[j].label, shape=(max(n[j], 1),))
            lab[: n[j]] = a[: 4 * n[j]: 4].astype(np.int32) + 3
            outs[j].status = 0
            outs[j].n_in = n[j]
        return 0

    mq = api.MultiGpuQueue([0, 1, 2], max_points=16, slots_per_device=2, max_batch=2, process_fn=fake)
    got = []
    cons = threading.Thread(target=lambda: [got.append(mq.next(20000)) for _ in range(40)])
    cons.start()

    def produce(p):
        for k in range(20):
            pts = np.zeros((1 + (k % 7), 4), np.float32)
            pts[:, 0] = 100 * p + k
            assert mq.submit(pts, tag=1000 * p + k, timeout_ms=20000, by_reference=bool(k & 1)) == URF_OK

    th = [threading.Thread(target=produce, args=(p,)) for p in range(2)]
    for t in th:
        t.start()
    for t in th + [cons]:
        t.join(60)
        assert not t.is_alive()
    assert all(g is not None for g in got)
    for p in range(2):
        mine = [t for t, _ in got if t // 1000 == p]
        assert mine == sorted(mine) and len(mine) == 20
    for t, r in got:
        assert r.n_in == 1 + ((t % 1000) % 7) and np.all(r.label == 100 * (t // 1000) + (t % 1000) + 3)
    st = mq.stats()
    assert st["n_devices"] == 3 and sum(st["submitted"]) == 40 and sum(st["delivered"]) == 40 and min(st["submitted"]) > 0
    mq.close()
    assert mq.next(1000) is None
    mq.destroy()


@pytest.mark.gpu
def test_gpu_mq_shards_one_stream_over_contexts():
    """urf_mq with real contexts (three on device 0 — the sharding logic is the same with one context per GPU): one
    producer streams 30 distinct scans, every result equals Detector.filtered's for that scan and arrives in order."""
    from urban_road_filter_b200 import FULL_ROI
    from urban_road_filter_b200.synth import make_scan
    assert torch.cuda.is_available()
    clouds = [make_scan("C1", 200 + k, order=("column", "ring")[k % 2]) for k in range(30)]
    n = max(c.shape[0] for c in clouds)
    prm = make_params(**FULL_ROI)
    ref = api.Detector(max_points=n, max_batch=1, params=prm)
    want = [ref.filtered(c, want_ring=False, want_order=False) for c in clouds]
    ref.close()
    mq = api.MultiGpuQueue([0, 0, 0], max_points=n, slots_per_device=4, max_batch=4, params=prm)
    got = []
    cons = threading.Thread(target=lambda: [got.append(mq.next(120000)) for _ in range(len(clouds))])
    cons.start()
    for k, c in enumerate(clouds):
        assert mq.submit(c, tag=k, timeout_ms=120000, by_reference=bool(k % 3 == 0)) == URF_OK
    cons.join(300)
    assert not cons.is_alive() and all(g is not None for g in got)
    assert [t for t, _ in got] == list(range(len(clouds)))
    for t, r in got:
        w = want[t]
        assert (r.status, r.n_roi, r.n_road, r.n_curb, r.n_vert) == (w.status, w.n_roi, w.n_road, w.n_curb, w.n_vert)
        np.testing.assert_array_equal(r.label, w.label)
        np.testing.assert_array_equal(r.vert, w.vert)
    st = mq.stats()
    assert sum(st["delivered"]) == 30 and min(st["submitted"]) > 0
    with pytest.raises(api.UrfError):
        mq.submit(clouds[0], tag=99)          # noqa: B018  (set_params below needs an idle mq; this scan is collected first)
        mq.set_params(prm)
    assert mq.next(120000) is not None
    mq.set_params(prm)
    mq.close()
    mq.destroy()

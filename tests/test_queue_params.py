"""Parameter updates on a running urf_queue / urf_mq (urf_queue_update_params, urf_mq_update_params), without a GPU: the
queues run around stand-in batch functions, and their parameter hook (urf_queue_set_params_hook) stands for the
urf_set_params_next call a real queue's worker makes. Checked here: each scan runs with the generation in force when it
was accepted, no batch mixes generations, each batch is preceded by its generation's set (field by field), batches already
in flight keep the old set, and the refusals (invalid set, closed queue). The ThreadSanitizer program
tests/kat/queue_params_stress.cpp runs the same rules with several producers and an updater at random moments."""
import ctypes as C
import os
import subprocess
import threading
import time

import numpy as np
import pytest

from urban_road_filter_b200 import api, make_params
from urban_road_filter_b200.ctypes_abi import URF_ERR_CLOSED, URF_ERR_INVALID, URF_OK, URF_QUEUE_DROP_OLDEST, UrfParams
from util import ROOT

from test_queue import expect_labels, scan
from test_queue_async import FakeDevice, hold_first_enqueue

SETS = {1: make_params(curb_points=7, min_x=-30.0), 2: make_params(star_shaped_method=0), 3: make_params(channels=16, xDirection=1)}


def same_params(a: UrfParams, b: UrfParams) -> bool:
    return all(getattr(a, f) == getattr(b, f) for f, _ in UrfParams._fields_)


class Recorder:
    """The parameter hook, and what each stand-in batch saw: its scan ids (first y of a scan) and the last hook call made on
    the calling worker thread before it (generation and a copy of the set), or None before the first."""

    def __init__(self):
        self.last = {}                                   # worker thread -> (gen, set)
        self.hooks = []                                  # (gen, set) of every hook call
        self.batches = []                                # (scan ids, (gen, set) or None)
        self.lock = threading.Lock()

    def hook(self, user, prm, gen):
        p = UrfParams.from_buffer_copy(prm.contents)
        with self.lock:
            self.last[threading.get_ident()] = (gen, p)
            self.hooks.append((gen, p))
        return URF_OK

    def saw(self, xyzi, n, batch):
        ids = [int(np.ctypeslib.as_array(C.cast(xyzi[j], C.POINTER(C.c_float)), shape=(n[j], 4))[0, 1]) for j in range(batch)]
        with self.lock:
            self.batches.append((ids, self.last.get(threading.get_ident())))


class RecordingBatch:
    """urf_process_batch stand-in (labels as test_queue.FakeBatch) that records its batches; `gate` holds it back."""

    def __init__(self, rec: Recorder):
        self.rec = rec
        self.gate = threading.Event()
        self.gate.set()
        self.started = threading.Semaphore(0)

    def __call__(self, user, xyzi, n, batch, outs):
        self.started.release()
        self.gate.wait()
        self.rec.saw(xyzi, n, batch)
        for j in range(batch):
            pts = np.ctypeslib.as_array(C.cast(xyzi[j], C.POINTER(C.c_float)), shape=(n[j], 4))
            lab = np.ctypeslib.as_array(outs[j].label, shape=(n[j],))
            lab[:] = pts[:, 0].astype(np.int32) + 1000 * int(pts[0, 1])
            outs[j].status, outs[j].n_in, outs[j].n_roi = 0, n[j], n[j]
        return 0


def check_batches(rec: Recorder, gen_of: dict):
    """Every batch holds one generation, and the last hook call before it named that generation with its set (none before a
    generation-0 batch that no update preceded)."""
    assert rec.batches
    for ids, last in rec.batches:
        gens = {gen_of[i] for i in ids}
        assert len(gens) == 1, f"batch {ids} mixes generations {gens}"
        g = gens.pop()
        if g == 0:
            assert last is None, f"batch {ids}: a hook call before a generation-0 batch"
        else:
            assert last is not None and last[0] == g, f"batch {ids}: last hook {last and last[0]}, want {g}"
            assert same_params(last[1], SETS[g]), f"batch {ids}: the hook was given another set than generation {g}'s"


def drain(q, count, label8=False):
    got = []
    while len(got) < count:
        out = q.next_batch(8, timeout_ms=5000, copy=True)
        assert out, "timed out"
        got += out
    return got


@pytest.mark.parametrize("label8", [False, True])
def test_one_producer_generations_follow_submission(label8):
    rec = Recorder()
    fb = RecordingBatch(rec)
    q = api.ScanQueue(None, max_points=32, slots=32, max_batch=4, process_fn=fb, label8=label8)
    q.set_params_hook(rec.hook)
    fb.gate.clear()                                      # scan 0 is taken alone, the rest piles up behind it
    assert q.submit(scan(0), tag=0, timeout_ms=1000) == URF_OK
    assert fb.started.acquire(timeout=5)
    for k in range(1, 10):
        assert q.submit(scan(k), tag=k, timeout_ms=1000) == URF_OK
    assert q.update_params(SETS[1]) == 1
    for k in range(10, 20):
        assert q.submit(scan(k), tag=k, timeout_ms=1000) == URF_OK
    assert q.update_params(SETS[2]) == 2
    assert q.update_params(SETS[3]) == 3                 # back to back: no scan carries generation 2
    for k in range(20, 30):
        assert q.submit(scan(k), tag=k, timeout_ms=1000) == URF_OK
    fb.gate.set()
    got = drain(q, 30, label8)
    assert [t for t, _ in got] == list(range(30))
    assert [r.params_gen for _, r in got] == [0] * 10 + [1] * 10 + [3] * 10
    for t, r in got:
        want = expect_labels(t)
        np.testing.assert_array_equal(r.label, want.astype(np.int8) if label8 else want)
    check_batches(rec, {t: r.params_gen for t, r in got})
    assert [g for g, _ in rec.hooks] == [1, 3]           # a superseded generation no scan carries is never applied
    # batches are cut at the generation changes and nowhere else: 0 | 1-4 | 5-8 | 9 | 10-13 | 14-17 | 18-19 | 20-23 | ...
    assert [ids for ids, _ in rec.batches] == [[0], [1, 2, 3, 4], [5, 6, 7, 8], [9], [10, 11, 12, 13], [14, 15, 16, 17],
                                               [18, 19], [20, 21, 22, 23], [24, 25, 26, 27], [28, 29]]
    assert same_params(q.params_of(1), SETS[1]) and same_params(q.params_of(3), SETS[3]) and q.params_of(0) is None
    q.destroy()


class ParamDevice(FakeDevice):
    """FakeDevice whose batches run with the set last given to the hook: each scan's flags report that set's generation."""

    def __init__(self, **kw):
        super().__init__(**kw)
        self.gen = 0
        self.gens = []                                   # generation of each batch in flight, oldest first

    def hook(self, user, prm, gen):
        assert same_params(prm.contents, SETS[gen])
        self.events.append(("set", gen, 0))
        self.gen = gen
        return URF_OK

    def enqueue(self, user, xyzi, n, batch, outs):
        rc = super().enqueue(user, xyzi, n, batch, outs)
        if rc == 0:
            self.gens.append(self.gen)
        return rc

    def finish(self):
        batch, outs = self.flight[0][3:5]
        rc = super().finish()
        g = self.gens.pop(0)
        for j in range(batch):
            outs[j].flags = g
        return rc


def test_update_while_two_batches_are_in_flight_leaves_them_alone():
    fd = ParamDevice(fin_permits=0)
    q = api.ScanQueue(None, enqueue_fn=fd.enqueue, finish_fn=fd.finish, max_points=32, slots=8, max_batch=2)
    q.set_params_hook(fd.hook)
    hold_first_enqueue(fd, q, [0, 1, 2])
    fd.enq_gate.set()
    deadline = time.time() + 5
    while fd.most < 2 and time.time() < deadline:       # [0] and [1, 2] enqueued, neither finished
        time.sleep(0.01)
    assert fd.most == 2
    assert q.update_params(SETS[1]) == 1
    for k in (3, 4, 5):
        assert q.submit(scan(k), tag=k, timeout_ms=1000) == URF_OK
    fd.allow(10)
    got = drain(q, 6)
    assert [t for t, _ in got] == list(range(6))
    assert [r.params_gen for _, r in got] == [0, 0, 0, 1, 1, 1]
    assert [r.flags for _, r in got] == [0, 0, 0, 1, 1, 1]      # the two batches in flight kept the old set
    for t, r in got:
        np.testing.assert_array_equal(r.label, expect_labels(t))
    # the set is applied after the first batch finished (its slot is needed) and before the new generation's batch
    ev = [e for e in fd.events]
    assert ev[:3] == [("enq", 0, 1), ("enq", 1, 2), ("fin", 0, 1)]
    assert ev[3] == ("set", 1, 0) and ev[4][0] == "enq"
    assert q.stats()["most_in_flight"] == 2
    q.destroy()


def test_invalid_set_and_closed_queue_are_refused():
    rec = Recorder()
    q = api.ScanQueue(None, max_points=16, slots=4, max_batch=2, process_fn=RecordingBatch(rec))
    for bad in (make_params(channels=0), make_params(xDirection=3), make_params(interval=float("nan")), make_params(curb_points=0)):
        with pytest.raises(api.UrfError) as e:
            q.update_params(bad)
        assert e.value.code == URF_ERR_INVALID
    assert q.submit(scan(0), tag=0, timeout_ms=1000) == URF_OK
    assert q.next(5000)[1].params_gen == 0              # nothing changed
    assert q.update_params(SETS[1]) == 1                 # the refused sets took no generation number
    assert q.submit(scan(1), tag=1, timeout_ms=1000) == URF_OK
    assert q.next(5000)[1].params_gen == 1
    q.close()
    with pytest.raises(api.UrfError) as e:
        q.update_params(SETS[2])
    assert e.value.code == URF_ERR_CLOSED
    q.destroy()
    lib = api.load_library()
    assert lib.urf_queue_update_params(None, C.byref(SETS[1])) == URF_ERR_INVALID
    assert lib.urf_mq_update_params(None, C.byref(SETS[1])) == URF_ERR_INVALID
    assert lib.urf_set_params_next(None, C.byref(SETS[1])) == URF_ERR_INVALID


def test_failed_hook_fails_its_run_and_the_next_run_applies_again():
    rec = Recorder()
    calls = []

    def hook(user, prm, gen):
        calls.append(gen)
        return -3 if len(calls) == 1 else rec.hook(user, prm, gen)

    fb = RecordingBatch(rec)
    q = api.ScanQueue(None, max_points=16, slots=8, max_batch=4, process_fn=fb)
    q.set_params_hook(hook)
    assert q.update_params(SETS[1]) == 1
    assert q.submit(scan(0), tag=0, timeout_ms=1000) == URF_OK
    t, r = drain(q, 1)[0]
    assert (t, r.status, r.params_gen, r.label) == (0, -3, 1, None)   # like a refused enqueue
    assert q.submit(scan(1), tag=1, timeout_ms=1000) == URF_OK
    t, r = drain(q, 1)[0]
    assert (t, r.status, r.params_gen) == (1, URF_OK, 1) and calls == [1, 1]
    check_batches(rec, {1: 1})
    q.destroy()


def test_drop_oldest_with_updates():
    rec = Recorder()
    fb = RecordingBatch(rec)
    fb.gate.clear()
    q = api.ScanQueue(None, max_points=16, slots=3, max_batch=1, policy=URF_QUEUE_DROP_OLDEST, process_fn=fb)
    q.set_params_hook(rec.hook)
    assert q.submit(scan(0), tag=0) == URF_OK
    assert fb.started.acquire(timeout=5)                 # 0 runs with generation 0
    assert q.submit(scan(1), tag=1, timeout_ms=1000) == URF_OK
    assert q.update_params(SETS[1]) == 1
    assert q.submit(scan(2), tag=2, timeout_ms=1000) == URF_OK
    assert q.submit(scan(3), tag=3, timeout_ms=1000) == URF_OK       # replaces 1 (generation 0)
    assert q.update_params(SETS[2]) == 2
    assert q.submit(scan(4), tag=4, timeout_ms=1000) == URF_OK       # replaces 2 (generation 1)
    assert q.stats()["dropped"] == 2
    fb.gate.set()
    got = drain(q, 3)
    assert [(t, r.params_gen) for t, r in got] == [(0, 0), (3, 1), (4, 2)]
    check_batches(rec, {0: 0, 3: 1, 4: 2})
    assert [g for g, _ in rec.hooks] == [1, 2]
    q.destroy()


@pytest.mark.parametrize("label8", [False, True])
def test_mq_update_falls_at_one_point_of_the_global_order(label8):
    rec = Recorder()
    fb = RecordingBatch(rec)
    mq = api.MultiGpuQueue([0, 1, 2], max_points=16, slots_per_device=3, max_batch=2, process_fn=fb, label8=label8)
    mq.set_params_hook(rec.hook)
    got = []
    cons = threading.Thread(target=lambda: got.extend(drain(mq, 40, label8)))
    cons.start()
    gen_at = {}
    for k in range(40):
        if k in (10, 20, 30):
            assert mq.update_params(SETS[k // 10]) == k // 10
        assert mq.submit(scan(k), tag=k, timeout_ms=5000) == URF_OK
        gen_at[k] = 0 if k < 10 else min(k // 10, 3)
    cons.join(30)
    assert not cons.is_alive()
    assert [t for t, _ in got] == list(range(40))
    gens = [r.params_gen for _, r in got]
    assert gens == sorted(gens) and gens == [gen_at[k] for k in range(40)]
    check_batches(rec, {t: r.params_gen for t, r in got})
    assert same_params(mq.params_of(2), SETS[2]) and mq.params_of(0) is None
    mq.close()
    with pytest.raises(api.UrfError) as e:
        mq.update_params(SETS[1])
    assert e.value.code == URF_ERR_CLOSED
    mq.destroy()


def test_mq_update_with_several_producers():
    """Producers keep submitting while the main thread updates: along the delivery order the generations never go back,
    and each scan's generation lies between the updates that had returned before its submit began and those that had begun
    when it returned."""
    rec = Recorder()
    fb = RecordingBatch(rec)
    mq = api.MultiGpuQueue([0, 1, 2], max_points=16, slots_per_device=4, max_batch=3, process_fn=fb)
    mq.set_params_hook(rec.hook)
    P, K = 3, 40
    bounds, begun, returned = {}, [0], [0]
    got = []
    cons = threading.Thread(target=lambda: got.extend(drain(mq, P * K)))
    cons.start()

    def produce(p):
        for k in range(K):
            tag = 1000 * p + k
            lo = returned[0]
            assert mq.submit(scan(tag % 100), tag=tag, timeout_ms=5000) == URF_OK
            bounds[tag] = (lo, begun[0])

    prods = [threading.Thread(target=produce, args=(p,)) for p in range(P)]
    for t in prods:
        t.start()
    for g in (1, 2, 3):
        time.sleep(0.02)
        begun[0] = g
        assert mq.update_params(SETS[g]) == g
        returned[0] = g
    for t in prods:
        t.join(30)
    cons.join(30)
    assert not cons.is_alive() and len(got) == P * K
    gens = [r.params_gen for _, r in got]
    assert gens == sorted(gens)
    for t, r in got:
        lo, hi = bounds[t]
        assert lo <= r.params_gen <= hi, (t, r.params_gen, lo, hi)
    mq.destroy()


def test_hooks_are_for_stand_ins_only():
    lib = api.load_library()
    assert lib.urf_queue_set_params_hook(None, api.QUEUE_PARAMS_FN(lambda u, p, g: 0)) == URF_ERR_INVALID
    assert lib.urf_mq_set_params_hook(None, api.QUEUE_PARAMS_FN(lambda u, p, g: 0)) == URF_ERR_INVALID


@pytest.mark.parametrize("args", [("4", "1500", "6", "4", "0"), ("3", "1200", "5", "2", "1"), ("2", "1500", "4", "3", "2"),
                                  ("1", "3000", "2", "1", "0")])
def test_queue_params_thread_sanitizer_stress(args):
    """urf_queue.cpp built with -fsanitize=thread (tests/kat/queue_params_stress.cpp): producers x scans x slots x max_batch
    x policy bits (1 DROP_OLDEST, 2 int8 labels), one thread updating at random, some hook calls failing. The binary checks
    that no batch mixes generations, every scan carries the generation in force when it was accepted, and one producer's
    generations never go back; TSAN that there is no data race."""
    out = subprocess.run([os.path.join(ROOT, "build", "queue_params_stress"), *args], capture_output=True, text=True, timeout=600)
    print(out.stdout, out.stderr[-3000:])
    assert out.returncode == 0 and out.stdout.strip().endswith("OK") and "ThreadSanitizer" not in out.stderr

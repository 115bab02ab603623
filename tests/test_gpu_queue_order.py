"""The emission order through the streaming queues on the H100 (URF_QUEUE_ORDER): every result a urf_queue or urf_mq
delivers — labels, order[:n_order], ring_start[:n_rings + 1], counts, flags and vertices — equals, bit for bit, the
synchronous Detector.filtered_batch(want_order=True) of the same scan with the same parameters. Covered: float4 queues with
int32 and int8 label slots and 48-byte PointCloud2 record queues, small batches (CUDA-graph path) and batches above 8
(chunked path), urf_queue_next into caller buffers and urf_queue_next_batch views, the mq over every visible GPU, the golden
fixtures of the unmodified reference (road / curb / road_probably clouds and marker strips), the reference tie order, a
mid-stream update that changes channels and the ROI, and a scan with too few points in the stream."""
import ctypes as C
import threading

import numpy as np
import pytest
import torch

from urban_road_filter_b200 import FULL_ROI, api, make_params
from urban_road_filter_b200.ctypes_abi import URF_MAX_CHANNELS, URF_OK, URF_QUEUE_LABEL8, URF_QUEUE_ORDER, URF_TOO_FEW_POINTS
from urban_road_filter_b200.synth import SHAPES, make_scan
from util import Golden, assert_matches_golden, cloud2_records, golden_names

from test_gpu_reference_ties import NAMES as TIE_NAMES, _ties_fixture, check as check_ties, check_reference, expect, port  # noqa: F401

pytestmark = pytest.mark.gpu

FULL = make_params(**FULL_ROI)
REC48 = (48, (0, 4, 8, 16))           # Ouster records: x, y, z, intensity at 0, 4, 8, 16
FIELDS = ("status", "n_in", "n_roi", "n_rings", "n_order", "n_road", "n_curb", "n_vert", "flags")


def mixed_scans(count, seed, tiny_at=()):
    """C1 and C2 scans in turn, column- and ring-major, each with its own size; the scans at tiny_at keep 20 points (too
    few for the ROI: URF_TOO_FEW_POINTS)."""
    out = []
    for k in range(count):
        shape = ("C1", "C2")[k % 2]
        c = make_scan(shape, seed + k, order=("column", "ring")[(k // 2) % 2], cols=SHAPES[shape].cols - 7 * k)
        out.append(c[:20].copy() if k in tiny_at else c)
    return out


def reference(clouds, prm, tie="input"):
    """The synchronous call on a fresh context, one scan at a time: labels, order, ring_start, counts, flags, vertices."""
    det = api.Detector(max_points=max(c.shape[0] for c in clouds), max_batch=1, params=prm, tie_order=tie)
    out = [det.filtered_batch([c], want_ring=False, want_order=True)[0] for c in clouds]
    det.close()
    return out


def same(r, w, what):
    """r (queue) equals w (synchronous call) bit for bit; int8 labels compare by value."""
    for f in FIELDS:
        assert getattr(r, f) == getattr(w, f), f"{what}: {f} {getattr(r, f)} != {getattr(w, f)}"
    np.testing.assert_array_equal(r.label.astype(np.int32), w.label, err_msg=f"{what}: labels")
    assert r.order is not None and r.ring_start is not None, what
    assert r.order.dtype == np.int32 and r.order.tobytes() == w.order.tobytes(), f"{what}: emission order"
    assert r.ring_start.tobytes() == w.ring_start.tobytes(), f"{what}: ring_start"
    assert r.vert.tobytes() == w.vert.tobytes(), f"{what}: vertices"


class RecordQueue(api._StreamQueue):
    """urf_queue_create_cloud2 / urf_queue_submit_cloud2 behind the shared queue wrapper (next / next_batch)."""
    _PREFIX = "urf_queue_"

    def __init__(self, det, max_points, slots, max_batch, step, offs, label8=True):
        super().__init__(max_points, label8, det.params, order=True)
        self._det = det
        policy = URF_QUEUE_ORDER | (URF_QUEUE_LABEL8 if label8 else 0)
        rc = self.lib.urf_queue_create_cloud2(C.byref(self._h), det._ctx, max_points, slots, max_batch, policy, step, *offs)
        assert rc == URF_OK

    def submit_records(self, raw, n, tag, timeout_ms=-1):
        return self._call("submit_cloud2", raw.ctypes.data, n, tag, timeout_ms)

    def stats(self):
        return api.ScanQueue.stats(self)


def consume(q, count, use_next, check, timeout_s=300):
    """Consumer thread: takes `count` results (next, or next_batch views checked before the next call gives them back) and
    passes each to check(tag, result). Returns the thread and the list that receives its first exception."""
    err = []

    def run():
        try:
            seen = 0
            while seen < count:
                if use_next:
                    got = q.next(timeout_s * 1000)
                    assert got is not None, "timed out"
                    out = [got]
                else:
                    out = q.next_batch(8, timeout_s * 1000)
                    assert out, "timed out"
                for t, r in out:
                    check(t, r)
                seen += len(out)
        except BaseException as e:                        # noqa: BLE001 — re-raised in the main thread
            err.append(e)

    th = threading.Thread(target=run)
    th.start()
    return th, err


def finish(th, err, timeout_s=600):
    th.join(timeout_s)
    assert not th.is_alive(), "consumer did not finish"
    if err:
        raise err[0]


# (kind, int8 label slots): float4 / int32, float4 / int8, 48-byte records / int8
KINDS = [("float4", False), ("float4", True), ("rec48", True)]


@pytest.mark.parametrize("max_batch", [4, 16])
@pytest.mark.parametrize("kind,label8", KINDS)
def test_gpu_queue_order_matches_the_synchronous_call(kind, label8, max_batch):
    count = 40
    clouds = mixed_scans(count, 300 + max_batch, tiny_at=(7,))
    want = reference(clouds, FULL)
    n = max(c.shape[0] for c in clouds)
    det = api.Detector(max_points=n, max_batch=max_batch, params=FULL)
    if kind == "float4":
        q = api.ScanQueue(det, max_points=n, slots=count, max_batch=max_batch, label8=label8, order=True)
    else:
        step, offs = REC48
        raws = [cloud2_records(c, step, *offs, seed=k) for k, c in enumerate(clouds)]
        q = RecordQueue(det, n, count, max_batch, step, offs, label8)
    use_next = kind == "float4" and not label8                  # next into the caller's buffers; views otherwise
    th, err = consume(q, count, use_next, lambda t, r: same(r, want[t], f"{kind} label8={label8} scan {t}"))
    for k, c in enumerate(clouds):
        if kind == "float4":
            assert q.submit(c, tag=k, timeout_ms=300_000, by_reference=True) == URF_OK
        else:
            assert q.submit_records(raws[k], c.shape[0], k, 300_000) == URF_OK
    finish(th, err)
    st = q.stats()
    print(kind, label8, max_batch, st)
    assert (st["submitted"], st["processed"], st["delivered"], st["dropped"]) == (count, count, count, 0)
    assert want[7].status == URF_TOO_FEW_POINTS
    if max_batch > 8 and kind == "float4":                     # by-reference submits outrun the device: big batches
        assert st["largest_batch"] > 8
    q.close()
    q.destroy()
    det.close()


@pytest.mark.parametrize("label8", [False, True])
def test_gpu_mq_order_on_every_gpu(label8):
    devices = list(range(torch.cuda.device_count()))
    devices = devices if len(devices) > 1 else [0, 0]
    count = 36
    clouds = mixed_scans(count, 900, tiny_at=(11,))
    want = reference(clouds, FULL)
    n = max(c.shape[0] for c in clouds)
    mq = api.MultiGpuQueue(devices, max_points=n, slots_per_device=6, max_batch=4, params=FULL, label8=label8, order=True)
    th, err = consume(mq, count, not label8, lambda t, r: same(r, want[t], f"mq label8={label8} scan {t}"))
    for k, c in enumerate(clouds):
        assert mq.submit(c, tag=k, timeout_ms=300_000, by_reference=bool(k % 2)) == URF_OK
    finish(th, err)
    st = mq.stats()
    assert sum(st["delivered"]) == count and all(d > 0 for d in st["delivered"]), st
    mq.close()
    mq.destroy()


def test_gpu_queue_order_reproduces_the_reference_goldens():
    """Every fixture the queue can hold (all but the 1M-point C5 ones), each under its own parameters through a mid-stream
    update of one ORDER queue: labels, the road / curb / road_probably clouds the unmodified reference published, and its
    marker strips (through the parameter set the result's params_gen names)."""
    names = [nm for nm in golden_names() if not nm.startswith("c5_")]
    goldens = [Golden(nm) for nm in names]
    n = max(g.cloud.shape[0] for g in goldens)
    det = api.Detector(max_points=n, max_batch=4, params=FULL)
    q = api.ScanQueue(det, max_points=n, slots=4, max_batch=4, label8=True, order=True)
    checked = []

    def check(t, r):
        g = goldens[t]
        prm = q.params_of(r.params_gen)
        assert bytes(prm) == bytes(g.params()), g.name
        assert_matches_golden(g, r, api.build_markers)
        if g.published and not r.flags & 4:
            assert np.array_equal(r.cloud_indices("road"), g.road_ids) and np.array_equal(r.cloud_indices("curb"), g.curb_ids)
            assert np.array_equal(r.cloud_indices("road_probably"), g.prob_ids), g.name
        checked.append(g.name)

    th, err = consume(q, len(goldens), False, lambda t, r: check(t, _widened(r)))
    for k, g in enumerate(goldens):
        assert q.update_params(g.params()) == k + 1
        assert q.submit(g.cloud, tag=k, timeout_ms=300_000) == URF_OK
    finish(th, err)
    assert checked == names
    q.close()
    q.destroy()
    det.close()


def _widened(r):
    """The result with int32 labels (assert_matches_golden compares them with np.array_equal against int32)."""
    if r.label is not None:
        r.label = r.label.astype(np.int32)
    return r


def test_gpu_queue_order_in_the_reference_tie_order(port):    # noqa: F811 — the module fixture of the ties tests
    """The tie clouds of tests/tie_policy.py through an ORDER queue on a context in the reference tie order: what the CPU
    oracle (the reference's Lomuto order) and the unmodified reference published, as for the synchronous entry points."""
    cases = [(nm, *expect(port, nm)) for nm in TIE_NAMES]
    n = max(pts.shape[0] for _, pts, _, _ in cases)
    det = api.Detector(max_points=n, max_batch=2, params=cases[0][2], tie_order="reference")
    q = api.ScanQueue(det, max_points=n, slots=4, max_batch=2, order=True)
    meta, arrays = _ties_fixture()

    def check(t, r):
        nm, pts, prm, o = cases[t]
        check_ties(r, o, nm + " (queue)", ring=False)
        check_reference(r, pts, prm, meta[nm], arrays, nm)

    th, err = consume(q, len(cases), True, check)
    for k, (nm, pts, prm, _) in enumerate(cases):
        q.update_params(prm)
        assert q.submit(pts, tag=k, timeout_ms=300_000) == URF_OK
    finish(th, err)
    q.close()
    q.destroy()
    det.close()


@pytest.mark.parametrize("label8", [False, True])
def test_gpu_queue_order_across_a_channels_and_roi_update(label8):
    """A running ORDER queue whose parameters change twice: ROI and channels 64 -> 16 (the default ROI), then back to the full
    ROI with channels 32. Every result equals a fresh synchronous run with its own generation's set."""
    sets = [FULL, make_params(channels=16), make_params(**FULL_ROI, channels=32)]
    count, at = 30, (10, 20)
    clouds = mixed_scans(count, 500, tiny_at=(25,))
    gen_of = [sum(k >= a for a in at) for k in range(count)]
    want = {g: reference(clouds, sets[g]) for g in range(3)}
    n = max(c.shape[0] for c in clouds)
    det = api.Detector(max_points=n, max_batch=4, params=FULL)
    q = api.ScanQueue(det, max_points=n, slots=8, max_batch=4, label8=label8, order=True)

    def check(t, r):
        assert r.params_gen == gen_of[t], (t, r.params_gen)
        same(r, want[gen_of[t]][t], f"scan {t} generation {gen_of[t]}")

    th, err = consume(q, count, not label8, check)
    for k, c in enumerate(clouds):
        if k in at:
            assert q.update_params(sets[at.index(k) + 1]) == at.index(k) + 1
        assert q.submit(c, tag=k, timeout_ms=300_000) == URF_OK
    finish(th, err)
    assert want[1][0].n_rings != want[0][0].n_rings or want[1][0].n_roi != want[0][0].n_roi   # the sets do differ
    q.close()
    q.destroy()
    det.close()


def test_gpu_queue_order_too_few_points():
    """A scan with URF_TOO_FEW_POINTS between published ones: n_order 0, its slot's ring_start all zeros, its neighbours
    unaffected."""
    clouds = mixed_scans(3, 77, tiny_at=(1,))
    want = reference(clouds, FULL)
    n = max(c.shape[0] for c in clouds)
    det = api.Detector(max_points=n, max_batch=4, params=FULL)
    q = api.ScanQueue(det, max_points=n, slots=4, max_batch=4, label8=True, order=True)
    for k, c in enumerate(clouds):
        assert q.submit(c, tag=k, timeout_ms=300_000) == URF_OK
    got = []
    while len(got) < 3:
        out = q.next_batch(3, 300_000)
        assert out
        for t, r in out:                                          # views: checked before the next call
            same(r, want[t], f"scan {t}")
            if t == 1:
                assert r.status == URF_TOO_FEW_POINTS and r.n_order == 0 and r.order.size == 0
                full = np.ctypeslib.as_array(C.cast(r.ring_start.ctypes.data, C.POINTER(C.c_int32)), shape=(URF_MAX_CHANNELS + 1,))
                assert not full.any()
        got += [t for t, _ in out]
    assert got == [0, 1, 2]
    q.close()
    q.destroy()
    det.close()

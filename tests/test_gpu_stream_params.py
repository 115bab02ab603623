"""Parameter updates with batches in flight, on the H100: urf_set_params_next between two enqueued batches, and
urf_queue_update_params / urf_mq_update_params on running queues. Every result is compared, bit for bit, with a fresh
synchronous Detector run with its generation's parameters (labels, counts, flags, vertices, and ring / order / ring_start
where asked for), and carries that generation in params_gen. The parameter pairs change the launch itself: the ROI,
the star-shaped search off, x-zero off, curb_points 5 -> 7 (k_ring_detect4 -> k_ring_detect), channels 64 -> 16 (grids and
ring caps), blind_spots and xDirection."""
import threading

import numpy as np
import pytest
import torch

from urban_road_filter_b200 import FULL_ROI, api, make_params

from test_gpu_async_batches import Batch, assert_same, scans

pytestmark = pytest.mark.gpu

FULL = make_params(**FULL_ROI)
SETS = {
    "default": make_params(),
    "full": FULL,
    "star_off": make_params(**FULL_ROI, star_shaped_method=0),
    "xzero_off": make_params(**FULL_ROI, x_zero_method=0),
    "curb7": make_params(**FULL_ROI, curb_points=7),
    "ch16": make_params(**FULL_ROI, channels=16),
    "blind_xdir": make_params(**FULL_ROI, blind_spots=0, xDirection=1),
}

# (shape, input, int8 labels, ring + order wanted, (batch A, batch B), set of A, set of B). A and B of up to 8 scans take the
# CUDA-graph path of slot 0 (B runs in slot 1, and C, which is A again, re-captures the graph while B is in flight); 24
# scans the chunked pipeline
CASES = [
    ("C1", "float4", False, True, (8, 8), "default", "full"),
    ("C2", "rec48", False, True, (24, 24), "full", "ch16"),
    ("C1", "float4", False, True, (1, 8), "full", "star_off"),
    ("C4", "rec22", True, False, (8, 24), "full", "xzero_off"),
    ("C1", "rec22", True, True, (24, 8), "full", "curb7"),
    ("C2", "float4", False, True, (8, 24), "full", "blind_xdir"),
    ("C2", "float4", True, True, (8, 8), "ch16", "full"),
]


def reference(batch, prm, tie, n):
    """The synchronous call with `prm` on a fresh context: its results and its launch count."""
    det = api.Detector(max_points=n, max_batch=24, params=prm, tie_order=tie)
    out = batch.sync(det)
    launches = det.last_launch_count()
    det.close()
    return out, launches


@pytest.mark.parametrize("tie", ["input", "reference"])
@pytest.mark.parametrize("shape,kind,label8,want,sizes,pa,pb", CASES)
def test_gpu_set_params_next_between_batches_in_flight(shape, kind, label8, want, sizes, pa, pb, tie):
    assert torch.cuda.is_available()
    A = Batch(scans(shape, sizes[0], 100, 48), kind, label8, want)
    B = Batch(scans(shape, sizes[1], 300, 96, cut0=5), kind, label8, want)
    n = max(c.shape[0] for c in A.clouds + B.clouds)
    want_a, launches_a = reference(A, SETS[pa], tie, n)
    want_b, launches_b = reference(B, SETS[pb], tie, n)

    det = api.Detector(max_points=n, max_batch=24, params=SETS[pa], tie_order=tie)
    ha, hb, hc = A.handle(), B.handle(), A.handle()
    det.enqueue(ha)                                                # slot 0, set A
    assert det.set_params_next(SETS[pb]) == 1                      # while A is in flight
    det.enqueue(hb)                                                # slot 1, set B
    assert det.finish_batch() is ha
    assert det.last_launch_count() == launches_a
    assert det.set_params_next(SETS[pa]) == 2                      # while B is in flight
    det.enqueue(hc)                                                # slot 0 again: the graph is captured anew for set A
    assert det.finish_batch() is hb
    assert det.last_launch_count() == launches_b
    assert det.finish_batch() is hc
    assert det.last_launch_count() == launches_a
    assert_same(ha.results, want_a, f"{shape} {kind} A ({pa})")
    assert_same(hb.results, want_b, f"{shape} {kind} B ({pb})")
    assert_same(hc.results, want_a, f"{shape} {kind} C ({pa})")
    assert [r.params_gen for r in ha.results] == [0] * sizes[0]
    assert [r.params_gen for r in hb.results] == [1] * sizes[1]
    assert [r.params_gen for r in hc.results] == [2] * sizes[0]
    # the synchronous calls take the new set too, and report its generation
    assert det.set_params_next(SETS[pb]) == 3
    got = B.sync(det)
    assert_same(got, want_b, f"{shape} {kind} B synchronous")
    assert all(r.params_gen == 3 for r in got)
    det.set_params(SETS[pa])                                       # idle: the plain setter; the generation stays
    got = A.sync(det)
    assert_same(got, want_a, f"{shape} {kind} A after urf_set_params")
    assert all(r.params_gen == 3 for r in got)
    det.close()


# (submit count at which the update is made, set): the stream starts with "full"
SCHEDULE = [(10, "default"), (20, "curb7"), (30, "ch16")]


def stream_expectations(shape, count):
    clouds = scans(shape, count, 900, 64)
    n = max(c.shape[0] for c in clouds)
    names = ["full"] + [s for _, s in SCHEDULE]
    refs = {}
    for name in names:
        det = api.Detector(max_points=n, max_batch=1, params=SETS[name])
        refs[name] = [det.filtered(c, want_ring=False, want_order=False) for c in clouds]
        det.close()

    def gen_of(k):
        return sum(k >= at for at, _ in SCHEDULE)

    return clouds, n, refs, names, gen_of


def run_stream(q, clouds, timeout_s=300):
    """A producer thread submits the scans; the main thread makes each update of SCHEDULE once the producer has submitted
    exactly that many scans (the producer waits for it), while the consumer thread collects the results."""
    count = len(clouds)
    got = []
    reached = {at: threading.Event() for at, _ in SCHEDULE}
    updated = {at: threading.Event() for at, _ in SCHEDULE}

    def produce():
        for k, c in enumerate(clouds):
            if k in reached:
                reached[k].set()
                assert updated[k].wait(timeout_s)
            assert q.submit(c, tag=k, timeout_ms=timeout_s * 1000, by_reference=bool(k % 2)) == api.URF_OK

    def consume():
        while len(got) < count:
            out = q.next_batch(8, timeout_s * 1000, copy=True)
            assert out
            got.extend(out)

    threads = [threading.Thread(target=produce), threading.Thread(target=consume)]
    for t in threads:
        t.start()
    for g, (at, name) in enumerate(SCHEDULE, start=1):
        assert reached[at].wait(timeout_s)
        assert q.update_params(SETS[name]) == g
        updated[at].set()
    for t in threads:
        t.join(timeout_s)
    assert not any(t.is_alive() for t in threads)
    return got


def check_stream(got, refs, names, gen_of, q):
    assert [t for t, _ in got] == list(range(len(got)))
    for t, r in got:
        g = gen_of(t)
        assert r.params_gen == g, (t, r.params_gen, g)
        w = refs[names[g]][t]
        assert (r.status, r.n_in, r.n_roi, r.n_rings, r.n_order, r.n_road, r.n_curb, r.n_vert, r.flags) == \
               (w.status, w.n_in, w.n_roi, w.n_rings, w.n_order, w.n_road, w.n_curb, w.n_vert, w.flags), (t, names[g])
        np.testing.assert_array_equal(r.label.astype(np.int32), w.label)
        assert r.vert.tobytes() == w.vert.tobytes(), (t, names[g])
        prm = q.params_of(g)
        assert prm is not None and bytes(prm) == bytes(SETS[names[g]])


@pytest.mark.parametrize("label8", [False, True])
@pytest.mark.parametrize("shape", ["C1", "C2"])
def test_gpu_scan_queue_updates_on_a_running_stream(shape, label8):
    clouds, n, refs, names, gen_of = stream_expectations(shape, 40)
    det = api.Detector(max_points=n, max_batch=4, params=FULL)
    q = api.ScanQueue(det, max_points=n, slots=8, max_batch=4, label8=label8)
    got = run_stream(q, clouds)
    check_stream(got, refs, names, gen_of, q)
    st = q.stats()
    assert (st["submitted"], st["processed"], st["delivered"], st["dropped"]) == (40, 40, 40, 0)
    q.close()
    q.destroy()
    det.close()


@pytest.mark.parametrize("shape", ["C1", "C2"])
def test_gpu_mq_updates_on_a_running_stream(shape):
    clouds, n, refs, names, gen_of = stream_expectations(shape, 40)
    mq = api.MultiGpuQueue([0, 0, 0], max_points=n, slots_per_device=4, max_batch=3, params=FULL)
    got = run_stream(mq, clouds)
    check_stream(got, refs, names, gen_of, mq)
    assert bytes(mq.params_of(0)) == bytes(FULL)
    mq.close()
    mq.destroy()

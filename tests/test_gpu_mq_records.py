"""PointCloud2 records through the multi-GPU queue on the H100 (urf_mq_create_cloud2, urf_mq_submit_cloud2[_ref]): every
result a record mq delivers — labels (int32 and int8 slots), counts, flags, vertices, params_gen and, with URF_QUEUE_ORDER,
order[:n_order] and ring_start[:n_rings + 1] — equals, bit for bit, the synchronous Detector.filtered_batch_records of the
same records with the same parameters, and what a float4 mq fed the same points delivers. Covered: 48-byte Ouster records
(intensity at 16) and 32-byte Velodyne-like records, copying and by-reference submits, batches on the CUDA-graph path and
on the chunked path (more than 8 scans pending), next into caller buffers and next_batch views, a mid-stream update that
changes channels and the ROI, a scan with too few points, the reference tie order, and a golden fixture of the unmodified
reference. All visible GPUs; with one GPU, two device queues on it."""
import numpy as np
import pytest
import torch

from urban_road_filter_b200 import FULL_ROI, api, make_params
from urban_road_filter_b200.ctypes_abi import URF_OK, URF_TOO_FEW_POINTS
from util import Golden, assert_matches_golden, cloud2_records

from test_gpu_queue_order import FIELDS, consume, finish, mixed_scans, same
from test_gpu_reference_ties import NAMES as TIE_NAMES, _ties_fixture, check as check_ties, check_reference, expect, port  # noqa: F401

pytestmark = pytest.mark.gpu

FULL = make_params(**FULL_ROI)
FORMATS = {"rec48": (48, 0, 4, 8, 16),      # Ouster: x, y, z, intensity at 0, 4, 8, 16
           "rec32": (32, 0, 4, 8, 16)}      # Velodyne-like: x, y, z at 0, 4, 8, intensity at 16, ring and time after it


def devices():
    n = torch.cuda.device_count()
    return list(range(n)) if n > 1 else [0, 0]


def reference_records(raws, fmt, prm, tie="input"):
    """The synchronous record call on a fresh context, one scan at a time, with the emission order."""
    step = fmt[0]
    det = api.Detector(max_points=max(r.size // step for r in raws), max_batch=1, params=prm, tie_order=tie)
    out = [det.filtered_batch_records([r], *fmt, want_order=True, label8=False)[0] for r in raws]
    det.close()
    return out


def snapshot(r):
    """A copy of a (possibly lent) result that outlives the next delivery call."""
    c = api.ScanResult()
    for f in FIELDS + ("params_gen",):
        setattr(c, f, getattr(r, f))
    c.label = r.label.astype(np.int32)
    c.ring = None
    c.order, c.ring_start, c.vert = r.order.copy(), r.ring_start.copy(), r.vert.copy()
    return c


# (records, int8 label slots, max_batch): every format with both slot kinds and both batch paths
CASES = [("rec48", True, 16), ("rec48", False, 4), ("rec32", True, 4), ("rec32", False, 16)]


@pytest.mark.parametrize("kind,label8,max_batch", CASES)
def test_gpu_record_mq_matches_the_synchronous_call_and_a_float4_mq(kind, label8, max_batch):
    """48 scans, the one at 7 with too few points; at scan 32 an update to channels 16 and the default ROI. The float4 mq gets
    the same points by reference. Record submits are by reference too with max_batch 16, so that scans pile up behind the
    devices and batches take the chunked path; with max_batch 4 every fourth one is a copying submit."""
    fmt = FORMATS[kind]
    count, at = 48, 32
    sets = [FULL, make_params(channels=16)]
    clouds = mixed_scans(count, 700 + max_batch, tiny_at=(7,))
    raws = [cloud2_records(c, *fmt, seed=k) for k, c in enumerate(clouds)]
    gen_of = [int(k >= at) for k in range(count)]
    want = {g: reference_records(raws, fmt, sets[g]) for g in (0, 1)}
    assert want[0][7].status == URF_TOO_FEW_POINTS
    assert want[1][0].n_rings != want[0][0].n_rings or want[1][0].n_roi != want[0][0].n_roi    # the sets do differ
    n = max(c.shape[0] for c in clouds)
    got = {}
    for feed in ("records", "float4"):
        mq = api.MultiGpuQueue(devices(), max_points=n, slots_per_device=count, max_batch=max_batch, params=FULL, label8=label8,
                               order=True, records=fmt if feed == "records" else None)
        got[feed] = {}

        def check(t, r, feed=feed):
            assert r.params_gen == gen_of[t], (feed, t, r.params_gen)
            same(r, want[gen_of[t]][t], f"{feed} {kind} label8={label8} scan {t}")
            got[feed][t] = snapshot(r)

        th, err = consume(mq, count, not label8, check)     # next into the wrapper's buffers, or next_batch views
        for k, c in enumerate(clouds):
            if k == at:
                assert mq.update_params(sets[1]) == 1
            if feed == "records":
                assert mq.submit_records(raws[k], c.shape[0], tag=k, timeout_ms=300_000, by_reference=max_batch > 8 or k % 4 != 3) == URF_OK
            else:
                assert mq.submit(c, tag=k, timeout_ms=300_000, by_reference=True) == URF_OK
        finish(th, err)
        st = mq.stats()
        print(feed, kind, label8, max_batch, st)
        assert sum(st["delivered"]) == count and all(d > 0 for d in st["delivered"]), st
        if max_batch > 8:                                   # by-reference submits outrun the devices: chunked-path batches
            assert max(st["largest_batch"]) > 8, st
        mq.close()
        mq.destroy()
    for t in range(count):                                  # the record mq and the float4 mq agree scan by scan
        same(got["records"][t], got["float4"][t], f"{kind} label8={label8} scan {t}: records against float4")
        assert got["records"][t].params_gen == got["float4"][t].params_gen


def test_gpu_record_mq_in_the_reference_tie_order(port):    # noqa: F811 — the module fixture of the ties tests
    """The tie clouds of tests/tie_policy.py as 32-byte records through a record mq in the reference tie order: what the CPU
    oracle (the reference's Lomuto order) and the unmodified reference published."""
    fmt = FORMATS["rec32"]
    cases = [(nm, *expect(port, nm)) for nm in TIE_NAMES]
    n = max(pts.shape[0] for _, pts, _, _ in cases)
    mq = api.MultiGpuQueue(devices(), max_points=n, slots_per_device=4, max_batch=2, params=cases[0][2], order=True, records=fmt)
    mq.set_tie_order("reference")
    meta, arrays = _ties_fixture()

    def check(t, r):
        nm, pts, prm, o = cases[t]
        assert r.params_gen == t + 1
        check_ties(r, o, nm + " (record mq)", ring=False)
        check_reference(r, pts, prm, meta[nm], arrays, nm)

    th, err = consume(mq, len(cases), True, check)
    for k, (nm, pts, prm, _) in enumerate(cases):
        assert mq.update_params(prm) == k + 1
        assert mq.submit_records(cloud2_records(pts, *fmt, seed=k), pts.shape[0], tag=k, timeout_ms=300_000) == URF_OK
    finish(th, err)
    mq.close()
    mq.destroy()


def test_gpu_record_mq_reproduces_a_golden_fixture():
    """c2_default_s0 as 48-byte records, by reference, next to two scans of other sets: labels, the road / curb /
    road_probably clouds and the marker strips the unmodified reference published."""
    fmt = FORMATS["rec48"]
    g = Golden("c2_default_s0")
    other = mixed_scans(2, 40)
    clouds = [other[0], g.cloud, other[1]]
    raws = [cloud2_records(c, *fmt, seed=k) for k, c in enumerate(clouds)]
    n = max(c.shape[0] for c in clouds)
    mq = api.MultiGpuQueue(devices(), max_points=n, slots_per_device=4, max_batch=4, params=FULL, label8=True, order=True,
                           records=fmt)
    for k, c in enumerate(clouds):
        if k == 1:
            assert mq.update_params(g.params()) == 1
        if k == 2:
            assert mq.update_params(FULL) == 2
        assert mq.submit_records(raws[k], c.shape[0], tag=k, timeout_ms=300_000, by_reference=True) == URF_OK
    seen = []
    while len(seen) < 3:
        out = mq.next_batch(3, 300_000)
        assert out
        for t, r in out:                                    # views: checked before the next call
            seen.append(t)
            if t != 1:
                continue
            assert bytes(mq.params_of(r.params_gen)) == bytes(g.params())
            r.label = r.label.astype(np.int32)
            assert_matches_golden(g, r, api.build_markers)
            if g.published and not r.flags & 4:
                assert np.array_equal(r.cloud_indices("road"), g.road_ids) and np.array_equal(r.cloud_indices("curb"), g.curb_ids)
                assert np.array_equal(r.cloud_indices("road_probably"), g.prob_ids)
    assert seen == [0, 1, 2]
    mq.close()
    mq.destroy()

"""PointCloud2 records of several sensor formats in one batch and one stream on the H100 (urf_process_cloud2_batch_mixed,
urf_enqueue_cloud2_batch_mixed, urf_queue_create_formats, urf_mq_create_formats). Every result of a mixed batch — labels
(int32 and int8), ring, order, ring_start, counts, flags, vertices, params_gen — equals, bit for bit, the synchronous
filtered_batch_records of that scan alone in its own format, and `filtered` of its float4 points. Covered: 48-byte Ouster
(intensity at 16), 32-byte and packed 22-byte Velodyne, 16-byte float4 and 12-byte xyz records in one batch, on the
CUDA-graph path and on the chunked path; two mixed batches in flight from pinned buffers; both tie orders on dual-return
and duplicate-point tie clouds; a golden fixture carried in two formats; a batch whose largest point_step makes the record
staging grow; the launch count of a mixed batch; and a formats ScanQueue and MultiGpuQueue (int8 slots, URF_QUEUE_ORDER,
all visible GPUs) across a channels and ROI update."""
import numpy as np
import pytest
import torch

from urban_road_filter_b200 import FULL_ROI, api, make_params
from urban_road_filter_b200.ctypes_abi import URF_OK
from util import Golden, assert_matches_golden, cloud2_records

from test_gpu_queue_order import FIELDS, consume, finish, mixed_scans, same
from test_gpu_reference_ties import check as check_ties, expect, port  # noqa: F401

pytestmark = pytest.mark.gpu

FULL = make_params(**FULL_ROI)
OS48 = api.CloudFormat(48, 0, 4, 8, 16)          # Ouster: x, y, z, intensity at 0, 4, 8, 16
V32 = api.CloudFormat(32, 0, 4, 8, 16)           # Velodyne-like, ring and time after the intensity
V22 = api.CloudFormat(22, 0, 4, 8, 12)           # packed Velodyne: records are not 4-byte aligned
XYZ = api.CloudFormat(12, 0, 4, 8, -1)           # bare x, y, z: no intensity
TABLE = [OS48, V32, V22, api.FLOAT4_FORMAT, XYZ]


def devices():
    n = torch.cuda.device_count()
    return list(range(n)) if n > 1 else [0, 0]


def as_records(clouds, fmts):
    return [cloud2_records(c, *f, seed=k) for k, (c, f) in enumerate(zip(clouds, fmts))]


def unpacked(c, f):
    """The float4 points the device unpacks from c's records in format f (intensity 0 without an intensity field)."""
    p = np.ascontiguousarray(c, np.float32).copy()
    if f.off_intensity < 0:
        p[:, 3] = 0
    return p


def full_same(r, w, what, ring=True):
    same(r, w, what)
    if ring:
        assert r.ring.tobytes() == w.ring.tobytes(), f"{what}: ring"
    assert r.params_gen == w.params_gen, what


def alone(clouds, raws, fmts, prm, label8, tie="input"):
    """Each scan alone on a fresh context: filtered_batch_records in its own format, and filtered on its float4 points."""
    det = api.Detector(max_points=max(c.shape[0] for c in clouds), max_batch=1, params=prm, tie_order=tie)
    rec = [det.filtered_batch_records([r], *f, want_order=True, label8=label8, want_ring=True)[0] for r, f in zip(raws, fmts)]
    f4 = [det.filtered(unpacked(c, f)) for c, f in zip(clouds, fmts)]
    det.close()
    return rec, f4


@pytest.mark.parametrize("batch,label8", [(5, False), (20, True)])
def test_gpu_mixed_batch_equals_each_scan_alone(batch, label8):
    """Five formats in turn: 5 scans with int32 labels take the CUDA-graph path, 20 scans with int8 labels the chunked one."""
    clouds = mixed_scans(batch, 900 + batch, tiny_at=(3,))
    fmts = [TABLE[k % len(TABLE)] for k in range(batch)]
    raws = as_records(clouds, fmts)
    want, want_f4 = alone(clouds, raws, fmts, FULL, label8)
    det = api.Detector(max_points=max(c.shape[0] for c in clouds), max_batch=batch, params=FULL)
    got = det.filtered_batch_mixed(raws, fmts, want_order=True, label8=label8, want_ring=True)
    for k, (r, w, w4) in enumerate(zip(got, want, want_f4)):
        full_same(r, w, f"scan {k} {fmts[k]}")
        full_same(r, w4, f"scan {k} {fmts[k]} against float4")
    det.close()


def test_gpu_mixed_launch_count_and_staging_growth():
    """A mixed batch launches what a one-format record batch of the same shape launches. Its records are staged at the
    batch's largest point_step: 6 full scans of 64-byte records outgrow slot 0's max_points * 64 staging bytes, and the
    grown buffer serves the next mixed batch (and a one-format one) as well."""
    clouds = mixed_scans(6, 77)
    n = max(c.shape[0] for c in clouds)
    det = api.Detector(max_points=n, max_batch=6, params=FULL)
    base = det.filtered_batch_records(as_records(clouds, [OS48] * 6), *OS48, want_order=True, label8=False)
    launches = det.last_launch_count()
    for fmts in ([OS48, V22, XYZ, V32, OS48, api.FLOAT4_FORMAT], [api.CloudFormat(64, 52, 56, 60, 0), XYZ] * 3):
        raws = as_records(clouds, fmts)
        got = det.filtered_batch_mixed(raws, fmts, want_order=True, label8=False)
        assert det.last_launch_count() == launches, fmts
        want, _ = alone(clouds, raws, fmts, FULL, False)
        for k, (r, w, b) in enumerate(zip(got, want, base)):
            full_same(r, w, f"scan {k} {fmts[k]}", ring=False)
            same(r, b, f"scan {k} {fmts[k]} against the 48-byte batch")
    again = det.filtered_batch_records(as_records(clouds, [OS48] * 6), *OS48, want_order=True, label8=False)
    assert det.last_launch_count() == launches
    for k, (r, b) in enumerate(zip(again, base)):
        same(r, b, f"scan {k}: one format after the growth")
    det.close()


def test_gpu_two_mixed_batches_in_flight():
    """enqueue A, enqueue B, finish A, enqueue C, finish B, finish C, ... from pinned handles; every result equals its scan
    alone."""
    clouds = mixed_scans(16, 501)
    n = max(c.shape[0] for c in clouds)
    batches = [list(range(4 * i, 4 * i + 4)) for i in range(4)]
    fmts = [TABLE[(k * 2) % len(TABLE)] for k in range(16)]
    raws = as_records(clouds, fmts)
    want, _ = alone(clouds, raws, fmts, FULL, True)
    det = api.Detector(max_points=n, max_batch=4, params=FULL)
    hbs = [api.BatchHandle.of_mixed([raws[k] for k in b], [fmts[k] for k in b], want_ring=True, want_order=True, label8=True,
                                    pinned=True) for b in batches]
    done = []
    det.enqueue(hbs[0])
    for i in range(1, len(hbs)):
        det.enqueue(hbs[i])
        done.append(det.finish_batch())
    done.append(det.finish_batch())
    for hb, b in zip(done, batches):
        for r, k in zip(hb.results, b):
            full_same(r, want[k], f"scan {k} {fmts[k]}")
    det.close()


@pytest.mark.parametrize("tie", ["input", "reference"])
def test_gpu_mixed_batch_in_both_tie_orders(port, tie):    # noqa: F811 — the module fixture of the ties tests
    """Dual-return and duplicated-point tie clouds, each in three formats in one batch: every copy equals its scan alone in
    that tie order, and in the reference order the CPU oracle's (the reference's Lomuto order)."""
    for nm in ("dual_appended", "dual_interleaved", "duplicates"):
        pts, prm, o = expect(port, nm)
        fmts = [V22, OS48, api.FLOAT4_FORMAT]
        clouds = [pts] * 3
        raws = as_records(clouds, fmts)
        want, _ = alone(clouds, raws, fmts, prm, False, tie)
        det = api.Detector(max_points=pts.shape[0], max_batch=3, params=prm, tie_order=tie)
        got = det.filtered_batch_mixed(raws, fmts, want_order=True, label8=False, want_ring=True)
        for k, (r, w) in enumerate(zip(got, want)):
            full_same(r, w, f"{nm} {tie} {fmts[k]}")
            if tie == "reference":
                check_ties(r, o, f"{nm} {fmts[k]} (mixed batch)", ring=False)
        det.close()


def test_gpu_mixed_batch_reproduces_a_golden_fixture():
    """c2_default_s0 as 48-byte and as packed 22-byte records in one batch: both reproduce the unmodified reference's labels,
    clouds and marker strips."""
    g = Golden("c2_default_s0")
    fmts = [OS48, V22]
    raws = as_records([g.cloud, g.cloud], fmts)
    det = api.Detector(max_points=g.cloud.shape[0], max_batch=2, params=g.params())
    for k, r in enumerate(det.filtered_batch_mixed(raws, fmts, want_order=True, label8=False)):
        assert_matches_golden(g, r, api.build_markers)
        if g.published and not r.flags & 4:
            assert np.array_equal(r.cloud_indices("road"), g.road_ids), fmts[k]
            assert np.array_equal(r.cloud_indices("curb"), g.curb_ids), fmts[k]
    det.close()


@pytest.mark.parametrize("kind", ["queue", "mq"])
def test_gpu_formats_stream_across_a_channels_and_roi_update(kind):
    """A formats ScanQueue (one GPU) or MultiGpuQueue (all visible GPUs; with one GPU, two device queues on it), int8 slots and
    URF_QUEUE_ORDER: 40 scans of the five formats in turn, copying and by-reference submits, with max_batch 12 so that the
    worker takes mixed batches on both batch paths, and at scan 24 an update to channels 16 and the default ROI. Every result
    equals its scan alone under its generation's set."""
    count, at = 40, 24
    sets = [FULL, make_params(channels=16)]
    clouds = mixed_scans(count, 1300, tiny_at=(5,))
    fmts = [k % len(TABLE) for k in range(count)]
    raws = as_records(clouds, [TABLE[f] for f in fmts])
    gen_of = [int(k >= at) for k in range(count)]
    want = {g: alone(clouds, raws, [TABLE[f] for f in fmts], sets[g], True)[0] for g in (0, 1)}
    n = max(c.shape[0] for c in clouds)
    if kind == "queue":
        det = api.Detector(max_points=n, max_batch=12, params=FULL)
        q = api.ScanQueue(det, max_points=n, slots=count, max_batch=12, label8=True, order=True, formats=TABLE)
    else:
        q = api.MultiGpuQueue(devices(), max_points=n, slots_per_device=count, max_batch=12, params=FULL, label8=True, order=True,
                              formats=TABLE)

    def check(t, r):
        assert r.params_gen == gen_of[t], (t, r.params_gen)
        w = want[gen_of[t]][t]
        for f in FIELDS:
            assert getattr(r, f) == getattr(w, f), f"scan {t} {TABLE[fmts[t]]}: {f}"
        same(r, w, f"{kind} scan {t} {TABLE[fmts[t]]}")

    th, err = consume(q, count, kind == "queue", check)
    for k in range(count):
        if k == at:
            assert q.update_params(sets[1]) == 1
        assert q.submit_records(raws[k], clouds[k].shape[0], tag=k, timeout_ms=300_000, by_reference=k % 3 != 2,
                                fmt=fmts[k]) == URF_OK
    finish(th, err)
    st = q.stats()
    print(kind, st)
    q.close()
    q.destroy()

"""The reference tie order on the device (urf_set_tie_order(ctx, URF_TIES_REFERENCE); k_sort_rings -> k_lomuto_rings in
front of k_label): on every tie cloud of tests/tie_policy.py the device publishes what the CPU oracle publishes — labels,
ring ids, ring starts, the emission order and the marker vertices, bit for bit — and what the unmodified reference
published (tests/golden/ref/ties.npz), through every entry point that runs the pipeline. Plus whole dual-return scans in
which every ring ties (both azimuth directions), a tied ring larger than the kernel's
shared-memory capacity, the tie-free goldens (identical to the default order), switching back, and the queues."""
import ctypes as C
import json
import os

import numpy as np
import pytest
import torch

from oracle.pyoracle import PortOracle, RefOracle
from urban_road_filter_b200 import FULL_ROI, UrfParams, UrfResult, api, make_params
from urban_road_filter_b200.api import build_markers
from urban_road_filter_b200.synth import make_scan

import tie_policy as tp
from util import REF_DIR, Golden, cloud2_records, compare_strips, digest

pytestmark = pytest.mark.gpu

NAMES = list(tp.CASES)


@pytest.fixture(scope="module")
def port():
    return PortOracle()


@pytest.fixture(scope="module")
def det():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    d = api.Detector(max_points=300_032, max_batch=2, tie_order="reference")
    yield d
    d.close()


_EXP: dict = {}


def expect(port, name):
    if name not in _EXP:
        pts, prm = tp.CASES[name](port)
        _EXP[name] = (pts, prm, port.run(pts, prm, debug=True))
    return _EXP[name]


def check(r, o, what, order=True, ring=True):
    """r (device, reference tie order) against o (CPU oracle, the reference's Lomuto order on every ring that ties)."""
    assert r.status == o.status == 0, what
    np.testing.assert_array_equal(r.label, o.label, err_msg=f"{what}: labels")
    if ring and r.ring is not None:
        np.testing.assert_array_equal(r.ring, o.ring, err_msg=f"{what}: ring ids")
    assert (r.n_roi, r.n_rings, r.n_order, r.n_road, r.n_curb, r.n_vert) == (o.n_roi, o.n_rings, o.n_order, o.n_road, o.n_curb, o.n_vert), what
    assert r.vert.tobytes() == o.vert.tobytes(), f"{what}: vertices"
    if order:
        np.testing.assert_array_equal(r.ring_start, o.ring_start, err_msg=f"{what}: ring_start")
        np.testing.assert_array_equal(r.order, o.order, err_msg=f"{what}: emission order")


def _ties_fixture():
    z = np.load(os.path.join(REF_DIR, "ties.npz"))
    return json.loads(str(z["meta"])), {k: z[k] for k in z.files if k != "meta"}


def check_reference(r, pts, prm, ref, arrays, name):
    """What the unmodified reference published for this cloud: label / road / curb / road_probably digests and the raw
    marker strips (simplification off), as tests/test_ties.py checks the oracle."""
    lab = r.label[r.order]
    prob = r.order[r.ring_start[10]: r.ring_start[11]] if r.n_rings > 10 else r.order[:0]
    assert digest(r.label) == ref["label"], name
    assert digest(r.order[lab == 1]) == ref["road_ids"], name
    assert digest(r.order[lab == 2]) == ref["curb_ids"], name
    assert digest(prob) == ref["prob_ids"], name
    raw = UrfParams.from_buffer_copy(prm)
    raw.simple_poly_allow, raw.poly_z_avg_allow = 0, 0
    strips, _ = build_markers(raw, r.vert, 0)
    meta, pts_ = arrays[name + "_meta"], arrays[name + "_pts"]
    ref_strips, k = [], 0
    for sid, act, red, cnt in meta:
        ref_strips.append((int(sid), int(act), int(red), pts_[k: k + cnt]))
        k += cnt
    compare_strips(strips, ref_strips, name + " raw strips")


@pytest.mark.parametrize("name", NAMES)
def test_reference_ties_single_scan(det, port, name):
    """Graphed single scan with the emission order, and without it (the ring sort runs anyway: it decides the vertices)."""
    pts, prm, o = expect(port, name)
    det.set_params(prm)
    r = det.filtered(pts)
    check(r, o, name)
    meta, arrays = _ties_fixture()
    check_reference(r, pts, prm, meta[name], arrays, name)
    check(det.filtered(pts, want_order=False), o, name + " without order", order=False)


def test_reference_ties_chunked_host_batch(port):
    """Every tie cloud in host batches of 21 scans (chunked copy / compute pipeline) with tie-free scans between them."""
    groups = {}
    for name in NAMES:
        pts, prm, o = expect(port, name)
        groups.setdefault(bytes(prm), []).append((name, pts, o))
    d = api.Detector(max_points=32_768, max_batch=24, tie_order="reference")
    try:
        for items in groups.values():
            prm = expect(port, items[0][0])[1]
            d.set_params(prm)
            fill = [make_scan("C1", 90 + s, order=("column", "ring")[s % 2]) for s in range(21 - len(items))]
            clouds = [pts for _, pts, _ in items] + fill
            clouds = clouds[::2] + clouds[1::2]
            rs = d.filtered_batch(clouds)
            by_id = {id(pts): (n, o) for n, pts, o in items}
            for c, r in zip(clouds, rs):
                n, o = by_id[id(c)] if id(c) in by_id else ("filler", port.run(c, prm, debug=True))
                check(r, o, n + " in a batch")
    finally:
        d.close()


@pytest.mark.parametrize("groups", [1, 2])
@pytest.mark.parametrize("with_order", [True, False])
def test_reference_ties_device_resident_batch(port, groups, with_order):
    """urf_enqueue_batch_device_ex over one and two stream groups, with d_order and without (the order then goes to the
    context's own buffer; the vertices still follow it)."""
    by_prm = {}
    for name in NAMES:
        pts, prm, o = expect(port, name)
        by_prm.setdefault(bytes(prm), []).append((name, pts, o))
    S = max(expect(port, n)[0].shape[0] for n in NAMES)
    d = api.Detector(max_points=S, max_batch=16, tie_order="reference")
    try:
        for items in by_prm.values():
            clouds = [pts for _, pts, _ in items]
            while len(clouds) < 4:
                clouds.append(clouds[len(clouds) % len(items)])
            B = len(clouds)
            d.set_params(expect(port, items[0][0])[1])
            x = torch.zeros((B, S, 4), dtype=torch.float32, device="cuda")
            for b, c in enumerate(clouds):
                x[b, : c.shape[0]] = torch.from_numpy(c).cuda()
            lab = torch.full((B, S), -7, dtype=torch.int32, device="cuda")
            order = torch.full((B, S), -7, dtype=torch.int32, device="cuda")
            n = (C.c_int * B)(*[c.shape[0] for c in clouds])
            outs = (UrfResult * B)()
            torch.cuda.synchronize()
            d.set_option(2, groups)
            assert d.lib.urf_enqueue_batch_device_ex(d._ctx, x.data_ptr(), S, n, B, lab.data_ptr(),
                                                      order.data_ptr() if with_order else None) == 0
            assert d.lib.urf_finish_batch_device(d._ctx, outs) == 0
            lab, order = lab.cpu().numpy(), order.cpu().numpy()
            for b in range(B):
                name, _, o = items[b % len(items)]
                m = clouds[b].shape[0]
                r = api._scan_result(outs[b], lab[b, :m].copy(), None, order[b], None)
                r.ring_start = o.ring_start
                check(r, o, f"{name} device batch, {groups} groups", order=with_order)
                assert np.all(lab[b, m:] == -7)
                if not with_order:
                    assert np.all(order[b] == -7)
    finally:
        d.close()


@pytest.mark.parametrize("name", NAMES)
def test_reference_ties_packed_clouds(det, port, name):
    """urf_process_cloud2_packed: road / curb / road_probably follow the reference's order, record for record."""
    pts, prm, o = expect(port, name)
    n = pts.shape[0]
    det.set_params(prm)
    raw = cloud2_records(pts, 48, 0, 4, 8, 16, seed=n)
    r, cl = det.filtered_cloud2_packed(raw, n, 48, 0, 4, 8, 16, want_labels=True)
    check(r, o, name + " packed", ring=False)
    lab = o.label[o.order]
    ids = {"road": o.order[lab == 1], "curb": o.order[lab == 2], "roi": np.flatnonzero(o.label >= 0),
           "road_probably": o.order[o.ring_start[10]: o.ring_start[11]] if o.n_rings > 10 else o.order[:0]}
    for key, idx in ids.items():
        idx = np.asarray(idx, np.int64)
        exp = np.zeros((idx.size, 8), np.float32)
        exp[:, 0:3] = pts[idx, 0:3]
        exp[:, 3] = 1.0
        exp[:, 4] = pts[idx, 3]
        assert cl[key].shape == exp.shape and cl[key].tobytes() == exp.tobytes(), f"{name}: packed {key} cloud"


def test_reference_ties_xyz_label8(det, port):
    """The packed-xyz lean input with int8 labels."""
    for name in ("dual_interleaved", "duplicates", "xy4097_global", "nan_several"):
        pts, prm, o = expect(port, name)
        det.set_params(prm)
        (r,) = det.filtered_batch_records([np.ascontiguousarray(pts[:, :3])], 12, 0, 4, 8, want_order=True, label8=True)
        check(r, o, name + " xyz / label8", ring=False)


@pytest.mark.parametrize("name", ["dual_interleaved", "dual_appended", "duplicates", "equal_range_ring"])
def test_reference_ties_both_marker_kernels(det, port, name):
    """k_markers1 and, padded past 300,000 points outside the ROI, k_markers_grid + k_verts: both map the winner's
    emission position back through the order."""
    pts, prm, o = expect(port, name)
    det.set_params(prm)
    check(det.filtered(pts), o, name + " k_markers1")
    pad = np.tile(np.array([[1000.0, 0.0, 0.0, 1.0]], np.float32), (300_032 - pts.shape[0], 1))
    b = det.filtered(np.concatenate([pts, pad]))
    assert b.vert.tobytes() == o.vert.tobytes(), name + " k_markers_grid"
    np.testing.assert_array_equal(b.order[: o.n_order], o.order[: o.n_order])


def _dual_scan(shape, seed, reverse):
    """A whole scan in which every point has a second return at 2x range on its beam (same azimuth and ring), interleaved:
    every ring ties everywhere. reverse: the scan in the opposite azimuth direction."""
    pts = make_scan(shape, seed)
    if reverse:
        pts = pts[::-1].copy()
    sec = pts.copy()
    sec[:, :3] *= np.float32(2.0)
    out = np.empty((2 * pts.shape[0], 4), np.float32)
    out[0::2], out[1::2] = pts, sec
    return out


def _big_tied_ring(m=3000, seed=5):
    """One ring of m columns turning down in azimuth, each with a second return at 2x range right after it: 2m points,
    more than k_lomuto_rings keeps in shared memory (4096), with about one partition per column."""
    rng = np.random.default_rng(seed)
    az = np.deg2rad(359.0 - 358.0 * np.arange(m) / m)
    planar = rng.uniform(4.0, 20.0, m)
    ring = np.zeros((m, 4), np.float32)
    ring[:, 0], ring[:, 1] = planar * np.cos(az), planar * np.sin(az)
    ring[:, 2] = -np.tan(np.deg2rad(10.0)) * planar
    ring[:, 3] = rng.uniform(0, 255, m)
    sec = ring.copy()
    sec[:, :3] *= np.float32(2.0)
    out = np.empty((2 * m, 4), np.float32)
    out[0::2], out[1::2] = ring, sec
    return out, make_params(interval=3.0, **FULL_ROI)


STRESS = {
    "c2_dual_up": lambda: (_dual_scan("C2", 3, False), None),
    "c2_dual_down": lambda: (_dual_scan("C2", 4, True), None),
    "ring6000_down": _big_tied_ring,
}


@pytest.mark.parametrize("name", list(STRESS))
def test_reference_ties_stress(port, name):
    """Every ring of a whole dual-return OS1-64 scan tied (64 rings of 4096 points), in both azimuth directions; and one
    tied ring of 6000 points (work arrays in global memory)."""
    from urban_road_filter_b200.synth import SHAPES
    pts, prm = STRESS[name]()
    if prm is None:
        sh = SHAPES["C2"]
        prm = make_params(channels=sh.channels, interval=sh.interval, **FULL_ROI)
    o = port.run(pts, prm, debug=True)
    assert o.flags & 4
    d = api.Detector(max_points=pts.shape[0], max_batch=1, params=prm, tie_order="reference")
    try:
        r = d.filtered(pts)
        check(r, o, name)
        if RefOracle.available():
            ref = RefOracle().run(pts, prm)
            lab = r.label[r.order]
            np.testing.assert_array_equal(ref.label, r.label)
            np.testing.assert_array_equal(ref.road_ids, r.order[lab == 1])
            np.testing.assert_array_equal(ref.curb_ids, r.order[lab == 2])
    finally:
        d.close()


@pytest.mark.parametrize("name", ["c1_full_s0", "c2_default_s0", "c3_full_s0", "c4_full_s0", "c5_full_s0"])
def test_reference_order_is_the_default_without_ties(name):
    """Tie-free goldens: the reference order gives exactly the default order's outputs, which are the goldens'."""
    g = Golden(name)
    n = g.cloud.shape[0]
    d = api.Detector(max_points=n, max_batch=1, params=g.params())
    try:
        a = d.filtered(g.cloud)
        launches = d.last_launch_count()
        d.set_tie_order("reference")
        assert d.tie_order() == "reference"
        b = d.filtered(g.cloud)
        assert not (b.flags & 4)
        for f in ("label", "ring", "order", "ring_start"):
            np.testing.assert_array_equal(getattr(b, f), getattr(a, f), err_msg=f"{name}: {f}")
        assert b.vert.tobytes() == a.vert.tobytes()
        assert d.last_launch_count() == launches + 1                 # k_lomuto_rings
        d.set_tie_order("input")
        c = d.filtered(g.cloud)
        assert d.last_launch_count() == launches
        assert c.order.tobytes() == a.order.tobytes() and c.vert.tobytes() == a.vert.tobytes()
    finally:
        d.close()


def test_switching_back_restores_the_default_order(port):
    """After reference calls, the default order again puts ties in input order (the policy of tests/tie_policy.py)."""
    pts, prm, o = expect(port, "dual_interleaved")
    d = api.Detector(max_points=pts.shape[0], max_batch=1, params=prm)
    try:
        a = d.filtered(pts)
        n0 = d.last_launch_count()
        d.set_tie_order("reference")
        check(d.filtered(pts), o, "reference")
        d.set_tie_order("input")
        c = d.filtered(pts)
        assert d.last_launch_count() == n0
        for f in ("label", "order", "ring_start"):
            np.testing.assert_array_equal(getattr(c, f), getattr(a, f))
        assert c.vert.tobytes() == a.vert.tobytes() and c.flags == a.flags
        p = tp.policy(pts, o)
        np.testing.assert_array_equal(c.order, p.order)
    finally:
        d.close()


def test_mq_reference_ties(port):
    """urf_mq_set_tie_order: refused while a scan is in flight; queue results in the reference order equal
    Detector.filtered in the reference order."""
    names = ["dual_interleaved", "duplicates", "dual_appended"]
    pts0, prm, _ = expect(port, names[0])
    S = max(expect(port, n)[0].shape[0] for n in names)
    mq = api.MultiGpuQueue([0, 0], max_points=S, slots_per_device=4, max_batch=2, params=prm)
    try:
        mq.set_tie_order("reference")
        mq.submit(pts0, tag=0)
        with pytest.raises(api.UrfError):
            mq.set_tie_order("input")
        got = [mq.next(60_000)]
        for k, name in enumerate(names, 1):
            mq.submit(expect(port, name)[0], tag=k)
        got += [mq.next(60_000) for _ in names]
        for tag, r in got:
            name = names[0] if tag == 0 else names[tag - 1]
            _, _, o = expect(port, name)
            np.testing.assert_array_equal(r.label, o.label, err_msg=name)
            assert r.vert.tobytes() == o.vert.tobytes(), name
        mq.set_tie_order("input")
    finally:
        mq.close()

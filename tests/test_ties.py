"""Ties in azimuth and in farthest planar range, without a GPU (tests/tie_policy.py): the plain policy reference is checked
against the oracle port where no tie exists, against the CPU model of the kernels on every tie cloud, and the port against
what the unmodified reference published for the tie clouds (tests/golden/ref/ties.npz)."""
import json
import os

import numpy as np
import pytest

from oracle.pyoracle import PortOracle, RefOracle
from urban_road_filter_b200 import FULL_ROI, UrfParams, make_params
from urban_road_filter_b200.api import build_markers
from urban_road_filter_b200.synth import SHAPES, make_scan

import tie_policy as tp
from util import REF_DIR, CpuModel, Golden, cloud_digest, compare_strips, digest, golden_names


@pytest.fixture(scope="module")
def port():
    return PortOracle()


@pytest.fixture(scope="module")
def model():
    return CpuModel()


_CLOUDS: dict = {}


def tie_cloud(port, name):
    if name not in _CLOUDS:
        _CLOUDS[name] = tp.CASES[name](port)
    return _CLOUDS[name]


def assert_policy_is_port(pts, o):
    p = tp.policy(pts, o)
    assert p.tie == bool(o.flags & 4)
    if not p.tie:
        np.testing.assert_array_equal(p.order, o.order)
    np.testing.assert_array_equal(p.ring_start, o.ring_start)
    assert p.vert.tobytes() == o.vert.tobytes()


@pytest.mark.parametrize("name", golden_names())
def test_policy_equals_port_on_goldens(port, name):
    """The policy reference itself: on the fixture clouds the port's order (a stable sort by azimuth when nothing ties)
    and vertices are the policy's, and bit2 is set exactly where the policy finds a tie."""
    g = Golden(name)
    o = port.run(g.cloud, g.params(), debug=True)
    if o.status == 0:
        assert_policy_is_port(g.cloud, o)


@pytest.mark.parametrize("order", ["column", "ring"])
@pytest.mark.parametrize("shape", ["C1", "C2", "C3", "C4"])
def test_policy_equals_port_on_scans(port, shape, order):
    sh = SHAPES[shape]
    pts = make_scan(shape, 3, order=order)
    o = port.run(pts, make_params(channels=sh.channels, interval=sh.interval, **FULL_ROI), debug=True)
    assert o.status == 0 and not (o.flags & 4)
    assert_policy_is_port(pts, o)


@pytest.mark.parametrize("name", list(tp.CASES))
def test_policy_equals_cpu_model_on_tie_clouds(port, model, name):
    """The kernels' logic run on the CPU follows the written policy on every tie cloud: order, ring starts, vertices and
    flags bit1 / bit2; labels and ring ids equal the port's (DESIGN.md deviation 2: ties never change labels)."""
    pts, prm = tie_cloud(port, name)
    o = port.run(pts, prm, debug=True)
    p = tp.policy(pts, o)
    m = model.run(pts, prm)
    assert o.status == m.status == 0
    np.testing.assert_array_equal(m.label, o.label)
    np.testing.assert_array_equal(m.ring, o.ring)
    np.testing.assert_array_equal(m.order, p.order)
    np.testing.assert_array_equal(m.ring_start[: o.n_rings + 1], p.ring_start)
    assert m.vert.tobytes() == p.vert.tobytes()
    assert bool(m.flags & 4) == p.tie and (m.flags & 2) == (o.flags & 2)
    assert bool(m.flags & 8) == bool(np.any(np.isnan(o.az) & (o.ring >= 0)))
    if name in tp.EQUAL_RANGE:
        assert p.shared_max >= 100 and not p.tie
        np.testing.assert_array_equal(o.order, p.order)           # no azimuth tie: the port is the truth
        assert o.vert.tobytes() == p.vert.tobytes()


def test_tie_clouds_set_the_documented_flags(port):
    """bit2 is expected wherever a ring holds two equal azimuths; a lone NaN azimuth does not tie, although the port
    (which restates the reference's order for any ring holding a NaN) raises it; the equal-range clouds hold no tie."""
    expect_tie = {name: name not in tp.EQUAL_RANGE and name != "nan_lone" for name in tp.CASES}
    for name, want in expect_tie.items():
        pts, prm = tie_cloud(port, name)
        assert tp.policy(pts, port.run(pts, prm, debug=True)).tie == want, name
    o = port.run(*tie_cloud(port, "nan_lone"))
    assert o.flags & 4, "the port restates the reference's Lomuto order for any ring holding a NaN"


_REF = None


def ref_fixture():
    global _REF
    if _REF is None:
        z = np.load(os.path.join(REF_DIR, "ties.npz"))
        _REF = json.loads(str(z["meta"])), {k: z[k] for k in z.files if k != "meta"}
    return _REF


def _strips(meta, pts):
    out, k = [], 0
    for sid, act, red, cnt in meta:
        out.append((int(sid), int(act), int(red), pts[k: k + cnt]))
        k += cnt
    return out


@pytest.mark.parametrize("name", list(tp.CASES))
def test_port_equals_reference_on_tie_clouds(port, name):
    """The port restates the reference's Lomuto order, so on every tie cloud it publishes what the UNMODIFIED reference
    published: labels, the road / curb / road_probably clouds in emission order, and the marker strips (simplification
    off: exact vertices). Stored by tests/golden/make_golden.py --ref-checks; also run live where the reference is built."""
    meta, arrays = ref_fixture()
    ref = meta[name]
    pts, prm = tie_cloud(port, name)
    assert cloud_digest(pts) == ref["cloud_sha256"], "the builder no longer reproduces the stored input cloud"
    o = port.run(pts, prm)
    assert ref["published"] == (o.status == 0)
    lab = o.label[o.order]
    prob = o.order[o.ring_start[10]: o.ring_start[11]] if o.n_rings > 10 else o.order[:0]
    assert digest(o.label) == ref["label"]
    assert digest(o.order[lab == 1]) == ref["road_ids"]
    assert digest(o.order[lab == 2]) == ref["curb_ids"]
    assert digest(prob) == ref["prob_ids"]
    raw = UrfParams.from_buffer_copy(prm)
    raw.simple_poly_allow, raw.poly_z_avg_allow = 0, 0
    strips, _ = build_markers(raw, o.vert, 0)
    compare_strips(strips, _strips(arrays[name + "_meta"], arrays[name + "_pts"]), name + " raw strips")
    if RefOracle.available():
        r = RefOracle().run(pts, prm)
        np.testing.assert_array_equal(r.label, o.label)
        np.testing.assert_array_equal(r.road_ids, o.order[lab == 1])
        np.testing.assert_array_equal(r.curb_ids, o.order[lab == 2])
        np.testing.assert_array_equal(r.prob_ids, prob)

"""blindSpots windows, blind quarters and marker bins with azimuths exactly on their bounds, without a GPU
(tests/azimuth_edges.py): the builders reproduce the stored clouds, the oracle port publishes what the unmodified
reference published on them (tests/golden/ref/azimuth_edges.npz), and the CPU model of the kernels (curb bins, reach,
threshold rows, two look-ups per point, also checked against the window search covered_by_window) equals the port stage
by stage."""
import json
import os

import numpy as np
import pytest

from oracle.pyoracle import PortOracle, RefOracle
from urban_road_filter_b200 import UrfParams
from urban_road_filter_b200.api import build_markers

import azimuth_edges as ae
from util import REF_DIR, CpuModel, cloud_digest, compare_strips, digest, stage_diffs

NAMES = list(ae.CASES)


@pytest.fixture(scope="module")
def port():
    return PortOracle()


@pytest.fixture(scope="module")
def model():
    return CpuModel()


_CLOUDS: dict = {}


def edge_cloud(port, name):
    if name not in _CLOUDS:
        _CLOUDS[name] = ae.CASES[name](port)              # asserts every target on the final port run
    return _CLOUDS[name]


_REF = None


def ref_fixture():
    global _REF
    if _REF is None:
        z = np.load(os.path.join(REF_DIR, "azimuth_edges.npz"))
        _REF = json.loads(str(z["meta"])), {k: z[k] for k in z.files if k != "meta"}
    return _REF


def stored_cloud(name):
    meta, arrays = ref_fixture()
    pts = np.concatenate([ae.base_scan(name), arrays[name + "_tail"]])
    assert cloud_digest(pts) == meta[name]["cloud_sha256"], "the base scan no longer matches the stored cloud"
    return pts


def test_fixture_covers_every_case():
    meta, _ = ref_fixture()
    assert sorted(meta) == sorted(NAMES)


@pytest.mark.parametrize("name", NAMES)
def test_builder_reproduces_stored_cloud(port, name):
    """Each builder still hits its targets (it asserts them) and builds the cloud the reference was run on."""
    pts, _ = edge_cloud(port, name)
    assert cloud_digest(pts) == ref_fixture()[0][name]["cloud_sha256"]
    assert np.array_equal(pts, stored_cloud(name))


def _strips(meta, pts):
    out, k = [], 0
    for sid, act, red, cnt in meta:
        out.append((int(sid), int(act), int(red), pts[k: k + cnt]))
        k += cnt
    return out


@pytest.mark.parametrize("name", NAMES)
def test_port_equals_reference_on_edge_clouds(port, name):
    """Labels, the road / curb / road_probably clouds in emission order and the marker strips (simplification off)
    are what the unmodified reference published for the same cloud."""
    meta, arrays = ref_fixture()
    ref = meta[name]
    _, prm = edge_cloud(port, name)
    pts = stored_cloud(name)
    o = port.run(pts, prm)
    assert ref["published"] == (o.status == 0) and o.status == 0
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


@pytest.mark.parametrize("name", NAMES)
def test_cpu_model_equals_port_on_edge_clouds(port, model, name):
    """The kernels' logic on the CPU: every stage equals the port's (q1..q4, ring widths, reach, labels, order,
    vertices), and the model's threshold look-up agrees with its window search on every point (it fails otherwise).
    The numpy restatement of the windows gives the port's labels too."""
    _, prm = edge_cloud(port, name)
    pts = stored_cloud(name)
    o = port.run(pts, prm, debug=True)
    m = model.run(pts, prm)
    assert stage_diffs(o, m, pts.shape[0]) == []
    ae.check_labels(pts, o, prm)

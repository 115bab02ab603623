"""The oracle itself: the CPU restatement (oracle/urf_oracle.cpp) is pinned against the golden fixtures generated from the
UNMODIFIED reference (tests/golden/make_golden.py)."""
import json
import os

import numpy as np
import pytest

from oracle.pyoracle import PortOracle
from urban_road_filter_b200 import FULL_ROI, make_params
from urban_road_filter_b200.api import build_markers
from urban_road_filter_b200.synth import make_scan

from util import REF_DIR, Golden, assert_matches_golden, cloud_digest, digest, golden_names, random_param_case


@pytest.fixture(scope="module")
def port():
    return PortOracle()


@pytest.mark.parametrize("name", golden_names())
def test_port_matches_reference_golden(port, name):
    g = Golden(name)
    r = port.run(g.cloud, g.params())
    assert_matches_golden(g, r, build_markers)


@pytest.mark.parametrize("seed", range(6))
def test_port_matches_reference_random_params(port, seed):
    """Seeded random draws over the LidarFilters.cfg parameter ranges against what the unmodified reference published for
    them (tests/golden/ref/random_params.json: sha256 of its labels and of its road / curb clouds as input indices)."""
    ref = json.load(open(os.path.join(REF_DIR, "random_params.json")))[str(seed)]
    pts, prm = random_param_case(seed)
    assert cloud_digest(pts) == ref["cloud_sha256"], "the synthetic generator no longer reproduces the stored input cloud"
    p = port.run(pts, prm)
    assert ref["published"] == (p.status == 0)
    if ref["published"]:
        assert digest(p.label) == ref["label"]
        lab = p.label[p.order]                     # with azimuth ties too: the port restates the reference's Lomuto order
        assert digest(p.order[lab == 1]) == ref["road_ids"]
        assert digest(p.order[lab == 2]) == ref["curb_ids"]


def test_port_edge_cases(port):
    prm = make_params(**FULL_ROI)
    empty = port.run(np.zeros((0, 4), np.float32), prm)
    assert empty.status == 1 and empty.n_roi == 0
    nan = make_scan("C1", 0)[:2000].copy()
    nan[::7, 0] = np.nan
    nan[3::11, 2] = np.inf
    r = port.run(nan, prm)
    assert np.all(r.label[::7] == -1) and np.all(r.label[3::11] == -1)
    allzero = np.zeros((100, 4), np.float32)          # x + y + z == 0 -> dropped by the ROI lambda
    assert port.run(allzero, prm).status == 1

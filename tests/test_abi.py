"""The C-ABI boundary: liburf_b200.so loads without a GPU, exports every symbol include/urf.h declares, the ctypes mirror
has the C layouts, and compute entry points fail loudly (no CPU fallback) when there is no device."""
import ctypes as C
import os
import re
import subprocess
import tempfile

import numpy as np
import pytest
import torch

from urban_road_filter_b200 import UrfParams, UrfResult, UrfStrip, make_params
from urban_road_filter_b200.ctypes_abi import UrfClouds, UrfPointXYZI
from urban_road_filter_b200 import api
from util import ROOT


def test_every_declared_symbol_is_exported():
    hdr = open(os.path.join(ROOT, "include", "urf.h")).read()
    hdr = re.sub(r"/\*.*?\*/", "", hdr, flags=re.S)
    declared = set(re.findall(r"\b(urf_[a-z_0-9]+)\s*\(", hdr))
    assert {"urf_create", "urf_process", "urf_process_batch", "urf_set_params", "urf_build_markers"} <= declared
    lib = api.load_library()
    for name in sorted(declared):
        assert hasattr(lib, name), f"{name} declared in include/urf.h but not exported"
    assert set(api.EXPORTS) <= declared


def test_struct_layouts_match_the_header():
    src = r'''
#include <stdio.h>
#include <stddef.h>
#include "urf.h"
int main(void) {
  printf("%zu %zu %zu %zu %zu %zu %zu %zu %zu %zu %zu\n", sizeof(urf_params), sizeof(urf_result), sizeof(urf_strip),
         offsetof(urf_params, channels), offsetof(urf_params, interval), offsetof(urf_result, label), offsetof(urf_result, vert),
         sizeof(urf_point_xyzi), offsetof(urf_point_xyzi, intensity), sizeof(urf_clouds), offsetof(urf_clouds, n_road));
  return 0;
}'''
    with tempfile.TemporaryDirectory() as d:
        open(os.path.join(d, "t.c"), "w").write(src)
        subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), "-o", os.path.join(d, "t"), os.path.join(d, "t.c")], check=True)
        vals = [int(v) for v in subprocess.run([os.path.join(d, "t")], capture_output=True, text=True, check=True).stdout.split()]
    assert vals == [C.sizeof(UrfParams), C.sizeof(UrfResult), C.sizeof(UrfStrip), UrfParams.channels.offset,
                    UrfParams.interval.offset, UrfResult.label.offset, UrfResult.vert.offset,
                    C.sizeof(UrfPointXYZI), UrfPointXYZI.intensity.offset, C.sizeof(UrfClouds), UrfClouds.n_road.offset]
    assert C.sizeof(UrfPointXYZI) == 32          # pcl::PointXYZI (PCL_ADD_POINT4D + intensity, 16-byte aligned)


def test_defaults_match_cfg():
    lib = api.load_library()
    p = UrfParams()
    lib.urf_default_params(C.byref(p))
    q = make_params()
    for name, _ in UrfParams._fields_:
        assert getattr(p, name) == getattr(q, name), name
    assert lib.urf_version() == 100
    assert b"no CPU fallback" in lib.urf_strerror(-2)


@pytest.mark.skipif(torch.cuda.is_available(), reason="checks the no-GPU behaviour")
def test_no_gpu_means_error_not_fallback():
    with pytest.raises(api.UrfError) as e:
        api.Detector(1000)
    assert e.value.code == -2


def test_create_rejects_batches_beyond_the_grid_limit():
    """Every kernel takes its scan from blockIdx.y (at most 65535): urf_create refuses a larger max_batch with
    URF_ERR_CAPACITY before it touches a device, however small the scans."""
    lib = api.load_library()
    for max_batch in (65536, 65537, 1 << 20):
        ctx = C.c_void_p()
        assert lib.urf_create(C.byref(ctx), 0, 1, max_batch) == -5, max_batch
        assert not ctx.value
    if not torch.cuda.is_available():                  # 65535 passes the size checks and only then fails for want of a device
        assert lib.urf_create(C.byref(C.c_void_p()), 0, 1, 65535) == -2


def test_marker_tail_is_host_code():
    v = np.array([[1, 0, -1.8, 0], [2, 0, -1.8, 0], [3, 1, -1.8, 1], [4, 1, -1.7, 1], [5, 2, -1.8, 0], [6, 2, -1.8, 0]], np.float32)
    strips, ghost = api.build_markers(make_params(simple_poly_allow=0, poly_z_avg_allow=0), v, 5)
    assert [(s[0], s[1], s[2], len(s[3])) for s in strips] == [(0, 0, 0, 2), (1, 0, 1, 4), (2, 0, 0, 2), (3, 2, 0, 0), (4, 2, 0, 0), (5, 2, 0, 0)]
    assert ghost == 2
    assert api.build_markers(make_params(), v[:2], 7) == ([], 7)      # cM <= 2: nothing published, ghostcount kept

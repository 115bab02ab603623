"""The reference tie order without a GPU: urf_lomuto.cuh (what k_lomuto_rings runs on the device, here sequentially)
against the CPU oracle's restatement of the reference's Lomuto quicksort (tests/kat/lomuto_check.cpp), on random arrays
with ties and NaNs, monotone, rotated and dual-return rings, and the rings of every tie cloud of tests/tie_policy.py; and
the host side of the switch (argument checks, the in-flight rule of urf_mq_set_tie_order)."""
import ctypes as C
import os
import subprocess
import threading

import numpy as np
import pytest

from oracle.pyoracle import PortOracle
from urban_road_filter_b200 import api
from urban_road_filter_b200.ctypes_abi import URF_ERR_INVALID

import tie_policy as tp
from util import ROOT


def _ring_file(path):
    """Every ring of every tie cloud, its azimuths in bucket order (input order inside the ring), as lomuto_check reads them."""
    port = PortOracle()
    with open(path, "wb") as f:
        for name in tp.CASES:
            pts, prm = tp.CASES[name](port)
            o = port.run(pts, prm, debug=True)
            ring, az = np.asarray(o.ring), np.asarray(o.az, np.float32)
            for k in range(o.n_rings):
                a = az[ring == k]
                f.write(np.int32(a.size).tobytes())
                f.write(a.tobytes())


def test_lomuto_emulation_matches_the_quicksort(tmp_path):
    rings = os.path.join(tmp_path, "rings.bin")
    _ring_file(rings)
    out = subprocess.run([os.path.join(ROOT, "build", "lomuto_check"), "3000", "-f", rings], capture_output=True, text=True,
                         timeout=900)
    print(out.stdout[-6000:], out.stderr[-2000:])
    assert out.returncode == 0
    tail = out.stdout.strip().splitlines()[-1]
    assert tail.startswith("cases=") and tail.endswith("mismatches=0")
    assert int(tail.split()[0].split("=")[1]) > 3000
    stats = {l.split()[1]: dict(kv.split("=") for kv in l.split()[2:]) for l in out.stdout.splitlines() if l.startswith("stat ")}
    # a sensor ring in one direction without ties is one pass; its dual-return form needs about one partition per column
    assert stats["single_up_m2048_ring_start123.4"]["partitions"] == "0"
    assert 1000 < int(stats["dual_interleaved_down_m2048_ring_start0"]["partitions"]) < 4096


class _Gate:
    """Stand-in batch function that holds every batch until released."""

    def __init__(self):
        self.go = threading.Event()

    def __call__(self, user, xyzi, n, batch, outs):
        self.go.wait()
        for j in range(batch):
            outs[j].status, outs[j].n_in, outs[j].n_roi, outs[j].n_vert = 0, n[j], n[j], 0
        return 0


def test_mq_tie_order_only_while_idle():
    gate = _Gate()
    mq = api.MultiGpuQueue([0, 1], max_points=16, slots_per_device=2, max_batch=1, process_fn=gate)
    try:
        mq.set_tie_order("reference")                          # idle: accepted (stand-in devices have no context to set)
        mq.submit(np.zeros((16, 4), np.float32), tag=1)
        with pytest.raises(api.UrfError):
            mq.set_tie_order("input")                          # a scan in flight
        gate.go.set()
        mq.next(5000)
        mq.set_tie_order("input")
        with pytest.raises(ValueError):
            mq.set_tie_order("stable")
        lib = api.load_library()
        assert lib.urf_mq_set_tie_order(mq._m, 2) == URF_ERR_INVALID
    finally:
        mq.close()


def test_tie_order_argument_checks():
    lib = api.load_library()
    mode = C.c_int()
    assert lib.urf_set_tie_order(None, 1) == URF_ERR_INVALID
    assert lib.urf_get_tie_order(None, C.byref(mode)) == URF_ERR_INVALID
    assert lib.urf_mq_set_tie_order(None, 0) == URF_ERR_INVALID

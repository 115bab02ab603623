"""The per-scan workspace layout (urf_workspace.cuh) and the ownership of a context's CUDA resources.

Without a GPU: tests/kat/workspace_check.cpp runs the library's layout functions over a grid of capacities, launch strides,
batches, stream-group counts, host chunkings and channel counts, and checks that every sub-batch view stays inside its
allocation, that the views of one launch and the two host slots never share memory, and that the capacity sizes are the
ones the library has always allocated.

On the GPU: creating and destroying a detector that has touched every buffer allocated on demand (the second host slot,
the reference tie order's arrays, int8 labels, the packed clouds, a re-allocated record staging buffer) gives all of its
device memory back."""
import os
import subprocess

import numpy as np
import pytest

from urban_road_filter_b200 import api
from urban_road_filter_b200.synth import make_scan
from util import ROOT, cloud2_records


def test_workspace_layout():
    out = subprocess.run([os.path.join(ROOT, "build", "workspace_check")], capture_output=True, text=True, timeout=600)
    print(out.stdout[-4000:], out.stderr[-2000:])
    assert out.returncode == 0
    tail = out.stdout.strip().splitlines()[-1]
    assert tail.endswith("failures=0")
    assert int(tail.split()[0].split("=")[1]) > 100000


def _own_device_mib():
    """This process's device memory as the driver reports it (a read-only nvidia-smi query), or None if it is not listed."""
    out = subprocess.run(["nvidia-smi", "--query-compute-apps=pid,used_memory", "--format=csv,noheader,nounits"],
                         capture_output=True, text=True, check=True, timeout=60).stdout
    rows = [l.split(",") for l in out.strip().splitlines() if l.strip()]
    mine = [int(m) for p, m in rows if int(p) == os.getpid()]
    return sum(mine) if mine else None


def _round(clouds):
    """One detector's life, through every buffer it allocates on demand."""
    det = api.Detector(max_points=max(c.shape[0] for c in clouds), max_batch=len(clouds))
    try:
        det.enqueue_batch(clouds, label8=True)                         # the second host slot; int8 labels in slot 0
        det.enqueue_batch(clouds, label8=True)                         # ... and in slot 1
        det.finish_batch()
        det.finish_batch()
        recs = [cloud2_records(c, 48, 0, 4, 8, 16, seed=k) for k, c in enumerate(clouds)]
        det.filtered_batch_records(recs, 48, 0, 4, 8, 16)              # records beyond slot 0's staging: re-allocated
        det.filtered_cloud2_packed(recs[0], clouds[0].shape[0], 48, 0, 4, 8, 16)   # the packed clouds
        det.set_tie_order("reference")                                 # the reference tie order's arrays
        res = det.filtered_batch(clouds)
        assert len(res) == len(clouds)
    finally:
        det.close()


@pytest.mark.gpu
def test_destroy_returns_device_memory():
    """Catches a lost array, not every leak. The baseline is taken after one full round rather than before the first
    create, because the kernels' modules load lazily on their first launch. nvidia-smi reports whole MiB, so leaks below the
    allocator's granularity (packtot, events, pinned rows) go unseen. The test skips where nvidia-smi does not list the
    process, as inside a container's PID namespace."""
    clouds = [make_scan("C1", seed=k) for k in range(4)]
    # the first round loads the kernels' modules (lazily, on first launch) and settles the driver's own pools
    _round(clouds)
    before = _own_device_mib()
    if before is None:
        pytest.skip("nvidia-smi does not list this process (no per-process accounting here)")
    for _ in range(3):
        _round(clouds)
        assert _own_device_mib() == before

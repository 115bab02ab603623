"""Builds liburf_b200.so (nvcc, sm_90a: H100) in-tree. nvcc cross-compiles without a GPU, so this runs on the CPU box too."""
from __future__ import annotations

import os
import shutil
import subprocess

PKG = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(PKG)
CSRC = os.path.join(PKG, "csrc")
LIB = os.path.join(PKG, "liburf_b200.so")

NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17", "-fmad=false",
              "-Xcompiler", "-fPIC"]
SOURCES = ["urf_api.cu"]
HOST_SOURCES = ["urf_markers.cpp", "urf_queue.cpp", "urf_mq.cpp"]
HEADERS = ["urf_kernels.cuh", "urf_logic.cuh", "urf_device.cuh", "urf_workspace.cuh", "urf_math.cuh", "urf_stdsort.cuh", "urf_lomuto.cuh",
           "urf_host.hpp", "urf_params.hpp", "urf_queue_internal.hpp"]


def _nvcc() -> str:
    for c in (shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if c and os.path.exists(c):
            return c
    raise RuntimeError("nvcc not found")


def _stale(target: str, deps: list[str]) -> bool:
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(d) > t for d in deps)


def build_lib(force: bool = False, verbose: bool = False) -> str:
    deps = [os.path.join(CSRC, f) for f in SOURCES + HOST_SOURCES + HEADERS] + [os.path.join(ROOT, "include", "urf.h")]
    if not force and not _stale(LIB, deps):
        return LIB
    bdir = os.path.join(ROOT, "build")
    os.makedirs(bdir, exist_ok=True)
    objs = []
    for s in SOURCES:
        o = os.path.join(bdir, s + ".o")
        cmd = [_nvcc(), *NVCC_FLAGS, "-c", os.path.join(CSRC, s), "-o", o]
        if verbose:
            cmd.insert(1, "-Xptxas=-v")
        subprocess.run(cmd, check=True)
        objs.append(o)
    for s in HOST_SOURCES:
        o = os.path.join(bdir, s + ".o")
        subprocess.run(["g++", "-std=c++17", "-O2", "-fPIC", "-pthread", "-c", os.path.join(CSRC, s), "-o", o], check=True)
        objs.append(o)
    subprocess.run([_nvcc(), "-gencode", "arch=compute_90a,code=sm_90a", "-shared", "-o", LIB, *objs], check=True)
    return LIB


def build_oracle() -> None:
    """Test infrastructure: the CPU restatement always; the unmodified reference only where its sources exist (oracle/Makefile REF)."""
    subprocess.run(["make", "-C", os.path.join(ROOT, "oracle"), "port"], check=True, stdout=subprocess.DEVNULL)
    subprocess.run(["make", "-C", os.path.join(ROOT, "oracle"), "ref"], check=True, stdout=subprocess.DEVNULL)


def build_kat() -> None:
    """Host-side known-answer binaries used by tests/ (libm sweep, CPU model of the pipeline)."""
    bdir = os.path.join(ROOT, "build")
    os.makedirs(bdir, exist_ok=True)
    kat = os.path.join(ROOT, "tests", "kat")
    hdrs = [os.path.join(CSRC, h) for h in HEADERS]
    tgt = os.path.join(bdir, "math_sweep")
    if _stale(tgt, [os.path.join(kat, "math_sweep.cpp")] + hdrs):
        subprocess.run(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-I/usr/local/cuda/include", "-o", tgt, os.path.join(kat, "math_sweep.cpp"),
                        "-lpthread", "-lm"], check=True)
    tgt = os.path.join(bdir, "libmodel.so")
    if _stale(tgt, [os.path.join(kat, "model_check.cpp")] + hdrs):
        subprocess.run(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-fPIC", "-shared", "-I/usr/local/cuda/include",
                        "-o", tgt, os.path.join(kat, "model_check.cpp")], check=True)
    tgt = os.path.join(bdir, "stdsort_check")
    if _stale(tgt, [os.path.join(kat, "stdsort_check.cpp")] + hdrs):
        subprocess.run(["g++", "-std=c++17", "-O2", "-o", tgt, os.path.join(kat, "stdsort_check.cpp")], check=True)
    tgt = os.path.join(bdir, "star_prefix_check")
    if _stale(tgt, [os.path.join(kat, "star_prefix_check.cpp")] + hdrs):
        subprocess.run(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-I/usr/local/cuda/include", "-o", tgt,
                        os.path.join(kat, "star_prefix_check.cpp")], check=True)
    # the reference tie order (urf_lomuto.cuh, sequential run) against the CPU oracle's quicksort, compiled in as it is
    tgt = os.path.join(bdir, "lomuto_check")
    if _stale(tgt, [os.path.join(kat, "lomuto_check.cpp"), os.path.join(ROOT, "oracle", "urf_oracle.cpp")] + hdrs):
        subprocess.run(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-I/usr/local/cuda/include", "-o", tgt,
                        os.path.join(kat, "lomuto_check.cpp")], check=True)
    # the per-scan workspace layout (urf_workspace.cuh): views inside their allocations, sub-batches and host slots apart
    tgt = os.path.join(bdir, "workspace_check")
    if _stale(tgt, [os.path.join(kat, "workspace_check.cpp")] + hdrs):
        subprocess.run(["g++", "-std=c++17", "-O2", "-I/usr/local/cuda/include", "-o", tgt, os.path.join(kat, "workspace_check.cpp")],
                       check=True)
    # ThreadSanitizer build of the streaming queue around a stand-in batch function (no CUDA involved)
    tgt = os.path.join(bdir, "queue_stress")
    qsrc = [os.path.join(kat, "queue_stress.cpp"), os.path.join(CSRC, "urf_queue.cpp"), os.path.join(CSRC, "urf_mq.cpp"),
            os.path.join(kat, "queue_async_stubs.cpp"), os.path.join(kat, "queue_params_stubs.cpp"), os.path.join(kat, "queue_formats_stubs.cpp")]
    qdeps = [os.path.join(ROOT, "include", "urf.h"), os.path.join(CSRC, "urf_queue_internal.hpp"), os.path.join(CSRC, "urf_params.hpp")]
    if _stale(tgt, qsrc + qdeps):
        subprocess.run(["g++", "-std=c++17", "-O1", "-g", "-fsanitize=thread", "-pthread", "-o", tgt, *qsrc], check=True)
    # the same for batched delivery (urf_queue_next_batch / urf_mq_next_batch) and int8 label slots, for the worker's
    # two-batches-in-flight schedule around an asynchronous stand-in, for parameter updates on a running queue, and for
    # the emission order delivered with URF_QUEUE_ORDER, for PointCloud2 records through the multi-GPU queue, and for records
    # of several formats in one stream
    for name in ("queue_batch_stress", "queue_async_stress", "queue_params_stress", "queue_order_stress", "mq_records_stress",
                 "queue_formats_stress"):
        tgt = os.path.join(bdir, name)
        src = [os.path.join(kat, name + ".cpp")] + qsrc[1:]
        if _stale(tgt, src + qdeps):
            subprocess.run(["g++", "-std=c++17", "-O1", "-g", "-fsanitize=thread", "-pthread", "-o", tgt, *src], check=True)


def build_tools() -> str:
    """Host tools that link liburf_b200.so (tools/mq_bench: throughput of the multi-GPU ingest)."""
    bdir = os.path.join(ROOT, "build")
    os.makedirs(bdir, exist_ok=True)
    tgt = os.path.join(bdir, "mq_bench")
    src = os.path.join(ROOT, "tools", "mq_bench.cpp")
    if _stale(tgt, [src, os.path.join(ROOT, "include", "urf.h"), LIB]):
        subprocess.run(["g++", "-std=c++17", "-O2", "-pthread", "-o", tgt, src, "-L" + PKG, "-l:liburf_b200.so",
                        "-Wl,-rpath,$ORIGIN/../urban_road_filter_b200"], check=True)
    return tgt


def build_glue() -> str:
    """ros/urf_node.cpp (the ROS glue) compiled against the shim ROS/PCL headers of oracle/shim + a C test entry."""
    bdir = os.path.join(ROOT, "build")
    os.makedirs(bdir, exist_ok=True)
    tgt = os.path.join(bdir, "libglue.so")
    deps = [os.path.join(ROOT, "ros", "urf_node.cpp"), os.path.join(ROOT, "ros", "urf_node_cloud2.cpp"),
            os.path.join(ROOT, "ros", "urf_glue_common.hpp"), os.path.join(ROOT, "oracle", "shim", "shim_capture.h"),
            os.path.join(ROOT, "tests", "kat", "glue_entry.cpp"),
            os.path.join(ROOT, "include", "urf.h"), LIB]
    if _stale(tgt, deps):
        subprocess.run(["g++", "-std=c++17", "-O2", "-fPIC", "-shared", "-I" + os.path.join(ROOT, "oracle", "shim"),
                        "-I" + os.path.join(ROOT, "include"), "-o", tgt, os.path.join(ROOT, "tests", "kat", "glue_entry.cpp"),
                        "-L" + PKG, "-l:liburf_b200.so", "-Wl,-rpath,$ORIGIN/../urban_road_filter_b200"], check=True)
    return tgt


def build_glue_ros2() -> str:
    """ros2/urf_ros2_node.cpp (the ROS 2 node) compiled against the shim rclcpp headers of tests/ros2_shim + a C test entry."""
    bdir = os.path.join(ROOT, "build")
    os.makedirs(bdir, exist_ok=True)
    tgt = os.path.join(bdir, "libglue_ros2.so")
    shim = os.path.join(ROOT, "tests", "ros2_shim")
    deps = [os.path.join(ROOT, "ros2", "urf_ros2_node.cpp"), os.path.join(ROOT, "tests", "kat", "ros2_glue_entry.cpp"),
            os.path.join(ROOT, "include", "urf.h"), LIB]
    deps += [os.path.join(d, f) for d, _, fs in os.walk(shim) for f in fs]
    if _stale(tgt, deps):
        subprocess.run(["g++", "-std=c++17", "-O2", "-Wall", "-fPIC", "-shared", "-I" + shim, "-I" + os.path.join(ROOT, "include"),
                        "-o", tgt, os.path.join(ROOT, "tests", "kat", "ros2_glue_entry.cpp"),
                        "-L" + PKG, "-l:liburf_b200.so", "-Wl,-rpath,$ORIGIN/../urban_road_filter_b200"], check=True)
    return tgt


if __name__ == "__main__":
    print(build_lib(force=True, verbose=True))
    build_oracle()
    build_kat()

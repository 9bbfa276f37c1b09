"""Builds librafting_b200.so in-tree with nvcc for sm_90a (H100; no torch involved).

The .so files are build products: git-ignored, rebuilt by __graft_entry__.build() in every checkout.
"""
from __future__ import annotations

import os
import shutil
import subprocess

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "librafting_b200.so")
SOURCES = ["engine.cu"]
HEADERS = ["step_kernel.cuh", "step_body.inc", "seglog.cuh", "compact.cuh", "timers.cuh", "pair_kernel.cuh", "handlers.cuh", "tables.cuh",
           os.path.join("..", "..", "include", "rafting_b200.h")]
# the synthetic-stream generator (the simulated peers) is NOT part of the product library: tests, bench and the CPU
# reference arm load it on its own, so a process that times the CPU port never maps librafting_b200.so
WORKLOAD_LIB = os.path.join(HERE, "librafting_workload.so")
NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
    "-Xcompiler", "-fPIC", "-shared", "-Xptxas", "-v", "-Wno-deprecated-gpu-targets",
]


def nvcc() -> str:
    exe = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(exe):
        raise RuntimeError("nvcc not found: cannot build librafting_b200.so")
    return exe


def up_to_date(lib: str, deps: list, cmd: list) -> bool:
    """`lib` exists, is newer than every dependency and was built by exactly `cmd`: the command (architecture, flags,
    RAFTING_NVCC_EXTRA) is stamped beside the library, so a library built for another GPU or with other flags is rebuilt."""
    if not os.path.exists(lib) or any(os.path.getmtime(d) > os.path.getmtime(lib) for d in deps):
        return False
    try:
        with open(lib + ".cmd") as f:
            return f.read() == " ".join(cmd)
    except OSError:
        return False


def compile_lib(cmd: list, lib: str, what: str) -> str:
    """Runs `cmd` and stamps it beside `lib` once it succeeded; returns the compiler's output."""
    if os.path.exists(lib + ".cmd"):
        os.remove(lib + ".cmd")
    res = subprocess.run(cmd, capture_output=True, text=True)
    log = res.stdout + res.stderr
    if res.returncode != 0:
        raise RuntimeError(f"{what} failed:\n" + log[-4000:])
    with open(lib + ".cmd", "w") as f:
        f.write(" ".join(cmd))
    return log


def build(force: bool = False, verbose: bool = False) -> str:
    extra = os.environ.get("RAFTING_NVCC_EXTRA", "").split()      # e.g. -DRAFTING_MINBLOCKS=5 for tuning runs
    cmd = [nvcc()] + NVCC_FLAGS + extra + [os.path.join(CSRC, s) for s in SOURCES] + ["-o", LIB, "-ldl"]
    if not force and up_to_date(LIB, [os.path.join(CSRC, s) for s in SOURCES + HEADERS], cmd):
        return LIB
    log = compile_lib(cmd, LIB, "nvcc")
    with open(os.path.join(HERE, "build.log"), "w") as f:
        f.write(" ".join(cmd) + "\n" + log)
    if verbose:
        print(log)
    return LIB


def build_workload(force: bool = False) -> str:
    src = os.path.join(CSRC, "workload.cu")
    deps = [src, os.path.join(HERE, "..", "include", "rafting_workload.h"), os.path.join(HERE, "..", "include", "rafting_b200.h")]
    cmd = [nvcc()] + NVCC_FLAGS + [src, "-o", WORKLOAD_LIB]
    if not force and up_to_date(WORKLOAD_LIB, deps, cmd):
        return WORKLOAD_LIB
    compile_lib(cmd, WORKLOAD_LIB, "nvcc (workload)")
    return WORKLOAD_LIB


FLAGS_LIB = os.path.join(HERE, "librafting_b200_flags.so")


def build_flags(force: bool = False) -> str:
    """The default library under a second name, for tests/test_cluster_gpu.py::test_opt_in_protocol_fixes_on_the_device_in_lock_step,
    which loads it with RAFTING_B200_LIB=<path> and checks that the file name says "flags".  The opt-in protocol fixes
    (RAFTING_CFG_STRICT_CANDIDATE_VOTE, RAFTING_CFG_LENIENT_FOLLOWER_COMMIT) are part of the default library, so this is the
    same build of the same sources, copied rather than compiled twice; `force` forces the copy, not a second compile."""
    lib = build()
    if force or not up_to_date(FLAGS_LIB, [lib], [lib]):
        if os.path.exists(FLAGS_LIB + ".cmd"):
            os.remove(FLAGS_LIB + ".cmd")
        shutil.copy(lib, FLAGS_LIB)
        with open(FLAGS_LIB + ".cmd", "w") as f:
            f.write(lib)
    return FLAGS_LIB


DURABLE_LIB = os.path.join(HERE, "librafting_durable.so")


def build_durable(force: bool = False) -> str:
    """Host-only durability journal (include/rafting_durable.h): plain g++, no CUDA."""
    src = os.path.join(CSRC, "durable.cpp")
    hdr = os.path.join(HERE, "..", "include", "rafting_durable.h")
    cmd = [shutil.which("g++") or "g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-Wall", "-Wextra", src, "-o", DURABLE_LIB]
    if not force and up_to_date(DURABLE_LIB, [src, hdr], cmd):
        return DURABLE_LIB
    compile_lib(cmd, DURABLE_LIB, "g++")
    return DURABLE_LIB


INGEST_LIB = os.path.join(HERE, "librafting_ingest.so")


def build_ingest(force: bool = False) -> str:
    """Host-only transport framing (include/rafting_ingest.h): plain g++, no CUDA."""
    src = os.path.join(CSRC, "ingest.cpp")
    deps = [src, os.path.join(HERE, "..", "include", "rafting_ingest.h"), os.path.join(HERE, "..", "include", "rafting_b200.h")]
    cmd = [shutil.which("g++") or "g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-Wall", "-Wextra", src, "-o", INGEST_LIB]
    if not force and up_to_date(INGEST_LIB, deps, cmd):
        return INGEST_LIB
    compile_lib(cmd, INGEST_LIB, "g++")
    return INGEST_LIB


if __name__ == "__main__":
    print(build(force=True, verbose=True))
    print(build_flags(force=True))
    print(build_workload(force=True))
    print(build_durable(force=True))
    print(build_ingest(force=True))

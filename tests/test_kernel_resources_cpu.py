"""The register / shared-memory budget of the R = 3 leader-stream kernel, and the due selection's stack, read from the built
library (no GPU needed).

pair_kernel<3> runs 128-thread blocks.  At 64 registers, 8 blocks fill one SM's 65 536 registers, and 8 blocks per SM put
config #2's 64 K groups x 2 follower lanes in one wave on an H100's 132 SMs (DESIGN.md §5).  Each block also takes a
3-stage input ring of dynamic shared memory beside its static shared memory, and 8 of them must fit in the SM's 228 KB.
A kernel change that breaks either condition still computes the same outputs, only slower, so it is checked here."""
import os
import re
import shutil
import subprocess

import pytest

CUOBJDUMP = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"

BLOCKS_PER_SM = 8
MAX_REGS = 65536 // (BLOCKS_PER_SM * 128)
SMEM_PER_SM = 233472          # 228 KB on sm_90, the per-block 1 KB reserve included in SHARED below
RING = 3 * 7680               # launch_pair: 3 stages of pair::PStage (64 groups x 120 B of inbox)
MAX_STACK = 480               # pair_kernel<3>'s frame when its group scalars moved to shared memory; it should not grow


def _res_usage(kernel: str) -> dict:
    from rafting_b200 import _build
    lib = _build.build()
    out = subprocess.run([CUOBJDUMP, "-res-usage", lib], capture_output=True, text=True, check=True).stdout
    m = re.search(r"Function (\S*" + re.escape(kernel) + r"\S*):\s*\n\s*(REG:.*)", out)
    assert m, f"{kernel} not found in cuobjdump -res-usage of {lib}"
    return {k: int(v) for k, v in re.findall(r"(\w+):(\d+)", m.group(2))}


@pytest.mark.skipif(not os.path.exists(CUOBJDUMP), reason="cuobjdump not installed")
def test_pair_kernel_keeps_one_wave():
    r = _res_usage("pair11pair_kernelILi3E")
    assert r["REG"] <= MAX_REGS, f"pair_kernel<3> uses {r['REG']} registers: {BLOCKS_PER_SM} blocks per SM need <= {MAX_REGS}"
    assert BLOCKS_PER_SM * (r["SHARED"] + RING) <= SMEM_PER_SM, \
        f"pair_kernel<3>: {BLOCKS_PER_SM} x ({r['SHARED']} B static + {RING} B ring) exceeds {SMEM_PER_SM} B of shared memory per SM"
    assert r["STACK"] <= MAX_STACK, f"pair_kernel<3>'s stack frame grew to {r['STACK']} B (was {MAX_STACK})"


@pytest.mark.skipif(not os.path.exists(CUOBJDUMP), reason="cuobjdump not installed")
def test_due_selection_kernels_use_no_stack():
    """The due query and a due step's tail run these three kernels over every group of the shard: a stack frame or a spill
    would add local-memory traffic to a pass that reads 16 B per group."""
    from rafting_b200 import _build
    out = subprocess.run([CUOBJDUMP, "-res-usage", _build.build()], capture_output=True, text=True, check=True).stdout
    for kernel in ("due_member_kernel", "due_scan_kernel", "due_emit_kernel"):    # each instantiation, with and without fillers
        found = re.findall(r"Function (\S*" + kernel + r"\S*):\s*\n\s*(REG:.*)", out)
        assert found, f"{kernel} not found in cuobjdump -res-usage"
        for name, usage in found:
            r = {k: int(v) for k, v in re.findall(r"(\w+):(\d+)", usage)}
            assert r["STACK"] == 0 and r["LOCAL"] == 0, f"{name}: {r['STACK']} B of stack, {r['LOCAL']} B of local memory"

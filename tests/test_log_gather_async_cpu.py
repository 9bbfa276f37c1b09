"""rafting_log_gather_begin / _wait without a GPU: the two range kernels run one thread per entry over every entry of an
apply batch, so neither may carry a stack frame or local memory (read from the built library, as
tests/test_kernel_resources_cpu.py does), and the library and the binding both carry the two entry points."""
import os
import re
import shutil
import subprocess

import pytest

CUOBJDUMP = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"


@pytest.mark.skipif(not os.path.exists(CUOBJDUMP), reason="cuobjdump not installed")
def test_range_kernels_use_no_stack():
    from rafting_b200 import _build
    out = subprocess.run([CUOBJDUMP, "-res-usage", _build.build()], capture_output=True, text=True, check=True).stdout
    for kernel in ("range_probe_kernel", "range_emit_kernel"):
        found = re.findall(r"Function (\S*" + kernel + r"\S*):\s*\n\s*(REG:.*)", out)
        assert len(found) == 1, f"{kernel} not found in cuobjdump -res-usage"
        r = {k: int(v) for k, v in re.findall(r"(\w+):(\d+)", found[0][1])}
        assert r["STACK"] == 0 and r["LOCAL"] == 0, f"{kernel}: {r['STACK']} B of stack, {r['LOCAL']} B of local memory"


@pytest.mark.skipif(shutil.which("nm") is None, reason="no nm")
def test_entry_points_are_exported_and_declared():
    from rafting_b200 import _build, engine
    names = subprocess.run(["nm", "-D", "--defined-only", _build.build()], capture_output=True, text=True, check=True).stdout.split()
    for sym in ("rafting_log_gather_begin", "rafting_log_gather_wait"):
        assert sym in names and sym in engine.EXPORTS, sym
    assert hasattr(engine.Engine, "log_gather_begin") and hasattr(engine.Engine, "log_gather_wait")
    L = engine.lib()                                        # loading the library sets every declared signature
    assert len(L.rafting_log_gather_begin.argtypes) == 10 and len(L.rafting_log_gather_wait.argtypes) == 5

"""The C-ABI library loads without a GPU, exports every symbol include/rafting_b200.h declares,
its struct layouts match the ctypes mirror, and it refuses to run without a CUDA device."""
import ctypes as C
import os
import re

import pytest

from rafting_b200 import abi, engine

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared(header):
    src = open(os.path.join(ROOT, "include", header)).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(rafting_[a-z0-9_]+)\s*\(", src)) - {"rafting_splitmix64", "rafting_draw"})


def test_every_declared_symbol_is_exported():
    L = engine.lib()
    names = _declared("rafting_b200.h")
    assert len(names) >= 25
    for n in names:
        assert hasattr(L, n), f"{n} declared in include/rafting_b200.h but not exported by librafting_b200.so"
    assert set(engine.EXPORTS) <= set(names)
    from rafting_b200 import workload
    W = workload._bind()
    for n in _declared("rafting_workload.h"):
        assert hasattr(W, n), f"{n} declared in include/rafting_workload.h but not exported by librafting_workload.so"
        assert not hasattr(L, n), f"{n}: the stream generator must not live in the product library"


def test_durable_library_exports_its_header():
    from rafting_b200 import durable
    L = durable.lib()
    names = _declared("rafting_durable.h")
    assert len(names) >= 9
    for n in names:
        assert hasattr(L, n), f"{n} declared in include/rafting_durable.h but not exported by librafting_durable.so"


def test_ingest_library_exports_its_header():
    from rafting_b200 import ingest
    L = ingest.lib()
    names = _declared("rafting_ingest.h")
    assert len(names) >= 8
    for n in names:
        assert hasattr(L, n), f"{n} declared in include/rafting_ingest.h but not exported by librafting_ingest.so"


def test_struct_sizes_match_the_compiled_library():
    out = (C.c_uint32 * 7)()
    assert engine.lib().rafting_abi_sizes(out, 7) == 7
    mirror = [C.sizeof(x) for x in (abi.Cfg, abi.InboxC, abi.OutboxC, abi.GroupInit, abi.FollowerState,
                                    abi.GroupState, abi.LeaseC)]
    assert list(out) == mirror


def test_no_cpu_fallback_without_a_device():
    import torch
    if torch.cuda.is_available():
        pytest.skip("a CUDA device is present")
    with pytest.raises(engine.RaftingError) as ei:
        engine.Engine(abi.make_cfg())
    assert ei.value.rc == -6     # RAFTING_E_NODEVICE


def test_product_does_not_touch_the_oracle():
    pkg = os.path.join(ROOT, "rafting_b200")
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h", ".cpp")):
                txt = open(os.path.join(dirpath, f), errors="replace").read()
                assert "oracle/" not in txt.replace("nothing here includes or links oracle/", "").replace(
                    "Nothing here includes or links oracle/", "") or f in ("engine.cu",), f
                assert "import oracle" not in txt and "from oracle" not in txt, f


def test_native_code_reads_no_environment_switches():
    """What a step launches depends on its inputs and the engine's configuration only, never on the process environment."""
    csrc = os.path.join(ROOT, "rafting_b200", "csrc")
    for dirpath, _, files in os.walk(csrc):
        for f in files:
            if f.endswith((".cu", ".cuh", ".inc", ".cpp")):
                assert "getenv" not in open(os.path.join(dirpath, f), errors="replace").read(), f

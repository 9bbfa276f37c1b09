"""Field-by-field layout check of every Python mirror (MIRRORS of tools/gen_java_layout.py: ctypes Structures in
rafting_b200/abi.py, numpy record dtypes in abi.py / ingest.py / engine.py / durable.py / workload.py) against the C headers: a
probe compiled by gcc from include/*.h prints sizeof and offsetof for each struct and field, and the mirrors must agree.  Host
only — the headers are plain C."""
import importlib.util
import os
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_spec = importlib.util.spec_from_file_location("gen_java_layout", os.path.join(ROOT, "tools", "gen_java_layout.py"))
gen = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(gen)
MIRRORS, RENAMED, _fields = gen.MIRRORS, gen.RENAMED, gen.fields


@pytest.mark.skipif(shutil.which("gcc") is None, reason="no gcc")
def test_every_mirror_has_the_layout_the_headers_compile_to(tmp_path):
    lines = ['#include <stdio.h>', '#include <stddef.h>', '#include "rafting_b200.h"', '#include "rafting_ingest.h"',
             '#include "rafting_durable.h"', '#include "rafting_workload.h"', 'int main(void) {']
    for cname, m in MIRRORS.items():
        fields, _ = _fields(m)
        lines.append(f'  printf("{cname} %zu\\n", sizeof({cname}));')
        for n, _, _ in fields:
            cn = RENAMED.get(cname, {}).get(n, n)
            lines.append(f'  printf("{cname}.{n} %zu %zu\\n", offsetof({cname}, {cn}), sizeof((({cname}*)0)->{cn}));')
    lines += ['  return 0;', '}']
    src = tmp_path / "probe.c"
    src.write_text("\n".join(lines))
    exe = tmp_path / "probe"
    res = subprocess.run(["gcc", "-std=c11", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], capture_output=True, text=True)
    assert res.returncode == 0, res.stderr[-3000:]
    got = {}
    for ln in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.splitlines():
        k, *v = ln.split()
        got[k] = tuple(int(x) for x in v)
    for cname, m in MIRRORS.items():
        fields, size = _fields(m)
        assert got[cname] == (size,), f"sizeof({cname}) = {got[cname][0]}, the mirror has {size}"
        for n, off, sz in fields:
            assert got[f"{cname}.{n}"] == (off, sz), f"{cname}.{n}: C (offset, size) = {got[f'{cname}.{n}']}, mirror = {(off, sz)}"


@pytest.mark.skipif(shutil.which("gcc") is None, reason="no gcc")
def test_generated_java_layout_constants_are_current():
    """rafting_b200/java/.../Layout.java (offsets the Java side uses on direct ByteBuffers) is generated from the headers by
    tools/gen_java_layout.py; a header change without regenerating it fails here."""
    assert open(gen.OUT).read() == gen.generate(), "run `python tools/gen_java_layout.py`"

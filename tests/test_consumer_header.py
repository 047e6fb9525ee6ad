"""The public device header of resident consumers (include/apus_consumer.cuh) without a GPU: a consumer that includes
only that header compiles for sm_90a without spills, and apus_consumer_view_t has the layout the ctypes ConsumerView
gives it."""
import ctypes as C
import os
import shutil
import subprocess

import pytest

import resident
from apus_b200 import engine as E

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.skipif(shutil.which("nvcc") is None, reason="needs nvcc")
def test_resident_consumer_compiles_against_the_public_header_alone(tmp_path):
    """resident_rows.cu sees include/ and nothing of the engine's sources, and ptxas reports no spills"""
    _, log = resident.compile_so(str(tmp_path), ["-Xptxas", "-v"])
    assert "resident_rows_kernel" in log, log
    for line in log.splitlines():
        if "spill" in line:
            assert "0 bytes spill stores, 0 bytes spill loads" in line, line
    hdr = open(os.path.join(ROOT, "include", "apus_consumer.cuh")).read()
    includes = [ln.split()[1] for ln in hdr.splitlines() if ln.startswith("#include")]
    assert includes == ["<cuda_runtime.h>", "<stdint.h>", '"apus_gpu.h"'], includes


@pytest.mark.skipif(shutil.which("gcc") is None, reason="needs gcc")
def test_view_layout_matches_ctypes(tmp_path):
    """a C file that includes apus_gpu.h prints the size and every field offset of apus_consumer_view_t"""
    fields = [f for f, _ in E.ConsumerView._fields_]
    src = tmp_path / "view.c"
    src.write_text('#include <stddef.h>\n#include <stdio.h>\n#include "apus_gpu.h"\nint main(void) {\n'
                   '    printf("size %zu\\n", sizeof(apus_consumer_view_t));\n' +
                   "".join(f'    printf("{f} %zu\\n", offsetof(apus_consumer_view_t, {f}));\n' for f in fields) +
                   "    return 0;\n}\n")
    exe = tmp_path / "view"
    subprocess.run(["gcc", "-std=c99", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), "-o", str(exe), str(src)],
                   check=True)
    got = dict(ln.split() for ln in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.splitlines())
    assert int(got["size"]) == C.sizeof(E.ConsumerView)
    for f in fields:
        assert int(got[f]) == getattr(E.ConsumerView, f).offset, f

"""The public device header of resident readers (include/apus_reader.cuh) without a GPU: the test reader, which
includes only include/, compiles for sm_90a without spills; the reader header and the fence rule include exactly what
their comments name; apus_reader_view_t has the layout the ctypes ReaderView gives it; and the two C ABI calls refuse a
null replica."""
import ctypes as C
import os
import shutil
import subprocess

import pytest

import reader
from apus_b200 import engine as E

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _includes(name):
    hdr = open(os.path.join(ROOT, "include", name)).read()
    return [ln.split()[1] for ln in hdr.splitlines() if ln.startswith("#include")]


@pytest.mark.skipif(shutil.which("nvcc") is None, reason="needs nvcc")
def test_resident_reader_compiles_against_the_public_headers_alone(tmp_path):
    """resident_reads.cu sees include/ and nothing of the engine's sources, and ptxas reports no spills"""
    _, log = reader.compile_so(str(tmp_path), ["-Xptxas", "-v"])
    assert "resident_reads_kernel" in log, log
    spills = [ln for ln in log.splitlines() if "spill" in ln]
    assert spills, log
    for line in spills:
        assert "0 bytes spill stores, 0 bytes spill loads" in line, line


def test_headers_include_what_they_say():
    assert _includes("apus_reader.cuh") == ["<cuda_runtime.h>", "<stdint.h>", '"apus_gpu.h"', '"apus_fence_rule.h"',
                                            '"apus_consumer.cuh"']
    assert _includes("apus_fence_rule.h") == ["<stdint.h>"]
    engine_side = open(os.path.join(ROOT, "apus_b200", "csrc", "apus_fence.h")).read()
    assert '#include "../../include/apus_fence_rule.h"' in engine_side


@pytest.mark.skipif(shutil.which("gcc") is None, reason="needs gcc")
def test_view_layout_matches_ctypes(tmp_path):
    """a C file that includes apus_gpu.h prints the size and every field offset of apus_reader_view_t"""
    fields = [f for f, _ in E.ReaderView._fields_]
    src = tmp_path / "view.c"
    src.write_text('#include <stddef.h>\n#include <stdio.h>\n#include "apus_gpu.h"\nint main(void) {\n'
                   '    printf("size %zu\\n", sizeof(apus_reader_view_t));\n' +
                   "".join(f'    printf("{f} %zu\\n", offsetof(apus_reader_view_t, {f}));\n' for f in fields) +
                   "    return 0;\n}\n")
    exe = tmp_path / "view"
    subprocess.run(["gcc", "-std=c99", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), "-o", str(exe), str(src)],
                   check=True)
    got = dict(ln.split() for ln in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.splitlines())
    assert int(got["size"]) == C.sizeof(E.ReaderView)
    for f in fields:
        assert int(got[f]) == getattr(E.ReaderView, f).offset, f


def test_null_replica_is_refused():
    import __graft_entry__ as g
    g.build()
    lib = E.load_library()
    v = E.ReaderView()
    assert lib.apus_reader_attach(None, None, C.byref(v)) == E.APUS_ERROR
    assert lib.apus_last_error() == b"null argument"
    assert lib.apus_reader_detach(None) == E.APUS_ERROR
    assert lib.apus_last_error() == b"null argument"
    assert bytes(v) == bytes(C.sizeof(v)), "nothing was written"

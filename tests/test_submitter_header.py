"""The public device header of resident submitters (include/apus_submitter.cuh) without a GPU: a multi-CTA submitter
that includes only include/ compiles for sm_90a without spills, the header includes exactly what its comment names,
and apus_submitter_view_t has the layout the ctypes SubmitterView gives it.  The null-replica refusals of the two C ABI
calls need no GPU either."""
import ctypes as C
import os
import shutil
import subprocess

import pytest

import submitter
from apus_b200 import engine as E

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.skipif(shutil.which("nvcc") is None, reason="needs nvcc")
def test_resident_submitter_compiles_against_the_public_headers_alone(tmp_path):
    """resident_submit.cu sees include/ and nothing of the engine's sources, and ptxas reports no spills"""
    _, log = submitter.compile_so(str(tmp_path), ["-Xptxas", "-v"])
    assert "resident_submit_kernel" in log, log
    spills = [ln for ln in log.splitlines() if "spill" in ln]
    assert spills, log
    for line in spills:
        assert "0 bytes spill stores, 0 bytes spill loads" in line, line


def test_header_includes_what_it_says():
    hdr = open(os.path.join(ROOT, "include", "apus_submitter.cuh")).read()
    includes = [ln.split()[1] for ln in hdr.splitlines() if ln.startswith("#include")]
    assert includes == ["<cuda_runtime.h>", "<stdint.h>", '"apus_gpu.h"', '"apus_slot_format.h"', '"apus_consumer.cuh"']
    fmt = open(os.path.join(ROOT, "include", "apus_slot_format.h")).read()
    assert [ln.split()[1] for ln in fmt.splitlines() if ln.startswith("#include")] == \
        ["<stdint.h>", "<string.h>", '"apus_gpu.h"']


@pytest.mark.skipif(shutil.which("gcc") is None, reason="needs gcc")
def test_view_layout_matches_ctypes(tmp_path):
    """a C file that includes apus_gpu.h prints the size and every field offset of apus_submitter_view_t"""
    fields = [f for f, _ in E.SubmitterView._fields_]
    src = tmp_path / "view.c"
    src.write_text('#include <stddef.h>\n#include <stdio.h>\n#include "apus_gpu.h"\nint main(void) {\n'
                   '    printf("size %zu\\n", sizeof(apus_submitter_view_t));\n' +
                   "".join(f'    printf("{f} %zu\\n", offsetof(apus_submitter_view_t, {f}));\n' for f in fields) +
                   "    return 0;\n}\n")
    exe = tmp_path / "view"
    subprocess.run(["gcc", "-std=c99", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), "-o", str(exe), str(src)],
                   check=True)
    got = dict(ln.split() for ln in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.splitlines())
    assert int(got["size"]) == C.sizeof(E.SubmitterView)
    for f in fields:
        assert int(got[f]) == getattr(E.SubmitterView, f).offset, f


def test_null_replica_is_refused():
    import __graft_entry__ as g
    g.build()
    lib = E.load_library()
    v = E.SubmitterView()
    assert lib.apus_submitter_attach(None, None, C.byref(v)) == E.APUS_ERROR
    assert lib.apus_last_error() == b"null argument"
    assert lib.apus_submitter_detach(None) == E.APUS_ERROR
    assert lib.apus_last_error() == b"null argument"

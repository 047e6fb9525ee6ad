"""The public device headers without a GPU: every test kernel of tests/devicelogic/, which includes only include/, compiles
for sm_90a without spills; each header includes exactly what its comment names; and the views of the resident
consumer, submitter and reader have the C layout their ctypes structures give them."""
import ctypes as C
import os
import shutil
import subprocess

import pytest

import device_build as DB
from apus_b200 import engine as E

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# test kernel source -> the kernels in it; ptxas reports one spill line for each
KERNELS = {
    "resident_rows": ["resident_rows_kernel"],
    "resident_submit": ["resident_submit_kernel"],
    "resident_reads": ["resident_reads_kernel"],
    "header_probe": ["hp_copy_kernel", "hp_loads_kernel", "hp_consumer_kernel", "hp_submit_kernel"],
}

# header -> its #include lines, in order
INCLUDES = {
    "include/apus_consumer.cuh": ["<cuda_runtime.h>", "<stdint.h>", '"apus_gpu.h"'],
    "include/apus_submitter.cuh": ["<cuda_runtime.h>", "<stdint.h>", '"apus_gpu.h"', '"apus_slot_format.h"',
                                   '"apus_consumer.cuh"'],
    "include/apus_slot_format.h": ["<stdint.h>", "<string.h>", '"apus_gpu.h"'],
    "include/apus_reader.cuh": ["<cuda_runtime.h>", "<stdint.h>", '"apus_gpu.h"', '"apus_fence_rule.h"',
                                '"apus_consumer.cuh"'],
    "include/apus_fence_rule.h": ["<stdint.h>"],
    "apus_b200/csrc/apus_fence.h": ['"../../include/apus_fence_rule.h"'],      # the engine's fences use the same rule
}


@pytest.mark.skipif(shutil.which("nvcc") is None, reason="needs nvcc")
@pytest.mark.parametrize("name", list(KERNELS))
def test_kernel_compiles_against_the_public_headers_alone(name, tmp_path):
    _, log = DB.compile_so(name, str(tmp_path), ["-Xptxas", "-v"])
    for k in KERNELS[name]:
        assert k in log, log
    spills = [ln for ln in log.splitlines() if "spill" in ln]
    assert len(spills) == len(KERNELS[name]), log
    for line in spills:
        assert "0 bytes spill stores, 0 bytes spill loads" in line, line


@pytest.mark.parametrize("path", list(INCLUDES), ids=[os.path.basename(p).replace(".", "_") for p in INCLUDES])
def test_headers_include_what_they_say(path):
    hdr = open(os.path.join(ROOT, path)).read()
    assert [ln.split()[1] for ln in hdr.splitlines() if ln.startswith("#include")] == INCLUDES[path]


@pytest.mark.skipif(shutil.which("gcc") is None, reason="needs gcc")
@pytest.mark.parametrize("kind", ["consumer", "submitter", "reader"])
def test_view_layout_matches_ctypes(kind, tmp_path):
    """a C file that includes apus_gpu.h prints the size and every field offset of apus_<kind>_view_t"""
    ctype, view = f"apus_{kind}_view_t", getattr(E, kind.capitalize() + "View")
    fields = [f for f, _ in view._fields_]
    src = tmp_path / "view.c"
    src.write_text('#include <stddef.h>\n#include <stdio.h>\n#include "apus_gpu.h"\nint main(void) {\n'
                   f'    printf("size %zu\\n", sizeof({ctype}));\n' +
                   "".join(f'    printf("{f} %zu\\n", offsetof({ctype}, {f}));\n' for f in fields) +
                   "    return 0;\n}\n")
    exe = tmp_path / "view"
    subprocess.run(["gcc", "-std=c99", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), "-o", str(exe), str(src)],
                   check=True)
    got = dict(ln.split() for ln in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.splitlines())
    assert int(got["size"]) == C.sizeof(view)
    for f in fields:
        assert int(got[f]) == getattr(view, f).offset, f

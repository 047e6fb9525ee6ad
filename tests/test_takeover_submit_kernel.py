"""The test submitter that lives through take-overs (tests/devicelogic/takeover_submit.cu) without a GPU: it compiles
for sm_90a against include/ alone without spills, and its argument block and the submitter view have the sizes the
host side (tests/takeover_submit.py, apus_b200.engine.SubmitterView) gives them.  Also the C layout of the submitter's
device state, whose last word is the term the ring is held in."""
import ctypes as C
import os
import shutil
import subprocess

import pytest

import device_build as DB
import takeover_submit as TS
from apus_b200 import engine as E

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.skipif(shutil.which("nvcc") is None, reason="needs nvcc")
def test_kernel_compiles_without_spills_and_matches_its_host_side(tmp_path):
    so, log = DB.compile_so("takeover_submit", str(tmp_path), ["-Xptxas", "-v"])
    assert "takeover_submit_kernel" in log, log
    spills = [ln for ln in log.splitlines() if "spill" in ln]
    assert len(spills) == 1 and "0 bytes spill stores, 0 bytes spill loads" in spills[0], log
    L = C.CDLL(so)
    L.ts_args_size.restype = C.c_uint
    L.ts_view_size.restype = C.c_uint
    assert L.ts_args_size() == C.sizeof(TS.Args)
    assert L.ts_view_size() == C.sizeof(E.SubmitterView)


@pytest.mark.skipif(shutil.which("gcc") is None, reason="needs gcc")
def test_submitter_state_layout(tmp_path):
    """eight 64-bit words, lead_term where pad was; the dormant values are the ones engine.py names"""
    fields = ["lock", "submitted", "pay_head", "wrap_next", "consumed", "rejected", "first_rejected", "lead_term"]
    src = tmp_path / "state.c"
    src.write_text('#include <stddef.h>\n#include <stdio.h>\n#include "apus_gpu.h"\nint main(void) {\n'
                   '    printf("size %zu\\n", sizeof(apus_submitter_state_t));\n' +
                   "".join(f'    printf("{f} %zu\\n", offsetof(apus_submitter_state_t, {f}));\n' for f in fields) +
                   '    printf("held %llu\\n", (unsigned long long)APUS_SUBMITTER_HOST_HELD);\n'
                   '    printf("dormant %llu\\n", (unsigned long long)APUS_SUBMITTER_DORMANT);\n'
                   "    return 0;\n}\n")
    exe = tmp_path / "state"
    subprocess.run(["gcc", "-std=c99", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), "-o", str(exe), str(src)],
                   check=True)
    got = dict(ln.split() for ln in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.splitlines())
    assert int(got["size"]) == 64
    assert [int(got[f]) for f in fields] == [8 * k for k in range(8)]
    assert (int(got["held"]), int(got["dormant"])) == (E.SUBMITTER_HOST_HELD, E.SUBMITTER_DORMANT)

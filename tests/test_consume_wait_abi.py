"""CPU-side checks of the consume waits (apus_consume_wait): the library exports the three calls, the Python binding
lists them, its WAIT_* outcomes are the header's, and without a GPU a wait is refused rather than skipped."""
import ctypes as C
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CALLS = ("apus_consume_wait", "apus_consume_wait_release", "apus_consume_wait_status")


@pytest.fixture(scope="module")
def built():
    import __graft_entry__ as g
    g.build()
    from apus_b200 import engine
    return engine


def header_defines(prefix):
    txt = open(os.path.join(ROOT, "include", "apus_gpu.h")).read()
    return {m.group(1): int(m.group(2)) for m in re.finditer(rf"#define\s+({prefix}\w+)\s+(\d+)u?\b", txt)}


def test_the_three_calls_are_exported(built):
    lib = built.load_library()
    for s in CALLS:
        assert hasattr(lib, s), f"{s} is not exported by libapus_gpu.so"
        assert s in built.EXPORTS


def test_wait_outcomes_match_the_header(built):
    want = header_defines("APUS_WAIT_")
    assert sorted(want) == ["APUS_WAIT_READY", "APUS_WAIT_RELEASED", "APUS_WAIT_TIMED_OUT"], want
    for name, v in want.items():
        assert getattr(built, name[len("APUS_"):]) == v, name
    assert len(set(want.values())) == 3


def test_null_replica_is_refused(built):
    lib = built.load_library()
    assert lib.apus_consume_wait(None, 1, 1000, None, None) == built.APUS_ERROR
    assert lib.apus_consume_wait_release(None) == built.APUS_ERROR
    o, a = C.c_uint64(), C.c_uint64()
    assert lib.apus_consume_wait_status(None, C.byref(o), C.byref(a)) == built.APUS_ERROR

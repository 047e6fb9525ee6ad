"""CPU-side checks of the read fences (apus_read_fence): the library exports both calls, the Python binding lists them,
WAIT_NOT_LEADER is the header's, the three consume-wait outcomes keep their values, the status word pair takes spare
host words without moving any other, and without a replica a fence is refused."""
import ctypes as C
import os
import re

import pytest

ROOT = os.path.dirname(os.path.abspath(__file__ + "/.."))
CALLS = ("apus_read_fence", "apus_read_fence_status")


@pytest.fixture(scope="module")
def built():
    import __graft_entry__ as g
    g.build()
    from apus_b200 import engine
    return engine


def header_value(name):
    txt = open(os.path.join(ROOT, "include", "apus_gpu.h")).read()
    m = re.search(rf"#define\s+{name}\s+\(?(\d+)u?\)?", txt)
    assert m, f"{name} is not defined in apus_gpu.h"
    return int(m.group(1))


def test_both_calls_are_exported(built):
    lib = built.load_library()
    for s in CALLS:
        assert hasattr(lib, s), f"{s} is not exported by libapus_gpu.so"
        assert s in built.EXPORTS


def test_not_leader_matches_the_header_and_the_old_outcomes_stay(built):
    assert built.WAIT_NOT_LEADER == header_value("APUS_WAIT_NOT_LEADER") == 3
    assert (built.WAIT_READY, built.WAIT_TIMED_OUT, built.WAIT_RELEASED) == (0, 1, 2)
    for name, v in (("APUS_WAIT_READY", 0), ("APUS_WAIT_TIMED_OUT", 1), ("APUS_WAIT_RELEASED", 2)):
        assert header_value(name) == v, name


def test_status_words_take_spare_host_words():
    txt = open(os.path.join(ROOT, "apus_b200", "csrc", "apus_layout.h")).read()
    body = txt[txt.index("typedef struct apus_hostwords"):txt.index("} apus_hostwords_t;")]
    words = re.findall(r"uint64_t\s+(\w+)(?:\[(\d+)\])?;", body)
    at = {}
    off = 0
    for name, cnt in words:
        at[name] = off
        off += 8 * (int(cnt) if cnt else 1)
    # the words after the consume waits' three stay where they were: stop at 8 * 32
    assert at["fence_outcome"] == at["cons_wait_avail"] + 8 and at["fence_index"] == at["fence_outcome"] + 8
    assert at["pad1"] + 8 == 256, at


def test_null_replica_is_refused(built):
    lib = built.load_library()
    assert lib.apus_read_fence(None, 1000, None, None, None) == built.APUS_ERROR
    o, i = C.c_uint64(), C.c_uint64()
    assert lib.apus_read_fence_status(None, C.byref(o), C.byref(i)) == built.APUS_ERROR

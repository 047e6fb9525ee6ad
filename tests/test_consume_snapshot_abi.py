"""CPU-side checks of the snapshot calls of device consumers (apus_consume_mark, apus_consume_seed): the library exports
both, the Python binding lists them, the control block keeps the seed word where no kernel-owned word lies, and without a
replica both are refused rather than skipped."""
import ctypes as C
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CALLS = ("apus_consume_mark", "apus_consume_seed")


@pytest.fixture(scope="module")
def built():
    import __graft_entry__ as g
    g.build()
    from apus_b200 import engine
    return engine


def test_the_two_calls_are_exported(built):
    lib = built.load_library()
    for s in CALLS:
        assert hasattr(lib, s), f"{s} is not exported by libapus_gpu.so"
        assert s in built.EXPORTS
    hdr = open(os.path.join(ROOT, "include", "apus_gpu.h")).read()
    assert re.search(r"int\s+apus_consume_mark\(apus_replica_t \*r, uint64_t \*mark, void \*stream\);", hdr)
    assert re.search(r"int\s+apus_consume_seed\(apus_replica_t \*r, uint64_t cursor_offset, uint64_t next_idx\);", hdr)


def test_the_seed_word_takes_a_spare_word(built):
    """cons_seeded follows cons_on, in what was padding: every word before it keeps its offset, the block its size"""
    txt = open(os.path.join(ROOT, "apus_b200", "csrc", "apus_layout.h")).read()
    block = txt[txt.index("typedef struct apus_ctrl {"):txt.index("} apus_ctrl_t;")]
    tail = re.findall(r"uint64_t\s+(\w+)(?:\[(\d+)\])?;", block[block.index("uint64_t cons_rec"):])
    assert tail == [("cons_rec", "2"), ("cons_cur", "2"), ("cons_on", ""), ("cons_seeded", ""), ("pad4", "10")], tail


def test_null_replica_is_refused(built):
    lib = built.load_library()
    mark = (C.c_uint64 * 4)()
    assert lib.apus_consume_mark(None, C.addressof(mark), None) == built.APUS_ERROR
    assert lib.apus_consume_seed(None, 0, 1) == built.APUS_ERROR

"""The header probe for tests/test_gpu_header_primitives.py and tests/test_header_probe.py: tests/devicelogic/header_probe.cu
compiled with nvcc for sm_90a against include/ alone, tests/hostlogic/slot_writer.c built with gcc against
include/apus_slot_format.h, their ctypes structures, and this module's own statement of the submitter's placement rule
(Placement), which the tests check against the header compiled as C.  Importing this module starts no CUDA context."""
import ctypes as C
import os
import subprocess

import device_build as DB

WRITER_SRC = os.path.join(DB.HERE, "hostlogic", "slot_writer.c")

NOOP, CSM, CONFIG, HEAD, CONNECT, SEND, CLOSE = 0, 1, 2, 3, 4, 5, 6
ACCEPTED = (CSM, CONNECT, SEND, CLOSE)
MAX_LEN = 0xFFFF
SLOT_BYTES, SLOT_INLINE = 128, 80
SLOT_EXT, SLOT_WRAP = 1 << 29, 1 << 30
OK, TIMED_OUT, STOPPED, NEVER_FITS, SKIPPED = 0, 1, 2, 3, 0xFF
CONS_OK, CONS_LATER, CONS_BAD = 0, 1, 2
HEAD_BIT = 0x80000000
RESERVE, PUBLISH, WAIT = 1, 2, 3
PUT = 1
EXT_OF_REQUESTS = (1 << 64) - 1
HDR = 64

vp, u64, u32, u16 = C.c_void_p, C.c_uint64, C.c_uint32, C.c_uint16


class CopyCase(C.Structure):
    _fields_ = [("src", u64), ("dst", u64), ("len", u32), ("nthr", u32), ("groups", u32), ("via", u32)]


class Entry(C.Structure):
    """apus_consumer_entry_t"""
    _fields_ = [("idx", u64), ("req_id", u64), ("cmd_off", u64), ("off", u64), ("type", u32), ("len", u32),
                ("clt_id", u32), ("status", u32)]


class Req(C.Structure):
    _fields_ = [("type", u32), ("conn", u32), ("len", u32), ("pad", u32), ("req_id", u64), ("cmd_off", u64)]


class Step(C.Structure):
    _fields_ = [("op", u32), ("n", u32), ("req0", u32), ("flags", u32), ("ext", u64), ("timeout_ns", u64),
                ("ticket", u64)]


class Out(C.Structure):
    _fields_ = [("outcome", u64), ("first_ticket", u64), ("pos", u64), ("n", u64), ("wrap", u64), ("order", u64),
                ("pad0", u64), ("pad1", u64)]


def build_writer(outdir):
    """gcc slot_writer.c into outdir/slot_writer.so"""
    so = os.path.join(outdir, "slot_writer.so")
    subprocess.run(["gcc", "-O2", "-std=gnu99", "-Wall", "-Werror", "-shared", "-fPIC", "-I", DB.INCLUDE, "-o", so,
                    WRITER_SRC], check=True)
    return so


_lib = None
_writer = None


def lib():
    """the compiled probe, loaded once per process"""
    global _lib
    if _lib is None:
        L = DB.load_kernel("header_probe")
        L.hp_copy.argtypes = [vp, vp, vp, u32, vp]
        L.hp_loads.argtypes = [vp, vp, vp, vp, vp]
        L.hp_consumer.argtypes = [vp, vp, u32, vp, u32, vp, u32, vp]
        L.hp_submit.argtypes = [vp, vp, vp, vp, vp, vp, vp, u32, u32, vp]
        L.hp_sizes.restype = C.c_uint
        L.hp_sizes.argtypes = [C.c_uint]
        from apus_b200 import engine as E
        for k, s in enumerate((CopyCase, Entry, Req, Step, Out, E.ConsumerView, E.SubmitterView)):
            assert L.hp_sizes(k) == C.sizeof(s), s
        _lib = L
    return _lib


def writer():
    """the slot writer, built and loaded once per process"""
    global _writer
    if _writer is None:
        W = DB.load(build_writer)
        W.sw_put.restype = u32
        W.sw_put.argtypes = [vp, u32, vp, u64, u64, u32, u32, u16, u64, vp, u32]
        W.sw_reserve.restype = C.c_int
        W.sw_reserve.argtypes = [u32, u64, u64, u64, u64, u64, u64, u64, C.POINTER(u64)]
        W.sw_place.restype = C.c_int
        W.sw_place.argtypes = [u64, u64, u64, u64, C.POINTER(u64)]
        _writer = W
    return _writer


# ---------------------------------------------------------------------------------
# the placement rule, as the comments of include/apus_slot_format.h and apus_submitter.cuh state it
# ---------------------------------------------------------------------------------
def round16(x):
    return (x + 15) & ~15


def accepted(typ, ln):
    return typ in ACCEPTED and ln <= MAX_LEN


def written(typ, ln):
    """(type, len) as the submitter writes a request: itself, or a NOOP with no cmd"""
    return (typ, ln) if accepted(typ, ln) else (NOOP, 0)


def image_bytes(typ, ln):
    return {NOOP: 0, CONFIG: 16, HEAD: 8}.get(typ, 2 + ln)


def ext_bytes(typ, ln):
    """payload-ring bytes of a request as the submitter writes it: round16 of an image above 80 B, else 0"""
    typ, ln = written(typ, ln)
    nb = image_bytes(typ, ln)
    return round16(nb) if nb > SLOT_INLINE else 0


def place(R, head, tail, need):
    """A range of `need` bytes of a ring of R bytes, handed out after `head` bytes with the ring free from counter
    `tail` on.  A range that would cross the ring's end starts at 0 instead, and the bytes skipped count as used.  It
    fits when the bytes in use, the skip and the range together are at most R -- or, on an empty ring, when the range
    alone is.  It is a restart (WRAP) when it skipped, or when it starts at 0 without being the ring's very first range.
    Returns None or (pos, head after, wrap)."""
    p = head % R
    skip = R - p if p + need > R else 0
    if (head - tail) + skip + need > R and not (head == tail and need <= R):
        return None
    start = head + skip
    pos = start % R
    return pos, start + need, int(bool(skip) or (pos == 0 and start != 0))


def reserve(S, R, submitted, head, consumed, tail, n, need):
    """n tickets after `submitted` in a ring of S slots of which `consumed` are taken, and `need` payload bytes:
    None, or (pos, head after, wrap); a reservation with no payload bytes is (0, head, 0)"""
    if submitted + n - consumed > S:
        return None
    if need == 0:
        return 0, head, 0
    return place(R, head, tail, need)


class Placement:
    """The resident submitter's state as apus_submitter_reserve keeps it: tickets, the payload counter, pay_end of every
    slot, the cached consumed count and wrap_next.  `leader_consumed` is the leader's word; the cache is re-read from it
    only when the cached value leaves no room."""

    def __init__(self, S, R, submitted=0, head=0, consumed=None, wrap_next=0):
        self.S, self.R = S, R
        self.submitted, self.head = submitted, head
        self.consumed = submitted if consumed is None else consumed
        self.pay_end = [head] * S
        self.wrap_next = wrap_next

    def tail(self, consumed):
        return self.pay_end[(consumed - 1) % self.S] if consumed else 0

    def reserve(self, n, need, leader_consumed=None):
        """(outcome, first ticket, pos, wrap); NEVER_FITS and the no-room outcome TIMED_OUT change nothing but the
        cache"""
        if n == 0 or n > self.S or need > self.R:
            return NEVER_FITS, 0, 0, 0
        got = reserve(self.S, self.R, self.submitted, self.head, self.consumed, self.tail(self.consumed), n, need)
        if got is None and leader_consumed is not None:
            self.consumed = leader_consumed
            got = reserve(self.S, self.R, self.submitted, self.head, self.consumed, self.tail(self.consumed), n, need)
        if got is None:
            return TIMED_OUT, 0, 0, 0
        pos, head_out, wrap = got
        for k in range(n):
            self.pay_end[(self.submitted + k) % self.S] = head_out if k == n - 1 else self.head
        wrap = int(bool(need) and bool(wrap or self.wrap_next))
        if need:
            self.wrap_next = 0
        first = self.submitted + 1
        self.head, self.submitted = head_out, self.submitted + n
        return OK, first, pos, wrap

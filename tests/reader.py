"""Resident readers for the GPU tests and tools/resident_read_bench.py: tests/devicelogic/resident_reads.cu, compiled with
nvcc for sm_90a into a temporary directory against include/ alone, and a host handle per launch that keeps its fence
log.  Importing this module starts no CUDA context: torch is loaded where it is used."""
import ctypes as C
import time
from collections import namedtuple

import device_build as DB

END_STOP, END_TARGET, END_DEADLINE = 1, 2, 3
LOG_WORDS = 12

vp, u64, u32 = C.c_void_p, C.c_uint64, C.c_uint32

# one logged fence (resident_reads.cu)
Fence = namedtuple("Fence", "slot seq t L K mask outcome F applied T0 t_begin t_end")


class Args(C.Structure):
    """rd_args of resident_reads.cu"""
    _fields_ = [("t0_word", vp), ("log", vp), ("log_cap", u64), ("target", u64), ("timeout_ns", u64),
                ("deadline_ns", u64), ("gap_ns", u64), ("begun", vp), ("out", vp), ("slot0", u32), ("has_cv", u32)]


_lib = None


def lib():
    """the compiled reader, loaded (and its kernel loaded into the context) once per process"""
    global _lib
    if _lib is None:
        L = DB.load_kernel("resident_reads")
        L.rd_launch.argtypes = [vp, vp, vp, C.c_uint, vp]
        L.rd_load.restype = C.c_int
        L.rd_args_size.restype = C.c_uint
        assert L.rd_args_size() == C.sizeof(Args)
        assert L.rd_load() == 0
        _lib = L
    return _lib


class Reader:
    """one resident reader on `rep`: attach, launch resident_reads with `slots` fencing warps on `stream`, read its log
    once it has ended.  `t0_word`: the leader's committed-tickets word (Replica.committed_word()); `consumer`: a started
    resident.Resident of the same replica, whose position the reader waits on after each READY fence"""

    def __init__(self, rep, stream, slots=4, slot0=0, target=1 << 62, timeout_us=20_000_000, deadline_s=60, gap_us=0,
                 log_cap=4096, t0_word=0, consumer=None):
        import torch
        from apus_b200 import engine as E
        dev = torch.device("cuda", rep.device)
        self.rep, self.stream, self.slots, self.log_cap = rep, stream, slots, log_cap
        with torch.cuda.stream(stream):
            self.log = torch.zeros(slots * log_cap * LOG_WORDS, dtype=torch.int64, device=dev)
            self.out = torch.zeros(2 * slots, dtype=torch.int64, device=dev)
        self.begun_t = torch.zeros(slots, dtype=torch.int64).pin_memory()
        stream.synchronize()
        self.cv = consumer.view if consumer is not None else E.ConsumerView()
        self.a = Args(t0_word or None, self.log.data_ptr(), log_cap, target, timeout_us * 1000, int(deadline_s * 1e9),
                      gap_us * 1000, self.begun_t.data_ptr(), self.out.data_ptr(), slot0, 1 if consumer is not None else 0)
        self.view = None

    def start(self, view=None):
        """attach (or, given the `view` of a reader attached already, use it) and launch; returns once the kernel is
        enqueued"""
        self.view = self.rep.reader_attach(self.stream) if view is None else view
        assert lib().rd_launch(C.byref(self.view), C.byref(self.cv), C.byref(self.a), self.slots,
                               self.stream.cuda_stream) == 0
        return self

    def begun(self):
        """fences begun so far, per slot"""
        return [int(x) for x in self.begun_t]

    def done(self):
        return self.stream.query()

    def wait(self, timeout=60):
        t = time.time()
        while not self.stream.query():
            assert time.time() - t < timeout, "the reader did not end in time"
            time.sleep(0.002)

    def detach(self):
        self.rep.reader_detach()
        return self.result()

    def result(self):
        """after the kernel has ended: ({slot: why it ended}, [Fence ...] in slot and seq order)"""
        self.stream.synchronize()
        out = self.out.cpu().tolist()
        lg = self.log.cpu().view(self.slots, self.log_cap, LOG_WORDS).tolist()
        fences, why = [], {}
        for w in range(self.slots):
            why[self.a.slot0 + w] = out[2 * w + 1]
            fences += [Fence(*row) for row in lg[w][:out[2 * w]]]
        return why, fences

"""Submitters that live through take-overs, for tests/test_gpu_submit_takeover.py and tools/resident_failover_bench.py:
tests/devicelogic/takeover_submit.cu, compiled with nvcc for sm_90a into a temporary directory against include/ alone,
and a host handle per launch that keeps its request arrays and reads back the tickets, the term of each reservation and
the NOT_LEADER outcomes it waited out.  The request streams and oracle orders are those of tests/submitter.py.
Importing this module starts no CUDA context: torch is loaded where it is used."""
import ctypes as C

import numpy as np

import device_build as DB

WAIT = 1                                        # TS_WAIT
NOT_LEADER = 4                                  # APUS_SUBMITTER_NOT_LEADER

vp, u64, u32 = C.c_void_p, C.c_uint64, C.c_uint32


class Args(C.Structure):
    """ts_args of takeover_submit.cu"""
    _fields_ = [("types", vp), ("conns", vp), ("req_ids", vp), ("offsets", vp), ("values", vp), ("n", u64),
                ("batch", u32), ("mode", u32), ("timeout_ns", u64), ("tickets", vp), ("terms", vp), ("out", vp)]


_lib = None


def lib():
    """the compiled submitter, loaded (and its kernel loaded into the context) once per process"""
    global _lib
    if _lib is None:
        from apus_b200 import engine as E
        L = DB.load_kernel("takeover_submit")
        L.ts_launch.argtypes = [vp, vp, C.c_uint, vp]
        L.ts_load.restype = C.c_int
        L.ts_args_size.restype = C.c_uint
        L.ts_view_size.restype = C.c_uint
        assert L.ts_args_size() == C.sizeof(Args)
        assert L.ts_view_size() == C.sizeof(E.SubmitterView)
        assert L.ts_load() == 0
        _lib = L
    return _lib


class Submitter:
    """one launch of takeover_submit on `stream` for `requests` [(type, conn, req_id, payload)], `batch` requests per
    reservation, over `ctas` CTAs.  Construct it before the replica kernels are resident (its torch kernels must be
    loaded by then); start() takes the view that attach returned."""

    def __init__(self, stream, requests, batch=16, ctas=1, mode=0, timeout_s=120.0):
        import torch
        dev = stream.device
        n = len(requests)
        offs = np.zeros(n + 1, dtype=np.int64)
        offs[1:] = np.cumsum([len(p) for *_, p in requests])
        vals = np.frombuffer(b"".join(p for *_, p in requests) + b"\0", dtype=np.uint8)

        def t(a):
            return torch.from_numpy(np.ascontiguousarray(a)).to(dev)
        self.stream, self.n, self.ctas, self.view = stream, n, ctas, None
        with torch.cuda.stream(stream):
            self.types = t(np.array([r[0] for r in requests], dtype=np.uint8))
            self.conns = t(np.array([r[1] for r in requests], dtype=np.uint16).view(np.int16))
            self.req_ids = t(np.array([r[2] for r in requests], dtype=np.uint64).view(np.int64))
            self.offsets = t(offs)
            self.values = t(vals.copy())
            self.tickets = torch.zeros(max(n, 1), dtype=torch.int64, device=dev)
            self.terms = torch.zeros(max((n + batch - 1) // batch, 1), dtype=torch.int64, device=dev)
            self.out = torch.zeros(6, dtype=torch.int64, device=dev)
        stream.synchronize()
        self.a = Args(self.types.data_ptr(), self.conns.data_ptr(), self.req_ids.data_ptr(), self.offsets.data_ptr(),
                      self.values.data_ptr(), n, batch, mode, int(timeout_s * 1e9), self.tickets.data_ptr(),
                      self.terms.data_ptr(), self.out.data_ptr())

    def start(self, view):
        """launch on `view`, once per handle"""
        self.view = view
        assert lib().ts_launch(C.byref(self.view), C.byref(self.a), self.ctas, self.stream.cuda_stream) == 0
        return self

    def _out(self):
        self.stream.synchronize()
        return [int(x) for x in self.out.cpu()]

    def result(self):
        """after the kernel has ended: (failure (step, outcome) or None, requests published, tickets [n])"""
        o = self._out()
        return ((o[0] >> 8, o[0] & 0xFF) if o[0] else None), o[1], self.tickets[:self.n].cpu().tolist()

    def terms_of_chunks(self):
        """the term of each chunk's reservation (0 for a chunk never reserved)"""
        self.stream.synchronize()
        return self.terms.cpu().tolist()

    def not_leader(self):
        """the NOT_LEADER outcomes it waited out"""
        return self._out()[3]

    def first_commit_ns(self):
        """%globaltimer ns at which it saw its first chunk committed (WAIT), or 0"""
        return self._out()[4]

    def leading(self):
        """apus_submitter_leading as its CTA 0 ended (the term, or 0 while dormant)"""
        return self._out()[5]

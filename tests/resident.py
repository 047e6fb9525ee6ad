"""Resident consumers for the GPU tests and tools/resident_consumer_bench.py: tests/devicelogic/resident_rows.cu, compiled
with nvcc for sm_90a into a temporary directory against include/apus_consumer.cuh alone, and a host handle per launch
that keeps its rows, its cursor log and its control words.  Importing this module starts no CUDA context: torch is
loaded where it is used."""
import ctypes as C
import time

import device_build as DB

END_STOP, END_TARGET, END_BAD_IDX, END_FULL, END_DEADLINE = 1, 2, 3, 4, 5

vp, u64, u32 = C.c_void_p, C.c_uint64, C.c_uint32


class Args(C.Structure):
    """rr_args of resident_rows.cu"""
    _fields_ = [("idx", vp), ("types", vp), ("conns", vp), ("req_ids", vp), ("lens", vp), ("payloads", vp),
                ("stride", u64), ("row_cap", u64), ("target", u64), ("max_pass", u32), ("pad", u32),
                ("delay_ns", u64), ("deadline_ns", u64), ("rows_pub", vp), ("log", vp), ("log_cap", u64),
                ("ctl", vp), ("pos", vp), ("out", vp)]


_lib = None


def lib():
    """the compiled consumer, loaded (and its kernel loaded into the context) once per process"""
    global _lib
    if _lib is None:
        L = DB.load_kernel("resident_rows")
        L.rr_launch.argtypes = [vp, vp, vp]
        L.rr_load.restype = C.c_int
        L.rr_args_size.restype = C.c_uint
        assert L.rr_args_size() == C.sizeof(Args)
        assert L.rr_load() == 0
        _lib = L
    return _lib


class Resident:
    """one resident consumer on `rep`: attach, launch resident_rows on `stream`, read its rows once it has ended"""

    def __init__(self, rep, stream, stride=1500, row_cap=1 << 16, max_pass=256, delay_ns=0, target=1 << 62,
                 deadline_s=60, log_cap=1 << 16):
        import torch
        dev = torch.device("cuda", rep.device)
        self.rep, self.stream, self.stride, self.row_cap = rep, stream, stride, row_cap
        with torch.cuda.stream(stream):
            self.idx = torch.zeros(row_cap, dtype=torch.int64, device=dev)
            self.types = torch.zeros(row_cap, dtype=torch.uint8, device=dev)
            self.conns = torch.zeros(row_cap, dtype=torch.int16, device=dev)
            self.req_ids = torch.zeros(row_cap, dtype=torch.int64, device=dev)
            self.lens = torch.zeros(row_cap, dtype=torch.int16, device=dev)
            self.payloads = torch.zeros((row_cap, stride), dtype=torch.uint8, device=dev)
            self.log = torch.zeros(3 * log_cap, dtype=torch.int64, device=dev)
            self.out = torch.zeros(3, dtype=torch.int64, device=dev)
        self.rows_pub = torch.zeros(1, dtype=torch.int64).pin_memory()
        self.ctl = torch.zeros(2, dtype=torch.int32).pin_memory()
        self.pos = torch.zeros(3, dtype=torch.int64).pin_memory()
        self.a = Args(self.idx.data_ptr(), self.types.data_ptr(), self.conns.data_ptr(), self.req_ids.data_ptr(),
                      self.lens.data_ptr(), self.payloads.data_ptr(), stride, row_cap, target, max_pass, 0, delay_ns,
                      int(deadline_s * 1e9), self.rows_pub.data_ptr(), self.log.data_ptr(), log_cap,
                      self.ctl.data_ptr(), self.pos.data_ptr(), self.out.data_ptr())
        self.view = None

    def start(self):
        """attach and launch; returns once the kernel is enqueued"""
        self.view = self.rep.consumer_attach(self.stream)
        assert lib().rr_launch(C.byref(self.view), C.byref(self.a), self.stream.cuda_stream) == 0
        return self

    def rows_so_far(self):
        return int(self.rows_pub[0])

    def wait_rows(self, n, timeout=60):
        t = time.time()
        while self.rows_so_far() < n:
            assert time.time() - t < timeout, (self.rows_so_far(), n)
            time.sleep(0.001)

    def snapshot_position(self, timeout=30):
        """ask the kernel to stop examining and write its position: (cursor, next idx, rows)"""
        self.ctl[1] = 0
        self.ctl[0] = 1
        t = time.time()
        while int(self.ctl[1]) != 1:
            assert time.time() - t < timeout
            time.sleep(0.0005)
        return int(self.pos[0]), int(self.pos[1]), int(self.pos[2])

    def resume(self):
        self.ctl[0] = 2

    def detach(self):
        self.rep.consumer_detach()
        return self.result()

    def result(self):
        """after the kernel has ended: (why, rows, cursor log [(cursor, rows, %globaltimer ns)])"""
        self.stream.synchronize()
        why, n, nlog = (int(x) for x in self.out.cpu())
        lg = self.log[:3 * nlog].cpu().view(-1, 3).tolist()
        return why, n, [tuple(x) for x in lg]

    def rows(self):
        """the rows written, as consumers.Consumer keeps them: (idx, type, conn, req_id, cmd bytes)"""
        self.stream.synchronize()
        n = int(self.out.cpu()[1])
        idx, ty, co, rq, ln = (t[:n].cpu().numpy() for t in (self.idx, self.types, self.conns, self.req_ids, self.lens))
        pl = self.payloads[:n].cpu().numpy()
        return [(int(idx[q]), int(ty[q]), int(co[q]) & 0xFFFF, int(rq[q]), pl[q, :int(ln[q]) & 0xFFFF].tobytes())
                for q in range(n)]

"""apus_b200 -- H100-native Paxos log replication behind APUS's operator surface.

The product is the C-ABI shared library `libapus_gpu.so` (include/apus_gpu.h),
built from apus_b200/csrc for sm_90a (H100).  This package only binds it with ctypes for
tests, the benchmark and the launch scripts; there is no Python or CPU fallback:
importing `apus_b200.engine` fails loudly when the library has not been built.
"""
from .engine import (  # noqa: F401
    APUS_OK, APUS_ERROR, APUS_RETRY, NOOP, CSM, CONFIG, HEAD, CONNECT, SEND, CLOSE,
    RING_HOST_MAPPED, RING_DEVICE, LOG_SIZE, ApusError, Group, Replica, lib, load_library,
    F_DEVICE_APPLY, CONSUME_BAD_IDX,
)

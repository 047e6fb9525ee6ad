"""The header probe's host side without a GPU: the slot writer (tests/hostlogic/slot_writer.c) builds and writes a slot
where the format puts its fields, and header_probe's own statement of the submitter's placement rule agrees with
slot_reserve and slot_place of include/apus_slot_format.h compiled as C, over random scripts on rings of power-of-two
and other sizes.  The probe's compile test is in tests/test_public_headers.py."""
import ctypes as C
import shutil

import numpy as np
import pytest

import header_probe as HP


@pytest.mark.skipif(shutil.which("gcc") is None, reason="needs gcc")
def test_slot_writer_builds_and_writes_the_format():
    W = HP.writer()
    slots = np.full(4 * 128, 0xEE, dtype=np.uint8)
    pay = np.full(4096, 0xEE, dtype=np.uint8)
    cmd = np.arange(200, dtype=np.uint8)
    assert W.sw_put(slots.ctypes.data, 4, pay.ctypes.data, 6, 0, 0, HP.SEND, 0x1234, 0x0102030405060708,
                    cmd.ctypes.data, 60) == 62
    s = slots[128:256]                                  # ticket 6 of 4 slots: slot 1
    assert s[:16].tobytes() == (0x0102030405060708).to_bytes(8, "little") + (HP.SEND << 24).to_bytes(4, "little") + \
        (60).to_bytes(2, "little") + (0x1234).to_bytes(2, "little")
    img = bytes([60, 0]) + cmd[:60].tobytes()
    assert s[16:48].tobytes() == img[:32] and s[64:94].tobytes() == img[32:]
    assert s[48:64].tobytes() == (6).to_bytes(16, "little") and s[112:128].tobytes() == (6).to_bytes(16, "little")
    assert (pay == 0xEE).all()
    assert W.sw_put(slots.ctypes.data, 4, pay.ctypes.data, 7, 1024, 1, HP.CSM, 1, 9, cmd.ctypes.data, 150) == 152
    s = slots[256:384]
    assert s[8:12].view("<u4")[0] == HP.SLOT_EXT | HP.SLOT_WRAP | HP.CSM << 24 | 1024 // 16
    assert pay[1024:1176].tobytes() == bytes([150, 0]) + cmd[:150].tobytes() and (pay[1176:] == 0xEE).all()


def c_reserve(W, S, R, sub, head, consumed, tail, n, need):
    out = (C.c_uint64 * 3)()
    rc = W.sw_reserve(S, R, sub, head, consumed, tail, n, need, out)
    return None if rc else tuple(int(x) for x in out)


def c_place(W, R, head, tail, need):
    out = (C.c_uint64 * 3)()
    rc = W.sw_place(R, head, tail, need, out)
    return None if rc else tuple(int(x) for x in out)


@pytest.mark.skipif(shutil.which("gcc") is None, reason="needs gcc")
@pytest.mark.parametrize("R", [1 << 17, 33 * 4096, 4096 * 37, 1 << 20])
def test_placement_model_agrees_with_the_header(R):
    """random scripts of reservations and consumption: every placement of the model is slot_reserve's, including the
    exact fits at R and the skips one byte over; and slot_place on every edge of the ring"""
    W = HP.writer()
    rng = np.random.default_rng(R)
    for p in (0, 16, R - 4096, R - 16, R - 1, R // 2):
        for need in (1, 15, 16, R - p - 1, R - p, R - p + 1, R - p + 16, R, R + 1):
            for used in (0, 16, R - need - 16, R // 3):
                if need <= 0 or used < 0:
                    continue
                head = 3 * R + p
                assert HP.place(R, head, head - used, need) == c_place(W, R, head, head - used, need), (p, need, used)
    assert c_place(W, R, 5 * R, 5 * R, R) == (0, 6 * R, 1) and HP.place(R, 0, 0, R) == (0, R, 0)
    steps = 0
    for script in range(40):
        S = int(rng.choice([8, 64, 1024]))
        m = HP.Placement(S, R, submitted=int(rng.integers(0, 1 << 40)), head=int(rng.integers(0, 1 << 40)) // 16 * 16,
                         wrap_next=int(rng.integers(0, 2)))
        for _ in range(300):
            steps += 1
            if rng.random() < 0.3 and m.consumed < m.submitted:
                m.consumed = min(m.submitted, m.consumed + int(rng.integers(1, S + 1)))
            n = int(rng.integers(1, S + 1)) if rng.random() < 0.3 else int(rng.integers(1, 9))
            kind = rng.random()
            if kind < 0.2:
                need = 0
            elif kind < 0.3:
                need = int(rng.integers(1, R + 1))
            else:
                need = 16 * int(rng.integers(1, R // 64))
            tail = m.tail(m.consumed)
            want = c_reserve(W, S, R, m.submitted, m.head, m.consumed, tail, n, need)
            assert HP.reserve(S, R, m.submitted, m.head, m.consumed, tail, n, need) == want, (script, n, need)
            before = (m.submitted, m.head, m.wrap_next)
            oc, first, pos, wrap = m.reserve(n, need)
            if want is None:
                assert oc == HP.TIMED_OUT and (m.submitted, m.head, m.wrap_next) == before
                continue
            assert oc == HP.OK and (pos, m.head) == want[:2] and first == before[0] + 1
            assert wrap == int(bool(need) and bool(want[2] or before[2]))
            assert m.pay_end[(m.submitted - 1) % S] == m.head
            if rng.random() < 0.05:
                m.wrap_next = 1
    assert steps == 40 * 300

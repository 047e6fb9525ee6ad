"""GPU parity for 512-entry tiles and the batch scan of T1: laps of the benchmark's own request shape (64 B payload,
128 B stride: uniform claims, closed-form prefix sums) with pruning, laps of mixed shapes (claims of up to 512 slots
through the CTA-wide scan, next to uniform ones), and a check that claims really grow past 256 slots.  Marked gpu."""
import numpy as np
import pytest

import engine_util as EU
import streams as S
from engine_util import MODES, devices_for, eng, wrap_case  # noqa: F401

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(180)]


def mixed_stream(kind, seed, L):
    """64 B SENDs for 4.5 laps, and in between either a 200 B SEND every 37th request (stride 264: a claim that holds
    one is not uniform and takes the CTA-wide scan) or a CLOSE + CONNECT every 53rd (64 B entries: the 128 B entries
    leave the 128 B grid, so that wraps leave gaps inside a claim)"""
    rng = np.random.default_rng(seed)
    out = [(S.CONNECT, 0, 1, b"")]
    rid, nbytes, i = 2, 64, 0
    while nbytes < 4.5 * L:
        if kind == "mix200" and i % 37 == 36:
            ln = 200
        else:
            ln = 64
        if kind == "churn" and i % 53 == 52:
            out += [(S.CLOSE, 0, rid, b""), (S.CONNECT, 0, rid + 1, b"")]
            rid += 2
            nbytes += 128
        out.append((S.SEND, 0, rid, rng.integers(0, 256, ln, dtype=np.uint8).tobytes()))
        rid += 1
        nbytes += 64 + ln
        i += 1
    return out


# the u64 and mixed cases run engine_util.wrap_laps_with_pruning, as test_gpu_parity.test_wrap_laps_with_pruning does:
# about a third of the ring per launch, pruning at quiescent points, every byte against the oracle, and the holes of the
# last lap non-zero (what catches a prefill that stored zeros or loaded the wrong chunk)
@pytest.mark.parametrize("n,L,kind,seed,mode,step,ctas,ring", [
    wrap_case(5, 1 << 18, "u64", 90, "index_earlyack", ctas=1, id="5-262144-90-index_earlyack-1-host"),
    wrap_case(5, 1 << 18, "u64", 91, "walk_fenced", ctas=16, id="5-262144-91-walk_fenced-16-host"),
    # requests in HBM, one bulk call per launch: claims of 512 slots
    wrap_case(3, 1 << 18, "u64", 92, "index_earlyack", ctas=1, ring="device", id="3-262144-92-index_earlyack-1-device"),
])
def test_u64_laps(eng, orc, n, L, kind, seed, mode, step, ctas, ring):
    """the benchmark's request shape over 4.5 laps of a small ring with pruning"""
    EU.wrap_laps_with_pruning(eng, orc, n, L, kind, seed, mode, step, ctas, ring)


@pytest.mark.parametrize("kind,ctas,ring", [("mix200", 1, "device"), ("mix200", 4, "host"), ("churn", 1, "device"),
                                            ("churn", 16, "host")])
def test_mixed_shapes_laps(eng, orc, kind, ctas, ring):
    EU.wrap_laps_with_pruning(eng, orc, 3, 1 << 17, kind, 93, "index_earlyack", None, ctas, ring, stream_of=mixed_stream)


def test_claims_exceed_256_slots(eng, orc):
    """one bulk launch from a device ring into one worker CTA: the claims hold more than 256 slots on average"""
    n, L, nreq = 3, 1 << 24, 1 << 16
    payloads = np.random.default_rng(94).integers(0, 256, size=nreq * 64, dtype=np.uint8)
    with eng.Group(n, devices=devices_for(eng, n), log_size=L, ring_mode=eng.RING_DEVICE, ring_slots=1 << 17,
                   ring_bytes=1 << 20, leader_ctas=1, flags=MODES["index_earlyack"]) as g:
        g.prologue()
        g.submit(S.CONNECT, 0, 1, b"")
        g.submit_uniform(nreq, 64, 0, 2, payloads)
        g.run(timeout_ms=60_000)
        st = g.leader.stats()
        assert st["tickets_committed"] == nreq + 2
        claims = st["turn_ns"][6]
        assert claims > 0
        assert st["tickets_committed"] / claims > 256, (st["tickets_committed"], claims)

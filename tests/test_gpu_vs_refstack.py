"""The CUDA engine against the reference ITSELF, on the same box in the same test: the reference's unmodified
election / replication / commit code (oracle/_ref/libref_stack.so on the verbs shim, N host processes) and the GPU
engine (through the C ABI) are fed the same request stream; the logs they leave behind must be identical --
leader copy: every byte, reply bytes included; follower copies: every byte outside reply[0..12] (H5 mask,
SURVEY.md s8c) plus the follower's own ack byte (I7).  Leader index and term are whatever the reference's
election produced."""
import numpy as np
import pytest

import orc as O
import refstack as R
from engine_util import eng  # noqa: F401

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(300)]


@pytest.mark.parametrize("n,nconn,nreq,plen", [(3, 2, 300, 64), (5, 3, 200, 128), (3, 1, 120, -3000), (7, 4, 400, 64)])
def test_engine_log_equals_reference_log(eng, n, nconn, nreq, plen):
    if not R.available():
        pytest.skip("oracle/_ref/libref_stack.so absent (built only where /root/reference exists)")
    try:
        rr = R.run(n, nconn, nreq, plen, prune=1000.0)
    except RuntimeError as e:
        # the reference stack needs process_vm_writev between sibling processes; a box that forbids it cannot host the
        # CPU side of this comparison (the golden vectors of the same runs still apply: test_gpu_parity.py)
        pytest.skip(f"the reference stack could not run on this box: {str(e)[:200]}")
    lead, term = rr["leader"], rr["term"]
    nd = eng.lib().apus_device_count()
    with eng.Group(n, devices=[i % nd for i in range(n)], leader=lead, term=term, log_size=O.LOG_SIZE) as g:
        g.prologue()
        g.submit_stream(R.expected_stream(lead, nconn, nreq, plen))
        g.run()
        end = rr["results"][lead]["offsets"]["end"]
        for i in range(n):
            ro, eo = rr["results"][i]["offsets"], g.replicas[i].offsets()
            assert (eo["end"], eo["commit"], eo["head"], eo["len"]) == (ro["end"], ro["commit"], ro["head"], ro["len"]), (i, eo, ro)
            if i == lead:
                assert eo["tail"] == ro["tail"]
            got, want = g.replicas[i].image(0, end), rr["images"][i]
            ents = O.walk_entries(want, 0, end, O.LOG_SIZE)
            if i != lead:
                for off, _ in ents:
                    assert got[off + 28 + i] == 1 and want[off + 28 + i] == 1
                got, want = O.mask_replies(got, ents), O.mask_replies(want, ents)
            if not np.array_equal(got, want):
                dd = np.nonzero(got != want)[0]
                raise AssertionError(f"replica {i} (leader {lead}, term {term}): {len(dd)} bytes differ from the reference, "
                                     f"first at {int(dd[0])}: engine {got[dd[0]]} reference {want[dd[0]]}")
        assert g.leader.committed() == len(ents)

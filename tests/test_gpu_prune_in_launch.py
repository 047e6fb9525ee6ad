"""Device-side log pruning inside ONE launch that laps the ring many times, byte for byte against the CPU oracle.
Every follower's host applies the log (APUS_F_HOST_APPLY) through a recorder (tests/autoprune_replay.py): it reads
each committed range before it reports it as applied, and the leader's pruning rule reads those reports, so every
entry of every lap is read before the leader may overwrite it.  The recordings are cut at every read, replayed into
the oracle, every read is compared with the oracle as it was then, and every HEAD entry is checked against the reports
made before it was read.  At the end every byte and offset of every replica.  Marked gpu."""
import time

import numpy as np
import pytest

import autoprune_replay as AR
import engine_util as EU
import orc as O
import streams as S
from engine_util import MODES, eng, submit_all  # noqa: F401

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900)]

FOREVER = EU.FOREVER


def _case(n, L, kind, mode, ctas, ring, lagging, laps, id):
    return pytest.param(n, L, kind, mode, ctas, ring, lagging, laps, id=id)


CASES = [
    # the benchmark's shape: 5 replicas, 64 B payloads written by the fill kernel into the HBM ring, 16 leader CTAs,
    # claims of 512 slots; prompt hosts, so the leader prunes while every follower's report moves under it
    _case(5, 4 << 20, "synth64", "index_earlyack", 16, "synth", False, 8.5, "a-bench-shape-n5-4M-synth-ctas16"),
    # stride 1024 from the HBM ring: the holes-only prefill, with the HEAD entry at j == 0; walking followers
    _case(5, 1 << 18, "u960", "walk_fenced", 16, "device", False, 6.5, "b-u960-n5-256K-walk_fenced-ctas16"),
    # the drop-in's shape: 0..1500 B with connection churn on two CTAs, fed while resident through a payload ring that
    # laps too; ghost headers, and prunes to the lagging host's report while the other is at the commit
    _case(3, 1 << 18, "ragged1500", "index_fenced", 2, "host", True, 6.5, "c-ragged1500-n3-256K-index_fenced-ctas2-lag"),
    # HEAD pairs.  After a HEAD placed alone at pos0 (its sub-tile holds no entry: 64 + es > min(L - pos0, L - d - 65),
    # d the distance from the new head to end) the next entry must block at the new head and end, else the leader
    # places it.  The HEAD freed at least L/8 and E2 had left fewer than es + 65 bytes free, so the entry blocks only
    # if es > L/8 - 64 (no-wrap side: es > L - (used - L/8 + 64) - 65 with used <= L - 65; the wrap side gives the
    # same bound, the skipped stretch counting as used).  On 32 KiB that is 4032 B: most 3..9 KiB entries qualify
    _case(3, 1 << 15, "sized3k9k", "index_earlyack", 4, "host", True, 6.5, "d-sized3k9k-n3-32K-ctas4-lag-pairs"),
]


def _stream(kind, L, laps):
    if kind == "synth64":
        return None
    if kind == "u960":
        return S.uniform_stream(int(laps * L / 1024) + 1, 960, conns=1, seed=95)
    if kind == "ragged1500":
        return S.ragged_stream(int(laps * 1.15 * L / 814) + 1, 1500, conns=3, seed=97, close_every=20)
    return S.sized_stream(int(laps * L / 6200) + 1, 3072, 9216, seed=98)


@pytest.mark.parametrize("n,L,kind,mode,ctas,ring,lagging,laps", CASES)
def test_prune_in_one_launch_replayed(eng, orc, n, L, kind, mode, ctas, ring, lagging, laps):
    from apus_b200 import engine as E
    seed = 0xA070
    if kind == "synth64":
        nreq = int(laps * L / 128)
        stream = [(S.CONNECT, 0, 1, b"")] + [(S.SEND, 0, 2 + i, E.synth_payload(seed, 2 + i, 64)) for i in range(nreq)]
    else:
        stream = _stream(kind, L, laps)
    requests = [(O.CONFIG, 0, 0, b"")] + stream
    ring_mode = eng.RING_HOST_MAPPED if ring == "host" else eng.RING_DEVICE
    slots = 1 << max(14, len(requests).bit_length())
    ring_bytes = (1 << 17) if kind == "ragged1500" else 8 << 20
    reps = EU.host_apply_replicas(eng, n, L, MODES[mode], ring_mode, slots, ring_bytes, ctas)
    lead = reps[0]
    # the lagging host (the last follower) reads after a pause and reports a sixty-fourth of the ring at most
    recs = [AR.Recorder(reps[j], j, L, *((L // 64, 0.002) if lagging and j == n - 1 else (None, 0.0)))
            for j in range(1, n)]
    rp = AR.Replay(orc, n, L)
    t_start = time.time()
    try:
        for r in recs:
            r.start()
        t = lead.submit(E.CONFIG, 0, 0, E.cid_image(n))
        fed_later = kind == "ragged1500"
        if not fed_later:
            if kind == "synth64":
                lead.submit(S.CONNECT, 0, 1, b"")
                t = lead.submit_synth(nreq, S.SEND, 0, 2, 64, seed) + nreq - 1
            else:
                t = submit_all(lead, stream)
        EU.launch_each(eng, reps, FOREVER)
        if fed_later:
            t = submit_all(lead, stream)
        deadline = time.time() + 300
        while lead.committed() < t:
            for r in recs:
                r.check()
            assert time.time() < deadline, f"committed {lead.committed()} of {t}; leader {lead.offsets()} {lead.stats()}"
            time.sleep(0.005)
        final = lead.offsets()["end"]
        for r in recs:
            r.finish(final)
        EU.stop_each(eng, reps)
        t_run = time.time() - t_start

        AR.replay_recordings(rp, [r.rec for r in recs], requests)
        assert rp.pos == len(requests)
        for r in recs:                                   # every host read [0, the final end) (gaps fail the replay)
            assert max(s + len(b) for s, b, _ in r.rec.segs) == rp.written
            assert r.rec.reports[-1][0] == rp.written
        assert rp.written >= (8 if kind == "synth64" else 6) * L, rp.written / L
        # every byte and offset of every replica, reply bytes included; a follower's apply is its host's last report
        for i, r in enumerate(reps):
            eo, oo = r.offsets(), rp.c.offsets(i)
            for key in ("end", "commit", "head"):
                assert eo[key] == oo[key], (i, key, eo, oo)
            assert eo["apply"] == (oo["apply"] if i == 0 else final), (i, eo)
            ei, oi = r.image(), rp.c.image(i)
            d = np.nonzero(ei != oi)[0]
            assert len(d) == 0, f"replica {i}: {len(d)} bytes differ, first at {int(d[0])}"
        assert reps[0].offsets()["tail"] == rp.c.offsets(0)["tail"]
        st = lead.stats()
        assert st["bytes_replicated"] == rp.c.bytes_replicated()
        assert st["auto_heads"] == len(rp.heads), (st["auto_heads"], len(rp.heads))
        assert len(rp.heads) >= int(rp.written / L), (len(rp.heads), rp.written / L)     # at least one per lap
        AR.assert_heads_have_teeth(rp, rp.c.image(0))
        if kind == "sized3k9k":
            assert rp.pairs >= 1, f"no HEAD pair in {len(rp.heads)} HEAD entries"
        recorded = sum(len(b) for r in recs for _, b, _ in r.rec.segs)
        print(f"{rp.written / L:.2f} laps in one launch, {len(rp.heads)} HEAD entries replayed, {rp.pairs} pairs, "
              f"{recorded} bytes recorded in {sum(len(r.rec.segs) for r in recs)} reads, run {t_run:.1f} s, "
              f"total {time.time() - t_start:.1f} s")
    finally:
        for r in recs:
            r.stop.set()
        EU.stop_each(eng, reps)
        for r in reps:
            r.close()
        rp.close()

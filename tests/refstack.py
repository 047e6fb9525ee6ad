"""Run the reference's OWN software stack (oracle/_ref/libref_stack.so: unmodified src/dare/*.c + proxy.c +
db-interface.c + config-*.c with real libev/libconfig/BerkeleyDB, on oracle/verbs_shim) as N replica processes
and collect what it produced: every replica's log image and offsets, the followers' replayed byte streams,
the leader's latencies.  Test infrastructure (tests/ and bench.py's reference arm only)."""
import json
import os
import subprocess
import sys
import tempfile

import numpy as np

import streams as S

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
STACK = os.path.join(ROOT, "oracle", "_ref", "libref_stack.so")


def available():
    return os.path.exists(STACK)


def ragged_len(i, maxlen):
    """refstack_ragged_len() of oracle/ref_stack_access.c; 0 becomes 1 (a 0-byte read() is never forwarded)."""
    v = ((i * 2654435761) >> 7) % (maxlen + 1)
    return v or 1


def expected_stream(leader, nconn, nreq, plen):
    """The request stream refstack_drive() issues with ONE application thread, as (type, clt_id, req_id, payload):
    CONNECTs, SENDs round-robin, CLOSEs; connection_id = (leader_idx << 8) | k (proxy.c:101-106,123),
    req_id = per-connection counter from 1 (proxy.c:121-133)."""
    out, req = [], [0] * nconn
    for c in range(nconn):
        req[c] += 1
        out.append((S.CONNECT, (leader << 8) | c, req[c], b""))
    for i in range(nreq):
        c = i % nconn
        n = plen if plen >= 0 else ragged_len(i, -plen)
        n = n or 1
        req[c] += 1
        out.append((S.SEND, (leader << 8) | c, req[c], bytes(((i * 31 + k) & 0xFF) for k in range(n))))
    for c in range(nconn):
        req[c] += 1
        out.append((S.CLOSE, (leader << 8) | c, req[c], b""))
    return out


class Disturbed(RuntimeError):
    """The reference group did not come up as one leader + n-1 followers (its start-up election removes a server that is
    slow to answer -- check_failure_count -- which happens on a loaded box), or a replica produced nothing."""


def run(n, nconn, nreq, plen, attempts=3, **kw):
    """Returns dict(leader, term, results[i], images[i] (np.uint8 arrays of entries[0..end)), logs[i]).  A run whose group
    was disturbed at start-up (see Disturbed) is repeated, `attempts` times at most: the callers compare a quiet group's
    logs with the oracle, not the reference's behaviour under CPU starvation."""
    for k in range(attempts):
        if k and kw.get("keep"):
            subprocess.run(["rm", "-rf", kw["keep"]])       # what the disturbed attempt left behind
        try:
            return _run_once(n, nconn, nreq, plen, **kw)
        except Disturbed as e:
            sys.stderr.write(f"[refstack] attempt {k + 1}: {str(e)[:300]}\n")
            if k == attempts - 1:
                raise


def _run_once(n, nconn, nreq, plen, threads=1, prune=None, timeout=120, keep=None, steps=1, images=True, lib=None, transport=None):
    d = keep or tempfile.mkdtemp(prefix="apus-refstack-")
    os.makedirs(d, exist_ok=True)
    env = dict(os.environ)
    if prune is not None:
        env["REFSTACK_PRUNE"] = str(prune)
    env["REFSTACK_STEPS"] = str(steps)
    if lib:
        env["REFSTACK_LIB"] = lib                    # e.g. "libref_stack_O2.so": the same sources built with -O2
    if not images:
        env["REFSTACK_NO_IMAGE"] = "1"
    if transport:
        env["APUS_SHIM_TRANSPORT"] = transport       # "shm": log writes are memcpys into a shared mapping (verbs_shim.c)
    procs = [subprocess.Popen([sys.executable, os.path.join(HERE, "refstack_worker.py"), str(i), str(n), str(nconn),
                               str(nreq), str(plen), d, str(threads)], env=env, stdout=subprocess.PIPE,
                              stderr=subprocess.STDOUT) for i in range(n)]
    outs = []
    try:
        for p in procs:
            outs.append(p.communicate(timeout=timeout)[0].decode(errors="replace"))
    except subprocess.TimeoutExpired:
        raise Disturbed(f"the reference group did not finish within {timeout} s") from None
    finally:
        for p in procs:
            if p.poll() is None:
                p.kill()
    res, imgs, logs = [], [], []
    for i in range(n):
        path = os.path.join(d, f"result{i}.json")
        lp = os.path.join(d, f"node{i}", "dare.log")
        logs.append(open(lp, errors="replace").read() if os.path.exists(lp) else "")
        if not os.path.exists(path):
            raise Disturbed(f"reference replica {i} produced no result:\n{outs[i][-1500:]}\n{logs[i][-1500:]}")
        res.append(json.load(open(path)))
        ip = os.path.join(d, f"image{i}.bin")
        imgs.append(np.fromfile(ip, dtype=np.uint8) if os.path.exists(ip) else None)
    leaders = [r["idx"] for r in res if r["leader"]]
    if len(leaders) != 1:
        raise Disturbed(f"expected one leader, got {leaders}:\n" + "\n".join(l[-800:] for l in logs))
    # (counted by each replica when it wrote its result: the tear-down that follows logs removals of its own)
    removed = [i for i in range(n) if res[i].get("log_marks", {}).get("removals", 0)]
    if removed:
        raise Disturbed(f"the reference removed a server from the group while it ran (logs of {removed}); not a quiet run")
    # a follower the leader never reached at start-up (it did not grant log access within the settle time) waits in vain
    # for the leader's end and reports an empty log, while the other followers make the majority
    lead_o = res[leaders[0]].get("offsets", {})
    empty = [i for i in range(n) if i != leaders[0] and lead_o.get("end") != lead_o.get("len")
             and res[i].get("offsets", {}).get("end") == res[i].get("offsets", {}).get("len")]
    if empty:
        raise Disturbed(f"followers {empty} hold an empty log while the leader holds entries (not reached at start-up); "
                        "not a quiet run")
    led = sum(r.get("log_marks", {}).get("leaderships", 1 if r["leader"] else 0) for r in res)
    if led != 1:
        raise Disturbed(f"{led} leaderships in one run (a leader was deposed during start-up: one CONFIG entry per term); not a quiet run")
    if keep is None:
        subprocess.run(["rm", "-rf", d])
    return dict(leader=leaders[0], term=res[leaders[0]]["offsets"]["term"], results=res, images=imgs, logs=logs)

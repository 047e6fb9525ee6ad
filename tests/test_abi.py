"""CPU-side checks of the drop-in boundary: the shared library loads and exports every symbol include/apus_gpu.h
declares, the binding gives each the header's signature, the outcome values and the layout words the consumer calls
use stay where the header and apus_layout.h put them, and without a GPU every entry point fails loudly (there is no
CPU fallback)."""
import ctypes as C
import os
import re
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# C scalar types of the header -> the ctypes type that passes them at full width
SCALARS = {"uint8_t": C.c_uint8, "uint16_t": C.c_uint16, "uint32_t": C.c_uint32, "uint64_t": C.c_uint64,
           "int": C.c_int, "int64_t": C.c_int64, "size_t": C.c_size_t}


@pytest.fixture(scope="module")
def built():
    import __graft_entry__ as g
    g.build()
    from apus_b200 import engine
    return engine


def header(strip_comments=False):
    txt = open(os.path.join(ROOT, "include", "apus_gpu.h")).read()
    return re.sub(r"/\*.*?\*/", "", txt, flags=re.S) if strip_comments else txt


def declared_symbols():
    return sorted(set(re.findall(r"\b(apus_[a-z_0-9]+)\s*\(", header(strip_comments=True))))


def prototypes():
    """{name: (return type, [parameter declarations])} of every function the header declares"""
    out = {}
    for m in re.finditer(r"^([A-Za-z_][\w \t*]*?)\s*\b(apus_\w+)\s*\(([^()]*)\)\s*;", header(strip_comments=True),
                         flags=re.M):
        params = [" ".join(p.split()) for p in m.group(3).split(",")]
        out[m.group(2)] = (" ".join(m.group(1).split()), [] if params == ["void"] else params)
    return out


def layout_block(name):
    txt = open(os.path.join(ROOT, "apus_b200", "csrc", "apus_layout.h")).read()
    return txt[txt.index(f"typedef struct {name} {{"):txt.index(f"}} {name}_t;")]


def test_header_symbols_exported(built):
    lib = built.load_library()
    syms = declared_symbols()
    assert len(syms) >= 20
    for s in syms:
        assert hasattr(lib, s), f"{s} declared in include/apus_gpu.h but not exported"
    assert sorted(built.EXPORTS) == syms
    assert lib.apus_abi_version() == 2


def test_signatures_match_the_header(built):
    """every prototype of the header has its entry in the binding's table: the same number of parameters, the same
    scalar widths, a pointer type for each pointer or array, and the return type"""
    protos = prototypes()
    assert sorted(protos) == declared_symbols()
    assert sorted(built.SIGNATURES) == sorted(protos)

    def is_pointer(t):
        return t in (C.c_void_p, C.c_char_p) or issubclass(t, C._Pointer)

    for name, (ret, params) in protos.items():
        restype, argtypes = built.SIGNATURES[name]
        if ret == "const char *":
            assert restype is C.c_char_p, name
        elif "*" in ret:
            assert restype is C.c_void_p, (name, ret, restype)
        else:
            assert restype is (None if ret == "void" else SCALARS[ret]), (name, ret, restype)
        assert len(argtypes) == len(params), (name, params, argtypes)
        for k, (p, t) in enumerate(zip(params, argtypes)):
            if "*" in p or "[" in p:
                assert is_pointer(t), (name, k, p, t)
            else:
                assert t is SCALARS[p.rsplit(" ", 1)[0]], (name, k, p, t)


def test_snapshot_call_prototypes():
    """the exact prototypes of apus_consume_mark and apus_consume_seed"""
    hdr = header()
    assert re.search(r"int\s+apus_consume_mark\(apus_replica_t \*r, uint64_t \*mark, void \*stream\);", hdr)
    assert re.search(r"int\s+apus_consume_seed\(apus_replica_t \*r, uint64_t cursor_offset, uint64_t next_idx\);", hdr)


def test_wait_outcomes_match_the_header(built):
    """the outcomes of consume waits and read fences: exactly these four defines, and the binding's WAIT_* are them"""
    defs = dict(re.findall(r"#define\s+(APUS_WAIT_\w+)\s+(\S+)", header()))
    assert defs == {"APUS_WAIT_READY": "0u", "APUS_WAIT_TIMED_OUT": "1u", "APUS_WAIT_RELEASED": "2u",
                    "APUS_WAIT_NOT_LEADER": "3u"}, defs
    assert (built.WAIT_READY, built.WAIT_TIMED_OUT, built.WAIT_RELEASED, built.WAIT_NOT_LEADER) == (0, 1, 2, 3)


def test_the_seed_word_takes_a_spare_word():
    """cons_seeded follows cons_on, in what was padding: every word before it keeps its offset, the block its size"""
    block = layout_block("apus_ctrl")
    tail = re.findall(r"uint64_t\s+(\w+)(?:\[(\d+)\])?;", block[block.index("uint64_t cons_rec"):])
    assert tail == [("cons_rec", "2"), ("cons_cur", "2"), ("cons_on", ""), ("cons_seeded", ""), ("pad4", "10")], tail


def test_fence_status_words_take_spare_host_words():
    at, off = {}, 0
    for name, cnt in re.findall(r"uint64_t\s+(\w+)(?:\[(\d+)\])?;", layout_block("apus_hostwords")):
        at[name] = off
        off += 8 * (int(cnt) if cnt else 1)
    # the words after the consume waits' three stay where they were: stop at 8 * 32
    assert at["fence_outcome"] == at["cons_wait_avail"] + 8 and at["fence_index"] == at["fence_outcome"] + 8
    assert at["pad1"] + 8 == 256, at


def test_null_replica_is_refused(built):
    """every call that checks which replicas may consume, and the attach and detach of every resident kernel, refuses a
    null replica first, whatever its other arguments; an attach writes nothing to the view"""
    lib = built.load_library()
    buf = (C.c_uint64 * 16)()
    a = C.addressof(buf)
    w = [C.byref(C.c_uint64()) for _ in range(4)]
    views = [built.ConsumerView(), built.SubmitterView(), built.ReaderView()]
    calls = {
        "apus_consumer_attach": (None, C.byref(views[0])),
        "apus_submitter_attach": (None, C.byref(views[1])),
        "apus_reader_attach": (None, C.byref(views[2])),
        "apus_consumer_detach": (),
        "apus_submitter_detach": (),
        "apus_reader_detach": (),
        "apus_consume_device": (1, a, a, a, a, a, a, 8, a, None),
        "apus_consume_device_packed": (1, a, a, a, a, a, a, 8, a, None),
        "apus_consume_status": (w[0], w[1], w[2], w[3]),
        "apus_consume_wait": (1, 1000, a, None),
        "apus_consume_wait_release": (),
        "apus_consume_wait_status": (w[0], w[1]),
        "apus_consume_mark": (a, None),
        "apus_consume_seed": (0, 1),
        "apus_read_fence": (1000, a, a, None),
        "apus_read_fence_status": (w[0], w[1]),
    }
    for name, args in calls.items():
        assert name in built.EXPORTS, name
        assert getattr(lib, name)(None, *args) == built.APUS_ERROR, name
        assert lib.apus_last_error() == b"null argument", (name, lib.apus_last_error())
    for v in views:
        assert bytes(v) == bytes(C.sizeof(v)), type(v)


def test_nm_shows_kernel_and_c_abi(built):
    out = subprocess.run(["nm", "-D", "--defined-only", built.LIB_PATH], capture_output=True, text=True).stdout
    for s in declared_symbols():
        assert re.search(rf"\bT {s}\b", out), s


def test_sass_is_sm90a(built):
    out = subprocess.run(["cuobjdump", "-lelf", built.LIB_PATH], capture_output=True, text=True).stdout
    assert "sm_90a" in out


def test_no_cpu_fallback(built):
    """Without a visible GPU, creating a replica is an error, not a silent CPU path."""
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    with pytest.raises(built.ApusError):
        built.Replica(0, 0, 1)


def test_config_struct_matches_header(built):
    # struct_size is checked by the library itself; this pins the Python mirror
    assert C.sizeof(built.Config) == 56          # ABI 2: + hb_period_us, hb_timeout_us (48 B ABI-1 configs are accepted)
    assert C.sizeof(built.PeerHandle) == 128
    assert C.sizeof(built.LogOffsets) == 64
    assert C.sizeof(built.Stats) == 208


def test_engine_entry_resolves_reference_proxy(built):
    """libapus_dare.so exports the engine-entry symbols and satisfies every undefined symbol of the
    reference's unmodified proxy.c (oracle/_ref/libref_proxy.so), without a GPU."""
    dare = os.path.join(ROOT, "apus_b200", "libapus_dare.so")
    out = subprocess.run(["nm", "-D", "--defined-only", dare], capture_output=True, text=True).stdout
    for s in ("dare_server_init", "dare_server_shutdown", "is_leader", "get_node_id", "tailhead", "tailq_lock",
              "prev_log_entry_head"):
        assert re.search(rf"\b[TBDC] {s}\b", out), s
    refproxy = os.path.join(ROOT, "oracle", "_ref", "libref_proxy.so")
    if not os.path.exists(refproxy):
        pytest.skip("oracle/_ref/libref_proxy.so absent")
    code = ("import ctypes as C;"
            f"C.CDLL({built.LIB_PATH!r}, mode=C.RTLD_GLOBAL);"
            f"d=C.CDLL({dare!r}, mode=C.RTLD_GLOBAL);"
            f"p=C.CDLL({refproxy!r}, mode=C.RTLD_GLOBAL | 2);"   # RTLD_NOW: resolve everything
            "assert d.is_leader()==0; print('ok')")
    r = subprocess.run([os.sys.executable, "-c", code], capture_output=True, text=True)
    assert r.returncode == 0 and "ok" in r.stdout, r.stderr


def test_reference_interposer_links_on_engine_and_refuses_without_gpu(built, tmp_path):
    """oracle/_ref/interpose.so = the reference's unmodified spec_hooks.cpp + proxy.c + db-interface.c +
    config-proxy.c (vendored libconfig, BerkeleyDB) linked on libapus_dare.so/libapus_gpu.so
    (oracle/build_refapp.sh, INTEGRATION.md section 2): every symbol resolves, and an unmodified redis-server
    started the way benchmarks/run.sh:26 starts it reaches dare_server_init, which -- on a box without a GPU --
    refuses loudly instead of falling back to a CPU path (the app then simply runs unreplicated)."""
    ref = os.path.join(ROOT, "oracle", "_ref")
    inter, server = os.path.join(ref, "interpose.so"), os.path.join(ref, "redis-server")
    if not (os.path.exists(inter) and os.path.exists(server)):
        pytest.skip("oracle/_ref application binaries absent (oracle/build_refapp.sh needs /root/reference)")
    out = subprocess.run(["ldd", "-r", inter], capture_output=True, text=True)
    assert "undefined symbol" not in out.stdout + out.stderr, out.stdout + out.stderr
    assert "libapus_dare.so" in out.stdout and "libapus_gpu.so" in out.stdout
    assert "libibverbs" not in out.stdout and "libev." not in out.stdout
    if built.lib().apus_device_count() > 0:
        return                                        # with a GPU the full run is tests/test_gpu_redis_dropin.py
    cfg = tmp_path / "node.cfg"
    cfg.write_text('db_name = "node_test";\nreq_log = 0;\nip_address = "127.0.0.1";\nport = 18870;\n')
    env = dict(os.environ, server_type="start", server_idx="0", group_size="1", config_path=str(cfg),
               dare_log_file=str(tmp_path / "dare.log"), LD_PRELOAD=inter)
    p = subprocess.Popen([server, "--port", "18870", "--save", "", "--bind", "127.0.0.1"], cwd=tmp_path, env=env,
                         stdout=subprocess.PIPE, stderr=subprocess.STDOUT)
    try:
        import time
        log = ""
        for _ in range(100):
            time.sleep(0.1)
            if (tmp_path / "dare.log").exists():
                log = (tmp_path / "dare.log").read_text()
                if "no CPU fallback" in log:
                    break
        assert "no CUDA device: the engine has no CPU fallback" in log, log
        assert p.poll() is None                       # the application itself keeps running
    finally:
        p.kill()
        p.wait(timeout=10)


def test_memcached_under_engine_interposer_refuses_without_gpu(built, tmp_path):
    """The second application of the reference (BASELINE config 4): an unmodified four-thread memcached 1.4.21 started
    under the same interposer (linked on libapus_dare.so / libapus_gpu.so).  Without a GPU the engine refuses loudly and
    memcached keeps serving, unreplicated -- the hooks (accept / read / close from several worker threads) stay out of
    the way.  With a GPU the full run is tests/test_zz_gpu_memcached_dropin.py."""
    import socket
    import time
    ref = os.path.join(ROOT, "oracle", "_ref")
    inter, server = os.path.join(ref, "interpose.so"), os.path.join(ref, "memcached")
    if not (os.path.exists(inter) and os.path.exists(server)):
        pytest.skip("oracle/_ref/memcached or interpose.so absent (oracle/build_memcached.sh, build_refapp.sh need /root/reference)")
    if built.lib().apus_device_count() > 0:
        pytest.skip("a GPU is visible: this is the no-GPU half")
    cfg = tmp_path / "node.cfg"
    cfg.write_text('db_name = "node_test";\nreq_log = 0;\nip_address = "127.0.0.1";\nport = 21470;\n')
    env = dict(os.environ, server_type="start", server_idx="0", group_size="3", config_path=str(cfg),
               dare_log_file=str(tmp_path / "dare.log"), apus_rendezvous=str(tmp_path / "rdv"), LD_PRELOAD=inter)
    p = subprocess.Popen([server, "-u", "root", "-p", "21470", "-U", "0", "-t", "4", "-l", "127.0.0.1"], cwd=tmp_path, env=env,
                         stdout=subprocess.PIPE, stderr=subprocess.STDOUT)
    try:
        log = ""
        for _ in range(100):
            time.sleep(0.1)
            if (tmp_path / "dare.log").exists():
                log = (tmp_path / "dare.log").read_text()
                if "no CPU fallback" in log:
                    break
        assert "no CUDA device: the engine has no CPU fallback" in log, log
        assert p.poll() is None
        replies = []
        for c in range(4):                            # several connections: the worker threads' read() hooks
            s = socket.create_connection(("127.0.0.1", 21470))
            s.settimeout(5)
            s.sendall(b"set k%d 0 0 5\r\nhello\r\nget k%d\r\n" % (c, c))
            buf = b""
            while buf.count(b"\r\n") < 4:
                buf += s.recv(4096)
            replies.append(buf)
            s.close()
        assert all(r == b"STORED\r\nVALUE k%d 0 5\r\nhello\r\nEND\r\n" % c for c, r in enumerate(replies)), replies
    finally:
        p.kill()
        p.wait(timeout=10)

"""The decisions of a read fence -- apus_b200/csrc/apus_fence.h, the functions the fence kernel itself uses, compiled as
C: tests/hostlogic/read_fence_props.c checks, exhaustively for groups of 1 to 13 over connected masks and SID terms
around t, that a fence confirms its leader iff a majority of connected members is still at term <= t, that a member
that is not connected never counts, and that READY never holds short of the leader's commit or on an entry of an older
term.  No GPU."""
import os
import subprocess

HERE = os.path.dirname(os.path.abspath(__file__))


def test_read_fence_decisions(tmp_path):
    exe = str(tmp_path / "read_fence_props")
    subprocess.run(["gcc", "-O2", "-std=gnu99", "-Wall", "-o", exe, os.path.join(HERE, "hostlogic", "read_fence_props.c")],
                   check=True)
    out = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0 and out.stdout.startswith("fence ok"), out.stdout + out.stderr

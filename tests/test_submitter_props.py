"""The reservation arithmetic of resident submitters -- include/apus_slot_format.h, the functions the device API itself
calls, compiled as C: tests/hostlogic/submitter_props.c interleaves host submits, device batches and submitter
sessions (reserve, publish, detach with dropped reservations) of random sizes over many laps of both rings, and checks
that space is never over-committed and that external images stay contiguous except where APUS_SLOT_WRAP marks them.
No GPU."""
import os
import subprocess

HERE = os.path.dirname(os.path.abspath(__file__))


def test_submitter_reservations(tmp_path):
    exe = str(tmp_path / "submitter_props")
    subprocess.run(["gcc", "-O2", "-std=gnu99", "-Wall", "-Werror", "-o", exe,
                    os.path.join(HERE, "hostlogic", "submitter_props.c")], check=True)
    out = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0 and out.stdout.startswith("submitter ok"), out.stdout + out.stderr

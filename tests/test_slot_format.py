"""The submission-slot format (apus_b200/csrc/apus_slot.h, DESIGN.md section 2) -- the functions the host submit paths
and the fill kernels use, compiled as C: tests/hostlogic/slot_props.c runs random mixes of host requests (0..1500 B,
inline and external) and device batches with worst-case reservations through a small payload ring that wraps many
times, and checks that every image lies inside the ring and its reservation, that consecutive external images are
contiguous unless the later one carries WRAP (the leader's staging rule), that live images never overlap, and that a
host-written slot decodes field by field to apus_slot_t.  No GPU."""
import os
import subprocess

HERE = os.path.dirname(os.path.abspath(__file__))


def test_slot_format_properties(tmp_path):
    exe = str(tmp_path / "slot_props")
    subprocess.run(["gcc", "-O2", "-std=gnu99", "-Wall", "-Werror", "-o", exe, os.path.join(HERE, "hostlogic", "slot_props.c")],
                   check=True)
    out = subprocess.run([exe], capture_output=True, text=True, timeout=120)
    assert out.returncode == 0 and out.stdout.startswith("slot ok"), out.stdout + out.stderr

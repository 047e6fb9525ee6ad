"""The payload-ring reservation of packed device batches (apus_b200/csrc/apus_slot.h: slot_packed_reserve, the bound
apus_submit_device_packed reserves from n and values_bytes alone), compiled as C: tests/hostlogic/packed_reserve_props.c
checks, for random valid offset arrays with lengths 0, 78, 79, 80 and 65535 drawn often, that the batch's external images
fit the bound and that the bound never exceeds n * round16(2 + 65535).  No GPU."""
import os
import subprocess

HERE = os.path.dirname(os.path.abspath(__file__))


def test_packed_reservation_bound(tmp_path):
    exe = str(tmp_path / "packed_reserve_props")
    subprocess.run(["gcc", "-O2", "-std=gnu99", "-Wall", "-Werror", "-o", exe,
                    os.path.join(HERE, "hostlogic", "packed_reserve_props.c")], check=True)
    out = subprocess.run([exe], capture_output=True, text=True, timeout=120)
    assert out.returncode == 0 and out.stdout.startswith("packed ok"), out.stdout + out.stderr

"""The box-box clipper keeps its per-pair state in registers (no GPU needed: reads the SASS of the built library)."""
import os, re, shutil, subprocess
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_np_clip_uses_no_local_memory_and_shares_the_pair_across_lanes():
    """k_np_clip clips one pair with four lanes that exchange axis penetrations and point masks by shuffles, and indexes no array at run
    time, so the kernel has no local-memory loads or stores (a run-time index into a register array moves the array to local memory)."""
    exe = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    lib = os.path.join(ROOT, "nudge_b200", "lib", "libnudge_b200.so")
    if not os.path.exists(exe) or not os.path.exists(lib):
        pytest.skip("cuobjdump or the built library is missing")
    sass = subprocess.run([exe, "-sass", lib], capture_output=True, text=True, timeout=600).stdout
    ops, cur = [], None
    for line in sass.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            cur = m.group(1)
        elif cur and cur.startswith("_Z9k_np_clip"):
            ops.append(line)
    assert ops, "k_np_clip not found in the library"
    ops = "\n".join(ops)
    assert not re.search(r"\b(LDL|STL)\b", ops), "k_np_clip touches local memory"
    assert "SHFL.BFLY" in ops and "SHFL.IDX" in ops

"""The type A kernels keep their field elements in registers and shared-memory slots: no instruction of
theirs, or of the out-of-line field operations they call (Ops::sqr, Ops::sqrsub, ...), goes through
local memory.  A 16-limb routine whose indices are not compile-time constants puts its arrays in a
local-memory frame and puts L1 latency on the multiplier's critical path; this reads the SASS of the
built library (cuobjdump -sass) and fails if LDL or STL appears in one of these kernels."""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.environ.get("PBC_B200_LIB") or os.path.join(ROOT, "pbc_b200", "libpbc_b200.so")

# mangled-name prefixes: the Miller loops, the final exponentiation, the 16-limb batch inversion, the
# product of pairings, the fixed-argument pairing and the slot-multiplier probes
KERNELS = ("_ZN7pbcb20011k_a_miller9I", "_ZN7pbcb20018k_a_miller9_sharedI", "_ZN7pbcb20012k_a_finalexpI",
           "_ZN7pbcb20014k_batch_invertILi16E", "_ZN7pbcb2008k_a_prodI", "_ZN7pbcb20012k_a_pp_applyI",
           "_ZN7pbcb20013k_fpmul_slotsILi16E", "_ZN7pbcb20013k_fpmul_chainILi16E")


def _cuobjdump():
    exe = shutil.which("cuobjdump")
    if not exe:
        exe = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "cuobjdump")
    return exe if os.path.exists(exe) else None


def test_type_a_kernels_use_no_local_memory():
    exe = _cuobjdump()
    if not exe:
        pytest.skip("no cuobjdump")
    if not os.path.exists(LIB):
        pytest.skip("library not built")
    sass = subprocess.run([exe, "-sass", LIB], capture_output=True, text=True, check=True).stdout
    counts, fn = {}, None
    for line in sass.splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            fn = m.group(1) if m.group(1).startswith(KERNELS) else None
            if fn:
                counts[fn] = 0
        elif fn and re.search(r"\b(LDL|STL)(\.\S+)?\s", line):
            counts[fn] += 1
    found = {k for k in KERNELS if any(f.startswith(k) for f in counts)}
    assert found == set(KERNELS), "kernels missing from the SASS: %s" % sorted(set(KERNELS) - found)
    bad = {f: n for f, n in counts.items() if n}
    assert not bad, "local-memory loads/stores: %s" % bad

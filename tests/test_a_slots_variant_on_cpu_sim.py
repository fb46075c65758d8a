"""The type A Miller kernel the default build does not run: PBC_A_SLOTS = 7 (k_a_miller7, seven slots,
four blocks per SM, kept for A/B runs against the default nine-slot k_a_miller9).  The `-m gpu` type A
tests, unchanged, on the CPU simulator of that build, so both settings of the switch stay pinned."""
import os
import shutil
import subprocess
import sys

import pytest

from tests.test_kernels_on_cpu_sim import ROOT, _build, _env


def test_seven_slot_miller_kernel_gives_the_same_bytes(tmp_path):
    if not shutil.which("g++"):
        pytest.skip("no g++")
    so = _build(tmp_path, "-DPBC_A_SLOTS=7")
    cmd = [sys.executable, "-m", "pytest", "-q", "-m", "gpu", "-p", "no:cacheprovider",
           "-k", "not large_batch and not device_pointer and not tiles and not across_blocks",
           os.path.join(ROOT, "tests", "test_gpu_type_a.py")]
    try:
        import xdist  # noqa: F401
        cmd += ["-n", str(max(1, min(8, len(os.sched_getaffinity(0)))))]
    except Exception:
        pass
    out = subprocess.run(cmd, env=_env(so), capture_output=True, text=True, timeout=1500, cwd=ROOT)
    tail = out.stdout.strip().splitlines()[-1] if out.stdout.strip() else out.stderr[-500:]
    assert out.returncode == 0, out.stdout[-3000:]
    assert int(tail.split(" passed")[0].split()[-1]) >= 20, tail

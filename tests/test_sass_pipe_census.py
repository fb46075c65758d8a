"""What ptxas made of the 512-bit squaring, read from the built library without a GPU.  The source cannot show
how many additions and moves ptxas places on the multiplier pipe as IMAD.X / IMAD.MOV / IMAD; the SASS can
(tools/sass_pipe_census.py).  The timed loop of the register-resident probe k_fpmul_chain<16, true, 2> holds one
squaring: 392 products and 16 reduction factors are its floor of 408 multiplier-pipe instructions.  The
product-scanning squarer this field used before stood at 453 (375 IMAD.WIDE + 78 other IMAD) with 316 IADD3;
the row-wise squarer stands at 412 with 161.  The bound is a ratchet: lower it when the count falls."""
import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from tools import sass_pipe_census as census  # noqa: E402

LIB = os.environ.get("PBC_B200_LIB") or os.path.join(ROOT, "pbc_b200", "libpbc_b200.so")


@pytest.fixture(scope="module")
def kernels():
    if not census.cuobjdump():
        pytest.skip("no cuobjdump")
    if not os.path.exists(LIB):
        pytest.skip("library not built")
    ks = census.kernels(LIB)
    if not ks:
        pytest.skip("no SASS in the library (the CPU simulator)")
    return ks


def _loop(kernels, prefix):
    hit = [k for k in kernels if k.startswith(prefix)]
    assert len(hit) == 1, (prefix, hit)
    c = census.loop_census(kernels[hit[0]])
    assert c is not None, "no loop in %s" % hit[0]
    return c


def test_squaring_probe_stays_within_its_multiplier_pipe_budget(kernels):
    sqr = _loop(kernels, census.SQR_PROBE)
    # the loop holds exactly one squaring: not unrolled (below two), not hoisted out (above three quarters of one)
    assert 300 <= sqr["imad_wide"] <= 392, sqr
    assert sqr["mul_pipe"] <= 440, sqr
    assert sqr["ldl_stl"] == 0, sqr


def test_multiplication_probe_is_one_multiplication(kernels):
    mul = _loop(kernels, census.MUL_PROBE)
    assert 480 <= mul["imad_wide"] <= 512 and mul["mul_pipe"] <= 540 and mul["ldl_stl"] == 0, mul

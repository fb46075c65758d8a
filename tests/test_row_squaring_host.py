"""The row-wise squarer the type A kernels use (fp.cuh: sqr_wide, mont_sqr_os, and redc_wide with one
conditional subtraction), run on the CPU through the PTX interpreter (tests/host/make_host_fp.py) and
compared with Python integers: the exact double-width square on the operands that drive every carry path,
the Montgomery square for moduli across the range the type A parameters allow, and the single-pass
reduction up to its largest input."""
import os
import random
import shutil
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HOST = os.path.join(ROOT, "tests", "host")


@pytest.fixture(scope="module")
def harness(tmp_path_factory):
    if not shutil.which("g++"):
        pytest.skip("no g++")
    d = tmp_path_factory.mktemp("sqr_rows")
    hdr, exe = str(d / "host_fp.hpp"), str(d / "sqr_rows_host")
    subprocess.check_call([sys.executable, os.path.join(HOST, "make_host_fp.py"), hdr])
    subprocess.check_call(["g++", "-O1", "-std=c++17", "-Wno-unknown-pragmas", '-DHOST_FP_HEADER="%s"' % hdr,
                           "-o", exe, os.path.join(HOST, "sqr_rows_host.cpp")])
    return exe


def _a_param_q():
    sys.path.insert(0, ROOT)
    from pbc_b200.params import PARAMS
    for line in PARAMS["a"].splitlines():
        if line.startswith("q "):
            return int(line.split()[1])
    raise AssertionError("a.param has no q")


def _moduli(N):
    rnd = random.Random(5 + N)
    R = 1 << (32 * N)
    top = 32 * N
    out = [
        (1 << (top - 8)) | rnd.getrandbits(top - 8) | 1,       # 505 bits for N = 16, the smallest type A field
        (1 << (top - 1)) + rnd.randrange(1 << 20) * 2 + 1,     # just above 2^511: all-zero limbs
        (1 << (top - 1)) | rnd.getrandbits(top - 1) | 1,
        R - rnd.randrange(1, 1 << 20) * 2 - 1,                 # just below 2^512: all-ones limbs
    ]
    if N == 16:
        out.insert(0, _a_param_q())
    return out


def _limb_patterns(N):
    """all-ones limbs, alternating limbs, one set bit in each limb (lowest, highest, a middle one), each limb alone"""
    ones = (1 << (32 * N)) - 1
    pats = [0, 1, ones, ones - 1, 1 << (32 * N - 1), (1 << (32 * N - 1)) - 1,
            int("ffffffff00000000" * (N // 2), 16), int("00000000ffffffff" * (N // 2), 16),
            sum(1 << (32 * k) for k in range(N)), sum(1 << (32 * k + 31) for k in range(N)),
            sum(1 << (32 * k + (7 * k + 3) % 32) for k in range(N))]
    pats += [0xffffffff << (32 * k) for k in range(N)]
    pats += [ones ^ (0xffffffff << (32 * k)) for k in range(N)]
    return pats


def _run(exe, requests):
    text = "".join("%s %d %x %x\n" % r for r in requests)
    out = subprocess.run([exe], input=text, capture_output=True, text=True, timeout=900, check=True)
    return [int(x, 16) for x in out.stdout.split()]


@pytest.mark.parametrize("N", [16, 8])
def test_wide_square_is_exact(harness, N):
    rnd = random.Random(31 + N)
    vals = _limb_patterns(N) + [rnd.getrandbits(32 * N) for _ in range(300 if N == 16 else 100)]
    got = _run(harness, [("wsqr", N, 3, a) for a in vals])
    bad = [hex(a) for a, g in zip(vals, got) if g != a * a]
    assert len(got) == len(vals) and not bad, bad[:3]


@pytest.mark.parametrize("N", [16, 8])
def test_montgomery_square(harness, N):
    rnd = random.Random(37 + N)
    R = 1 << (32 * N)
    reqs, want = [], []
    for q in _moduli(N):
        Rinv = pow(R, -1, q)
        vals = [0, 1, 2, q - 1, q - 2, (q - 1) // 2, (q + 1) // 2, R % q] + [v % q for v in _limb_patterns(N)]
        vals += [rnd.randrange(q) for _ in range(60)]
        for a in vals:
            for op in (("sqr", "fpsqr") if N == 16 else ("sqr",)):
                reqs.append((op, N, q, a))
                want.append(a * a * Rinv % q)
    got = _run(harness, reqs)
    bad = [(r[0], hex(r[2]), hex(r[3])) for r, g, w in zip(reqs, got, want) if g != w]
    assert len(got) == len(want) and not bad, bad[:3]


def test_single_pass_reduction_of_values_below_qR(harness):
    rnd = random.Random(41)
    N, R = 16, 1 << 512
    reqs, want = [], []
    for q in _moduli(N):
        Rinv = pow(R, -1, q)
        ts = [0, 1, q, R - 1, R, (q - 1) * (q - 1), q * q - 1, (q - 1) * R, (q - 1) * R + R - 1, q * (R - 1)]
        ts += [rnd.randrange(q * q) for _ in range(40)] + [rnd.randrange(q * R) for _ in range(20)]
        for t in ts:
            if t < q * R:
                reqs.append(("redc1", N, q, t))
                want.append(t * Rinv % q)
    got = _run(harness, reqs)
    bad = [(hex(r[2]), hex(r[3])) for r, g, w in zip(reqs, got, want) if g != w]
    assert len(got) == len(want) and len(want) > 300 and not bad, bad[:3]

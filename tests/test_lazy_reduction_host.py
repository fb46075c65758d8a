"""The double-width primitives of fp.cuh that the type A Miller step reduces lazily with (mul_wide,
wide_add / wide_sub, wide_add_pR, wide_sub_pR_if_ge, redc_wide), run on the CPU through the PTX
interpreter (tests/host/make_host_fp.py) and compared with Python integers.  Every combination the step
uses (Ops::lazy in slots.cuh) must give the fully reduced residue (sum of products) R^-1 mod q, for
operands 0, 1, q - 1 and random ones, and for moduli across the range the type A parameters allow:
505 bits, just above 2^511, just below 2^512 and a.param's q."""
import os
import random
import shutil
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HOST = os.path.join(ROOT, "tests", "host")
N = 16
R = 1 << (32 * N)


@pytest.fixture(scope="module")
def harness(tmp_path_factory):
    if not shutil.which("g++"):
        pytest.skip("no g++")
    d = tmp_path_factory.mktemp("lazy")
    hdr, exe = str(d / "host_fp.hpp"), str(d / "lazy_host")
    subprocess.check_call([sys.executable, os.path.join(HOST, "make_host_fp.py"), hdr])
    subprocess.check_call(["g++", "-O1", "-std=c++17", "-Wno-unknown-pragmas", '-DHOST_FP_HEADER="%s"' % hdr,
                           "-o", exe, os.path.join(HOST, "lazy_redc_host.cpp")])
    return exe


def _a_param_q():
    sys.path.insert(0, ROOT)
    from pbc_b200.params import PARAMS
    for line in PARAMS["a"].splitlines():
        if line.startswith("q "):
            return int(line.split()[1])
    raise AssertionError("a.param has no q")


def _moduli():
    rnd = random.Random(5)
    return [
        _a_param_q(),
        (1 << 504) | rnd.getrandbits(504) | 1,                 # 505 bits, the smallest type A field
        (1 << 511) + rnd.randrange(1 << 20) * 2 + 1,           # just above 2^511: all-zero limbs
        (1 << 511) | rnd.getrandbits(511) | 1,
        R - rnd.randrange(1, 1 << 20) * 2 - 1,                 # just below 2^512: all-ones limbs
    ]


def _operands(q, rnd, count):
    edge = [0, 1, 2, q - 1, q - 2, (q - 1) // 2, R % q, ((1 << 480) - 1) % q]
    quads = [(a, b, c, d) for a in edge for b in (0, 1, q - 1) for c in (0, q - 1) for d in (1, q - 1)]
    quads += [tuple(rnd.randrange(q) for _ in range(4)) for _ in range(count)]
    return quads


def _run(exe, requests):
    text = "".join("%s %x %x %x %x %x %x\n" % r for r in requests)
    out = subprocess.run([exe], input=text, capture_output=True, text=True, timeout=900, check=True)
    return out.stdout.splitlines()


def test_wide_product_is_exact(harness):
    rnd = random.Random(3)
    ones = R - 1
    edge = [0, 1, ones, ones - 1, 1 << 511, (1 << 511) - 1, int("ffffffff00000000" * 8, 16), int("00000000ffffffff" * 8, 16),
            0xffffffff, 0xffffffff << 480, 1 << 32]
    pairs = [(a, b) for a in edge for b in edge] + [(rnd.getrandbits(512), rnd.getrandbits(512)) for _ in range(100)]
    q = _a_param_q()
    got = _run(harness, [("wmul", q, a, b, 0, 0, 0) for a, b in pairs])
    bad = [(hex(a), hex(b)) for (a, b), g in zip(pairs, got) if int(g, 16) != a * b]
    assert len(got) == len(pairs) and not bad, bad[:3]


def test_reduction_of_values_below_2qR(harness):
    rnd = random.Random(4)
    reqs, want = [], []
    for q in _moduli():
        Rinv = pow(R, -1, q)
        ts = [0, 1, q, q * R, q * R - 1, 2 * q * R - 1, 2 * q * R - R, R - 1, (q - 1) * (q - 1), 2 * (q - 1) * (q - 1),
              q * R + (q - 1) ** 2]
        ts += [rnd.randrange(2 * q * R) for _ in range(40)]
        for t in ts:
            assert 0 <= t < 2 * q * R
            reqs.append(("redc", q, t, 0, 0, 0, 0))
            want.append(t * Rinv % q)
    got = [int(g, 16) for g in _run(harness, reqs)]
    bad = [(hex(r[1]), hex(r[2])) for r, g, w in zip(reqs, got, want) if g != w]
    assert len(got) == len(want) and not bad, bad[:3]


def test_step_combinations(harness):
    """Re l = (U Z Qx + X T) / R; f0' = (P1 - P2 + q R) / R with S' = P1 + P2 (- q R); f1' = (P3 - S' + q R) / R"""
    rnd = random.Random(6)
    reqs, want = [], []
    for q in _moduli():
        Rinv = pow(R, -1, q)
        for a, b, c, d in _operands(q, rnd, 30):
            reqs.append(("sum", q, a, b, c, d, 0))
            want.append(str((a * b + c * d) * Rinv % q))
            s = a * b + c * d
            if s >= q * R:
                s -= q * R
            reqs.append(("kara0", q, a, b, c, d, 0))
            want.append("%d %d" % ((a * b - c * d) * Rinv % q, s))
            reqs.append(("kara1", q, (a + c) % q, (b + d) % q, 0, 0, s))
            want.append(str(((a + c) * (b + d) - a * b - c * d) * Rinv % q))
    got = _run(harness, reqs)
    got = [" ".join(str(int(x, 16)) for x in g.split()) for g in got]
    bad = [(r[0], hex(r[1]), hex(r[2]), hex(r[3])) for r, g, w in zip(reqs, got, want) if g != w]
    assert len(got) == len(want) and not bad, bad[:3]


def test_stored_sum_is_below_qR_whenever_it_can_reach_it(harness):
    """S = P1 + P2 >= q R happens for a.param's q (2 q^2 > q R): the stored S' must come back below q R"""
    q = _a_param_q()
    assert 2 * (q - 1) ** 2 >= q * R
    got = _run(harness, [("kara0", q, q - 1, q - 1, q - 1, q - 1, 0)])
    s = int(got[0].split()[1], 16)
    assert s == 2 * (q - 1) ** 2 - q * R and s < q * R

"""The limb-level field arithmetic the kernels compile (pbc_b200/csrc/fp.cuh, fq_small.cuh: inline-PTX
carry chains, operand- and product-scanning Montgomery multipliers, lazy double-width reduction) run
on the CPU: tests/host/make_host_fp.py routes every asm statement through a PTX interpreter
(tests/host/ptx_emul.hpp) and the same templates -- N = 5, 6, 16, 34 limbs, FULL or not -- are compared
with Python integers on random operands and on the carry-heavy edge values.  The GPU tests check the
same functions on the hardware; this pins the source-level logic without one."""
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
    d = tmp_path_factory.mktemp("limb")
    hdr, exe = str(d / "host_fp.hpp"), str(d / "limb_host")
    subprocess.check_call([sys.executable, os.path.join(HOST, "make_host_fp.py"), hdr])
    subprocess.check_call(["g++", "-O1", "-std=c++17", "-Wno-unknown-pragmas", '-DHOST_FP_HEADER="%s"' % hdr,
                           "-o", exe, os.path.join(HOST, "limb_arith_host.cpp")])
    return exe


def _moduli(N, full, rnd):
    """odd moduli of the shapes the kernels meet: FULL = top bit of the top limb set"""
    top = 32 * N
    if full:
        bits = [top]
    else:
        bits = [top - 1, top - 11, top - 40] if N > 6 else [top - 1, top - 2, top - 11]   # 149-, 158-, 159-bit q in 5 limbs
    out = []
    for b in bits:
        out.append((1 << (b - 1)) | rnd.getrandbits(b - 1) | 1)          # random
        out.append((1 << b) - rnd.randrange(1, 1 << 20) * 2 - 1)         # 2^b - small: all-ones limbs
        out.append((1 << (b - 1)) + rnd.randrange(1 << 20) * 2 + 1)      # 2^(b-1) + small: all-zero limbs
    return out


def _operands(p, N, rnd, count):
    edge = [0, 1, 2, p - 1, p - 2, (p - 1) // 2, (p + 1) // 2, (1 << (p.bit_length() - 1)) % p,
            ((1 << (32 * (N - 1))) - 1) % p, int("ffffffff00000000" * N, 16) % p, int("00000000ffffffff" * N, 16) % p]
    vals = [(a, b) for a in edge for b in (edge[0], edge[3], edge[5], edge[8], edge[10])]
    vals += [(rnd.randrange(p), rnd.randrange(p)) for _ in range(count)]
    return vals


def _run(exe, requests):
    text = "".join("%d %d %s %x %x %x %x %x\n" % r for r in requests)
    out = subprocess.run([exe], input=text, capture_output=True, text=True, timeout=900, check=True)
    return [int(x, 16) for x in out.stdout.split()]


CONFIGS = [(5, 0), (6, 0), (16, 1), (16, 0), (34, 0), (34, 1)]


@pytest.mark.parametrize("N,full", CONFIGS)
def test_montgomery_multipliers_and_additive_ops(harness, N, full):
    rnd = random.Random(1000 * N + full)
    R = 1 << (32 * N)
    reqs, want = [], []
    for p in _moduli(N, full, rnd):
        Rinv = pow(R, -1, p)
        for a, b in _operands(p, N, rnd, 12 if N > 16 else 30):
            ops = [("mul_ps", a * b * Rinv % p), ("sqr_ps", a * a * Rinv % p), ("add", (a + b) % p),
                   ("sub", (a - b) % p), ("neg", -a % p), ("halve", a * pow(2, -1, p) % p)]
            if N % 2 == 0:
                ops.append(("mul_os", a * b * Rinv % p))
            for op, w in ops:
                reqs.append((N, full, op, p, a, b, 0, 0))
                want.append(w)
    got = _run(harness, reqs)
    bad = [(r[2], hex(r[3])) for r, g, w in zip(reqs, got, want) if g != w]
    assert len(got) == len(want) and not bad, bad[:5]


def test_unreduced_scanned_operand_comes_out_reduced(harness):
    """the wire-to-Montgomery conversion multiplies R^2 (full operand) by the raw wire value (scanned
    operand), which may exceed p: the result must still be canonical (pairing_a1.cuh a1_load_point)"""
    rnd = random.Random(7)
    N = 34
    R = 1 << (32 * N)
    p = (1 << 1032) | rnd.getrandbits(1032) | 1
    r2 = R * R % p
    reqs, want = [], []
    for _ in range(20):
        x = rnd.getrandbits(1040)                       # 130 wire bytes, not reduced
        reqs.append((N, 0, "mul_os", p, r2, x, 0, 0))
        want.append(x * R % p)
    assert _run(harness, reqs) == want


def test_lazy_double_width_reduction(harness):
    """fq_mulw_call / fq_redc_call / fq_redc2_call (types F, D, G): a b and a b + c d reduced once"""
    rnd = random.Random(11)
    N, R = 5, 1 << 160
    reqs, want = [], []
    for p in _moduli(5, 0, rnd):
        Rinv = pow(R, -1, p)
        for a, b in _operands(p, 5, rnd, 40):
            c, d = rnd.randrange(p), rnd.randrange(p)
            reqs += [(N, 0, "fq_mul", p, a, b, 0, 0), (N, 0, "fq_mulcall", p, a, b, 0, 0), (N, 0, "fq_sqrcall", p, a, 0, 0, 0),
                     (N, 0, "fq_mul_os", p, a, b, 0, 0)]
            want += [a * b * Rinv % p, a * b * Rinv % p, a * a * Rinv % p, a * b * Rinv % p]
            if a * b + c * d < 2 * p * R:                # fq_redc2_call's contract
                reqs += [(N, 0, "fq_mac", p, a, b, c, d), (N, 0, "fq_mac_os", p, a, b, c, d)]
                want += [(a * b + c * d) * Rinv % p] * 2
        # the operand-scanning product on unreduced operands (sums of two residues, below 2^160) and on
        # all-ones limbs: every carry path of the even / odd accumulators
        ones = (1 << 160) - 1
        for a, b in [(ones, ones), (ones, 1), (ones - (1 << 32), ones), ((1 << 159) + 1, ones), (2 * p - 2, 2 * p - 1)]:
            if a * b < 2 * p * R:
                reqs.append((N, 0, "fq_mul_os", p, a, b, 0, 0))
                want.append(a * b * Rinv % p)
    got = _run(harness, reqs)
    bad = [(r[2], hex(r[3])) for r, g, w in zip(reqs, got, want) if g != w]
    assert not bad, bad[:5]


def test_operand_scanning_wide_product_is_exact(harness):
    """fqw_mul (fq_small.cuh): the 320-bit product on the even / odd accumulators against Python's a * b,
    on the operands that drive every carry path: all-ones limbs, single set bits, alternating limbs"""
    rnd = random.Random(23)
    ones = (1 << 160) - 1
    edge = [0, 1, ones, ones - 1, 1 << 159, (1 << 159) - 1, int("ffffffff00000000" * 3, 16) & ones,
            int("00000000ffffffff" * 3, 16) & ones, 0xffffffff, 0xffffffff << 128, (1 << 32), (1 << 64) - 1]
    pairs = [(a, b) for a in edge for b in edge] + [(rnd.getrandbits(160), rnd.getrandbits(160)) for _ in range(300)]
    p = (1 << 158) | 0x1234567 | 1                      # unused by fqw_mul, the harness wants one
    got = _run(harness, [(5, 0, "fq_wmul", p, a, b, 0, 0) for a, b in pairs])
    bad = [(hex(a), hex(b)) for (a, b), g in zip(pairs, got) if g != a * b]
    assert not bad, bad[:5]


def test_accumulating_products_and_row_wise_reduction(harness):
    """FqAcc / fqw_redc_os (fq_small.cuh): sums of up to four 5 x 5 products kept unmerged on the even / odd
    accumulators with carry counts, against Python integers on the operands that drive every carry path; the row-wise
    Montgomery reduction for t < q R (one conditional subtraction) and t < 2 q R (two), including t_lo = 0, t = 0 and the
    largest inputs"""
    rnd = random.Random(47)
    N, R = 5, 1 << 160
    ones = R - 1
    edge = [0, 1, ones, ones - 1, 1 << 159, (1 << 159) - 1, int("ffffffff00000000" * 3, 16) & ones,
            int("00000000ffffffff" * 3, 16) & ones, 0xffffffff, 0xffffffff << 128, (1 << 64) - 1]
    p0 = (1 << 158) | 0x1234567 | 1
    reqs, want = [], []
    quads = [(a, b, c, d) for a in edge for b in edge[:6] for c in edge[2:5] for d in edge[1:4]]
    quads += [tuple(rnd.getrandbits(160) for _ in range(4)) for _ in range(200)]
    for a, b, c, d in quads:
        if a * b + c * d + a * d < 1 << 320:
            reqs.append((N, 0, "fq_acc3", p0, a, b, c, d)); want.append(a * b + c * d + a * d)
        if a * b + c * d + a * d + c * b < 1 << 320:
            reqs.append((N, 0, "fq_acc4", p0, a, b, c, d)); want.append(a * b + c * d + a * d + c * b)
    for p in _moduli(5, 0, rnd):
        Rinv = pow(R, -1, p)
        pairs = _operands(p, 5, rnd, 60) + [(2 * p - 1, p - 1), (R - 1, 1), (1 << 159, 2), (0, 5), (R >> 1, 2), (p - 1, p - 1),
                                            (ones, ones), (ones, p), (2 * p - 2, 2 * p - 1), (R >> 32, 1 << 32)]
        for a, b in pairs:
            if a * b < p * R:
                reqs.append((N, 0, "fq_mul_rows", p, a, b, 0, 0)); want.append(a * b * Rinv % p)
            if a * b < 2 * p * R and 3 * p <= R:
                reqs.append((N, 0, "fq_mul_rows2", p, a, b, 0, 0)); want.append(a * b * Rinv % p)
    got = _run(harness, reqs)
    bad = [(r[2], hex(r[3]), hex(r[4]), hex(r[5])) for r, g, w in zip(reqs, got, want) if g != w]
    assert len(got) == len(want) and len(want) > 800 and not bad, bad[:5]

"""The field, tower and lazy-reduction kernels on operands that are extreme INSIDE the Montgomery domain.

Every kernel computes on limbs w R mod q (R = 2^(32 N)), so the wire values 0, 1, q - 1, ... the other
parity tests use become pseudo-random limb patterns after conversion: the carry chains and the
lazy-reduction bounds (sums of double-width products kept below 2 q R, offsets such as 2 q^2 that keep a
difference positive) never see their largest or smallest inputs there.  Here a target set T of
INTERNAL values -- 0, 1, 2, q - 1, q - 2, (q +- 1)/2, q - 2^(32 k) and 2^(32 k) - 1 at every limb
boundary, the limb patterns of the host tests, the largest value below q's top limb -- is sent as the wire
value t R^-1 mod q, so that the kernel holds exactly t.  The towers get internally extreme coefficients
through the inverse of the basis maps the library uses (F_q^3: x = lam w - s; F_q^12: phi2 and tau^j).
R only steers which limbs the kernels see: every expectation is computed from the wire values with Python
integers or the oracle, so each check is a plain differential test against exact arithmetic.

N, the limb count of each family, is read from the sources (pairing_a.cuh, fq_small.cuh,
engine_d_wide.cu, pairing_a1.cuh), so a change of width cannot quietly turn the targets into random
values.  Coverage limit: the extremes reach the FIRST operation of each routine; values deep inside a
Miller loop or an exponentiation are reached only through the pairing tests."""
import json
import os
import random
import re

import pytest

from oracle import pbc_oracle as O
from pbc_b200.params import PARAMS
from tests.test_row_squaring_host import _limb_patterns

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "pbc_b200", "csrc")
D_WIDE = ("d175", "d190", "d196", "d201", "d224")


def _id(name):
    """test ids of the eight-limb type D sets carry d_wide (their own simulator runs them)"""
    return "d_wide_" + name if name in D_WIDE else name


def _src_int(fname, pattern):
    with open(os.path.join(CSRC, fname)) as f:
        m = re.search(pattern, f.read(), re.M)
    assert m, "%s: no match for %r" % (fname, pattern)
    return int(m.group(1))


LIMBS = {
    "a": _src_int("pairing_a.cuh", r"^constexpr int kNA = (\d+);"),
    "small": _src_int("fq_small.cuh", r"^#define PBC_NS (\d+)$"),
    "wide": _src_int("engine_d_wide.cu", r"^#define PBC_NS (\d+)$"),
    "a1": _src_int("pairing_a1.cuh", r"^constexpr int kNA1 = (\d+);"),
}
FAMILY_LIMBS = {"a": "a", "f": "small", "d159": "small", "g149": "small", "a1": "a1", "a1_small": "a1",
                "e": "a1", "e_s510": "a1", "e_s513": "a1"}
FAMILY_LIMBS.update({n: "wide" for n in D_WIDE})


def _param_text(name):
    if name in D_WIDE:
        fn = "d_wide_%s.json" % name
    elif name in ("a1_small", "e", "e_s510", "e_s513"):
        fn = name + ".json"
    else:
        return PARAMS[name]
    with open(os.path.join(ROOT, "tests", "golden", fn)) as f:
        return json.load(f)["param_text"]


def _q(text):
    """the field characteristic: q, or p for type a1"""
    tab = dict(ln.split()[:2] for ln in text.splitlines() if len(ln.split()) >= 2)
    return int(tab["q"] if "q" in tab else tab["p"])


def targets(q, N):
    """internal values below q, the named ones first"""
    named = [0, 1, 2, q - 1, q - 2, (q - 1) // 2, (q + 1) // 2]
    L = (q.bit_length() - 1) // 32                     # top non-zero limb of q
    named.append(((q >> (32 * L)) << (32 * L)) - 1)    # q's top limb less one, every lower limb 0xffffffff
    bound = []
    for k in range(1, N):
        bound += [q - (1 << (32 * k)), (1 << (32 * k)) - 1]
    pats = _limb_patterns(N)
    out, seen = [], set()
    for t in named + bound + pats:
        if 0 <= t < q and t not in seen:
            seen.add(t)
            out.append(t)
    return out


def _core(T, k=48):
    """the named targets and a fixed sample of the rest: the operands of the full cross product"""
    if len(T) <= k:
        return list(T)
    rest = T[8:]
    return T[:8] + random.Random(len(T)).sample(rest, k - 8)


class Dom:
    """internal value <-> wire value for one field (R = 2^(32 N))"""

    def __init__(self, q, N):
        self.q, self.N = q, N
        self.R = 1 << (32 * N)
        self.Ri = pow(self.R, -1, q)

    def wire(self, t):
        return t * self.Ri % self.q

    def internal(self, w):
        return w * self.R % self.q


_DEVS = {}


def _dev(name, extra=""):
    from pbc_b200.pairing import Pairing
    key = (name, extra)
    if key not in _DEVS:
        text = _param_text(name)
        _DEVS[key] = (Pairing(text + extra), text)
    return _DEVS[key]


def _enc(vals, wb):
    return b"".join(v.to_bytes(wb, "big") for v in vals)


def _dec(buf, wb):
    return [int.from_bytes(buf[i:i + wb], "big") for i in range(0, len(buf), wb)]


# ---- 2. F_q ops 0-7 on every family (ops 8, 9 on the eight-limb field) ---------------------------

FIELD_FAMILIES = ["a", "a1", "a1_small", "e", "e_s510", "e_s513", "f", "d159", "g149"] + list(D_WIDE)


def _binary_items(T, q, rnd):
    """the full cross product of the core targets, then every target against q - 1, 0 and random residues
    on either side: a few thousand items in one launch, so the lanes of a warp take different branches"""
    C = _core(T)
    xs = [a for a in C for b in C]
    ys = [b for a in C for b in C]
    for t in T:
        r1, r2 = rnd.randrange(q), rnd.randrange(q)
        xs += [t, q - 1, t, r1, t]
        ys += [q - 1, t, r2, t, 0]
    return xs, ys


FIELD = {0: lambda x, y, q: x * y % q, 1: lambda x, y, q: (x + y) % q, 2: lambda x, y, q: (x - y) % q,
         3: lambda x, y, q: pow(x, q - 2, q), 4: lambda x, y, q: x * pow(2, q - 2, q) % q,
         5: lambda x, y, q: -x % q, 6: lambda x, y, q: x * x % q, 7: lambda x, y, q: (x * y - y) % q,
         9: lambda x, y, q: x * y % q}


@pytest.mark.parametrize("name", FIELD_FAMILIES, ids=_id)
def test_field_ops_on_internal_extremes(name):
    pr, text = _dev(name)
    q = _q(text)
    N = LIMBS[FAMILY_LIMBS[name]]
    D = Dom(q, N)
    T = targets(q, N)
    wb = pr.g1_len // 2
    rnd = random.Random(sum(name.encode()))
    xs_t, ys_t = _binary_items(T, q, rnd)
    xs, ys = [D.wire(t) for t in xs_t], [D.wire(t) for t in ys_t]
    # the unary ops on every target; the inverse (a full exponentiation, slow on the 34-limb field's
    # simulator) on the named ones and a sample of the rest
    us = [D.wire(t) for t in T]
    inv = [D.wire(t) for t in (_core(T, 24) if N > 16 else T)]
    ops = [0, 1, 2, 3, 4, 5, 6, 7] + ([9] if name in D_WIDE else [])
    for op in ops:
        a, b = (xs, ys) if op in (0, 1, 2, 7, 9) else ((inv, inv) if op == 3 else (us, us))
        got = _dec(pr.fp_op(op, _enc(a, wb), _enc(b, wb), len(a)), wb)
        f = FIELD[op]
        bad = [(i, hex(D.internal(x)), hex(D.internal(y))) for i, (x, y, g) in enumerate(zip(a, b, got))
               if g != f(x, y, q)]
        assert not bad, "%s op %d: %d of %d wrong, first (item, internal a, internal b) %s" % (
            name, op, len(bad), len(a), bad[:4])


@pytest.mark.parametrize("name", ("d175", "d190", "d224"), ids=_id)
def test_wide_square_roots_on_internal_extremes(name):
    """op 8 (the Tonelli-Shanks square root element_from_hash takes where q = 1 mod 8: d175, d190, d224) on
    squares whose roots are internal extremes and on the extremes themselves (zero for a non-square)"""
    pr, text = _dev(name)
    q = _q(text)
    assert q % 8 == 1
    D = Dom(q, LIMBS["wide"])
    T = targets(q, D.N)
    wb = pr.g1_len // 2
    a = [D.wire(t) ** 2 % q for t in T] + [D.wire(t) for t in T]
    got = _dec(pr.fp_op(8, _enc(a, wb), _enc(a, wb), len(a)), wb)
    for x, y in zip(a, got):
        if pow(x, (q - 1) // 2, q) in (0, 1):
            assert y * y % q == x, (name, hex(D.internal(x)))
        else:
            assert y == 0, (name, hex(D.internal(x)))


# ---- 3. towers: coefficients extreme in the internal basis ---------------------------------------

def _d_basis(pr, q):
    """(forward, inverse) maps between the reference basis x and the internal basis w of F_q^3 (x = lam w - s,
    w^3 + p w + 1 = 0), the identity where the library computes in the reference basis"""
    from pbc_b200.pairing import PairingError
    try:
        s, lam, p = pr.derived_constant_n("basis_cubic", pr.g1_len // 2, 3)
    except PairingError:
        return None

    def fwd(a):                     # f3_to_internal
        a0, a1, a2 = a
        return ((a0 - a1 * s + a2 * s * s) % q, lam * (a1 - 2 * s * a2) % q, lam * lam * a2 % q)

    li = pow(lam, q - 2, q)

    def inv(b):                     # f3_to_reference
        b0, b1, b2 = b
        a2 = b2 * li * li % q
        a1 = (b1 * li + 2 * s * a2) % q
        return ((b0 + a1 * s - a2 * s * s) % q, a1, a2)

    return fwd, inv, p


def _w_mul(x, y, p, q):
    """product in F_q[w]/(w^3 + p w + 1): the internal basis of the F_q^3 kernels"""
    d = [0] * 5
    for i in range(3):
        for j in range(3):
            d[i + j] += x[i] * y[j]
    return ((d[0] - d[3]) % q, (d[1] - p * d[3] - d[4]) % q, (d[2] - p * d[4]) % q)


def _f3_extremes(q, T):
    """F_q^3 elements by internal coefficients.  Pairs of them, as the two operands of f3_mul / f3_sqr,
    reach the bounds of f3_fold_lazy (d0, d4 < q^2, d1, d3 < 2 q^2, d2 < 3 q^2):
      r0 = d0 + 2 q^2 - d3        max: x = y = (q-1, 0, 0);  min (4q - 2): x = y = (0, q-1, q-1)
      r1 = d1 + 2 q^2 - p d3 - d4 max: x = y = (q-1, q-1, 0); min: x = (0, 0, q-1), y = (0, q-1, q-1)
      r2 = d2 + q^2 - p d4        max: x = (q-1, q-1, 0), y = (0, q-1, q-1); min: x = y = (0, 0, q-1)
    all in the cross product of {0, q-1}^3 (the squares: the diagonal); the other targets on one
    coefficient at a time fill the carry chains"""
    m = q - 1
    E = [(a, b, c) for a in (0, m) for b in (0, m) for c in (0, m)]
    for t in T[1:8]:
        E += [(t, m, m), (m, t, m), (m, m, t), (t, t, t)]
    return E


def _d_items(q, T, rnd):
    E = _f3_extremes(q, T)
    X = [a for a in E for b in E]
    Y = [b for a in E for b in E]
    for _ in range(128):
        X.append(tuple(rnd.choice(T) for _ in range(3)))
        Y.append(tuple(rnd.choice(T) for _ in range(3)))
    return X, Y


D_TOWER = [("d159", ""), ("d159", "b200_reference_basis 1\n")] + \
          [(n, e) for n in D_WIDE for e in ("", "b200_reference_basis 1\n")]


@pytest.mark.parametrize("name,extra", D_TOWER, ids=["%s%s" % (_id(n), "_refbasis" if e else "") for n, e in D_TOWER])
def test_d_tower_on_internal_extremes(name, extra):
    """tower op 5 (f3_mul of the real halves), op 2 (f6d_inv: f3_sqr of both halves first) and op 0
    (f6d_mul: f3_mul of the two real halves first) with internally extreme F_q^3 coefficients"""
    pr, text = _dev(name, extra)
    orc = O.pairing_from_param(text)
    q = orc.q
    D = Dom(q, LIMBS[FAMILY_LIMBS[name]])
    T = targets(q, D.N)
    basis = _d_basis(pr, q)
    if basis is None:
        fwd = inv = lambda a: tuple(a)
    else:
        fwd, inv, pc = basis
        # host model of the basis change: a round trip, and a ring isomorphism onto F_q[w]/(w^3 + p w + 1)
        rnd = random.Random(5)
        for _ in range(4):
            a = tuple(rnd.randrange(q) for _ in range(3))
            b = tuple(rnd.randrange(q) for _ in range(3))
            assert fwd(inv(a)) == a and inv(fwd(a)) == a
            assert fwd(orc.Fq3.mul(a, b)) == _w_mul(fwd(a), fwd(b), pc, q)
    wb = pr.g1_len // 2

    def ref(e):                    # internal targets -> reference-basis wire coefficients
        return inv(tuple(D.wire(t) for t in e))

    X, Y = _d_items(q, T, random.Random(17))
    F3, F6 = orc.Fq3, orc.Fq6
    zero = (0, 0, 0)
    for op in (5, 2, 0):
        if op == 5:
            A = [(ref(x), zero) for x in X]
            B = [(ref(y), zero) for y in Y]
        else:
            A = [(ref(x), ref(y)) for x, y in zip(X, Y)]
            B = [(ref(y), ref(x)) for x, y in zip(X, Y)]
            if op == 2:
                keep = [i for i, a in enumerate(A) if a != (zero, zero)]
                A, B = [A[i] for i in keep], [B[i] for i in keep]
        enc = b"".join(_enc(a[0] + a[1], wb) for a in A)
        encb = b"".join(_enc(b[0] + b[1], wb) for b in B)
        got = pr.tower_op(op, enc, encb, len(A))
        L = pr.gt_len
        bad = []
        for i, (a, b) in enumerate(zip(A, B)):
            if op == 5:
                want = (F3.mul(a[0], b[0]), zero)
            elif op == 2:
                want = F6.inv(a)
            else:
                want = F6.mul(a, b)
            if got[i * L:(i + 1) * L] != F6.to_bytes(want):
                bad.append(i)
        assert not bad, "%s%s op %d: %d of %d wrong, first items %s" % (name, extra.strip(), op, len(bad), len(A), bad[:6])


def _f_basis(pr, q):
    """(forward, inverse) maps of F_q^12 coefficients between the reference basis (x, s) and the internal
    one (z = x / tau, i = s / sigma):  d_j = phi2(c_j) tau^j,  phi2(a + b s) = a + sigma b i,  i^2 = -1"""
    from pbc_b200.pairing import PairingError
    try:
        (sigma,) = pr.derived_constant("basis_sigma", 20)
        ta, tb = pr.derived_constant("basis_tau", 20)
        xa, xb = pr.derived_constant("basis_xi_small", 20)
    except PairingError:
        return None

    def kmul(x, y):
        return ((x[0] * y[0] - x[1] * y[1]) % q, (x[0] * y[1] + x[1] * y[0]) % q)

    def kinv(x):
        n = pow((x[0] * x[0] + x[1] * x[1]) % q, q - 2, q)
        return (x[0] * n % q, -x[1] * n % q)

    taup = [(1, 0)]
    for _ in range(5):
        taup.append(kmul(taup[-1], (ta, tb)))
    tauinv = [kinv(t) for t in taup]
    si = pow(sigma, q - 2, q)

    def fwd(c):
        return tuple(kmul((cj[0], sigma * cj[1] % q), taup[j]) for j, cj in enumerate(c))

    def inv(d):
        out = []
        for j, dj in enumerate(d):
            e = kmul(dj, tauinv[j])
            out.append((e[0], e[1] * si % q))
        return tuple(out)

    return fwd, inv, kmul, (xa, xb)


def _k12_mul(x, y, kmul, xi, q):
    """product in K[z]/(z^6 - xi'), K = F_q[i]/(i^2 + 1): the internal basis of the F_q^12 kernels"""
    d = [(0, 0)] * 11
    for i in range(6):
        for j in range(6):
            p = kmul(x[i], y[j])
            d[i + j] = ((d[i + j][0] + p[0]) % q, (d[i + j][1] + p[1]) % q)
    out = list(d[:6])
    for k in range(6, 11):
        p = kmul(d[k], xi)
        out[k - 6] = ((out[k - 6][0] + p[0]) % q, (out[k - 6][1] + p[1]) % q)
    return tuple(out)


def _f_patterns(q):
    """F_q^2 coefficients (re, im) in the internal basis.  f2_mul keeps re = x0 y0 - x1 y1 + q^2 and
    im = (x0 + x1)(y0 + y1) - x0 y0 - x1 y1 double width (both below 2 q^2):
      re max: (q-1, 0) x (q-1, 0);  re min (2q - 1): (0, q-1) x (0, q-1)   (only the subtracted term)
      im max: (q-1, q-1) x (q-1, q-1);  im min 0: q-1 against 0 in the Karatsuba pair, (q-1, 0) x (0, 0)
    f12_mul_line sums three such terms per coefficient (one of them c v, below q^2) before fq_redc2_call:
    below 5 q^2, the sum fq_redc2_call's second subtraction exists for.  Its maximum: every coefficient
    of v and of the line (q-1, 0) and c = q - 1 (re), every coefficient (q-1, q-1) (im)."""
    m = q - 1
    return [(0, 0), (m, 0), (0, m), (m, m), (1, m), (m, 1), ((q - 1) // 2, (q + 1) // 2), (m, (q + 1) // 2)]


@pytest.mark.parametrize("extra", ["", "b200_reference_basis 1\n"], ids=["internal_basis", "reference_basis"])
def test_f_tower_on_internal_extremes(extra):
    """tower ops 0 (f12_mul: f6_mul and its f2_mul on the input coefficients), 1 (f12_sqr), 2 (f12_inv) and
    4 (f12_mul_line: the fq_redc2_call sums on the input coefficients) with every coefficient drawn from
    the internally extreme F_q^2 patterns, all pattern pairs, plus mixed elements"""
    pr, text = _dev("f", extra)
    orc = O.pairing_from_param(text)
    q = orc.q
    D = Dom(q, LIMBS["small"])
    T = targets(q, D.N)
    basis = _f_basis(pr, q)
    F12 = orc.Fq12
    if basis is None:
        inv = lambda d: tuple(d)
    else:
        fwd, inv, kmul, xi = basis
        rnd = random.Random(6)
        for _ in range(3):
            a = tuple((rnd.randrange(q), rnd.randrange(q)) for _ in range(6))
            b = tuple((rnd.randrange(q), rnd.randrange(q)) for _ in range(6))
            assert fwd(inv(a)) == a and inv(fwd(a)) == a
            assert fwd(F12.mul(a, b)) == _k12_mul(fwd(a), fwd(b), kmul, xi, q)

    def ref(d):                    # internal targets -> reference-basis wire coefficients
        return inv(tuple((D.wire(c[0]), D.wire(c[1])) for c in d))

    P = _f_patterns(q)
    X = [tuple([p] * 6) for p in P for _ in P]
    Y = [tuple([r] * 6) for _ in P for r in P]
    rnd = random.Random(23)
    for _ in range(64):
        X.append(tuple((rnd.choice(T), rnd.choice(T)) for _ in range(6)))
        Y.append(tuple((rnd.choice(T), rnd.choice(T)) for _ in range(6)))
    # the line's c (coefficient 0, real part) at q - 1 and at 0
    for p in P:
        X.append(tuple([p] * 6))
        Y.append(((0, 0),) + tuple([p] * 5))
    A, B = [ref(x) for x in X], [ref(y) for y in Y]
    enc = lambda es: b"".join(F12.to_bytes(e) for e in es)
    L = pr.gt_len
    F2 = orc.Fq2
    for op in (0, 1, 2, 4):
        items = [i for i in range(len(A)) if op != 2 or any(any(c) for c in A[i])]
        a, b = [A[i] for i in items], [B[i] for i in items]
        got = pr.tower_op(op, enc(a), enc(b), len(a))
        bad = []
        for k, (x, y) in enumerate(zip(a, b)):
            if op == 0:
                want = F12.mul(x, y)
            elif op == 1:
                want = F12.sqr(x)
            elif op == 2:
                want = F12.inv(x)
            else:
                line = [F2.zero] * 6
                line[0] = (y[0][0], 0)
                line[3], line[4] = y[3], y[4]
                want = F12.mul(x, tuple(line))
            if got[k * L:(k + 1) * L] != F12.to_bytes(want):
                bad.append(items[k])
        assert not bad, "f%s op %d: %d of %d wrong, first items %s" % (extra.strip(), op, len(bad), len(a), bad[:6])


def test_g_tower_on_internal_extremes():
    """type g: F_q^5 products (f5_mul: up to 45 products below q^2 summed double width before one reduction,
    the bound 45 q^2 < q R) through tower op 5 and op 0; the maximum is every coefficient q - 1"""
    pr, text = _dev("g149")
    orc = O.pairing_from_param(text)
    q = orc.q
    D = Dom(q, LIMBS["small"])
    T = targets(q, D.N)
    m = q - 1
    E = [tuple([m] * 5), tuple([0] * 5), (m, 0, m, 0, m), (0, m, 0, m, 0), (1, m, m, m, m), (m, m, m, m, 1)]
    E += [tuple([t] * 5) for t in T[1:8]]
    X = [a for a in E for b in E]
    Y = [b for a in E for b in E]
    rnd = random.Random(29)
    for _ in range(64):
        X.append(tuple(rnd.choice(T) for _ in range(5)))
        Y.append(tuple(rnd.choice(T) for _ in range(5)))
    wb = pr.g1_len // 2
    w = lambda e: tuple(D.wire(t) for t in e)
    F5, F10 = orc.Fq5, orc.Fq10
    L = pr.gt_len
    for op in (5, 0):
        if op == 5:
            A = [(w(x), (0,) * 5) for x in X]
            B = [(w(y), (0,) * 5) for y in Y]
        else:
            A = [(w(x), w(y)) for x, y in zip(X, Y)]
            B = [(w(y), w(x)) for x, y in zip(X, Y)]
        got = pr.tower_op(op, b"".join(_enc(a[0] + a[1], wb) for a in A), b"".join(_enc(b[0] + b[1], wb) for b in B), len(A))
        bad = []
        for i, (a, b) in enumerate(zip(A, B)):
            want = (F5.mul(a[0], b[0]), F5.zero) if op == 5 else F10.mul(a, b)
            if got[i * L:(i + 1) * L] != F10.to_bytes(want):
                bad.append(i)
        assert not bad, "g149 op %d: %d of %d wrong, first items %s" % (op, len(bad), len(A), bad[:6])


# ---- 4. the slot routines of the type A Miller step (fp_op 8-14) ---------------------------------

A_SLOT_OPS = {  # op: (coordinates in a, in b, in out)
    8: (2, 2, 1), 9: (2, 2, 6), 10: (1, 1, 1), 11: (2, 2, 1), 12: (2, 2, 1), 13: (2, 2, 1), 14: (1, 1, 1)}


def _a_slot_want(op, a0, a1, b0, b1, q, R):
    """exact values from the wire operands; op 9's stored sum S' from the internal ones"""
    if op == 8:
        return [(a0 * b0 + a1 * b1) % q]
    if op == 9:
        A0, A1, B0, B1 = (v * R % q for v in (a0, a1, b0, b1))
        S = A0 * B0 + A1 * B1
        if S >= q * R:
            S -= q * R
        return [(a0 * b0 - a1 * b1) % q, (a0 * b1 + a1 * b0) % q, S % R, S // R, (a0 + a1) % q, (b0 + b1) % q]
    if op == 10:
        return [(2 * a0 * a0 - b0) % q]
    if op == 11:
        return [((a0 + a1) ** 2 - b0 - b1) % q]
    if op == 12:
        return [(a0 + a1) * (b0 + b1) % q]
    if op == 13:
        return [(a0 + a1) * (b0 - b1) % q]
    return [a0 * b0 % q]


def test_a_slot_routines_on_internal_extremes():
    """Ops::lazy in the three modes of a_step_9_line, Ops::sqrx in its two and Ops::mulx in its variants, on
    the same slot machine and mode flags as the Miller step.  The bounds they rest on:
      lazy(LZ_TWO): A0 B0 + A1 B1 < 2 q^2 < 2 q R       max: every operand q - 1
      LZ_SUB | LZ_ADD_QR: A0 B0 - A1 B1 + q R in (0, 2 q R)   min: A0 B0 = 0, A1 = B1 = q - 1; max: A1 B1 = 0
      LZ_KARATSUBA: S' = A0 B0 + A1 B1 - (q R if >= q R) < q R, stored raw: every operand q - 1 reaches
        S >= q R (the one case the conditional subtraction exists for), checked as an exact integer
      LZ_SUB_S: (A0 + A1)(B0 + B1) - S' + q R in (0, 2 q R)   min: A0 + A1 = 0 (q - 1 against 1), S' max
    all in the cross product of the first eight targets (0, 1, 2, q - 1, q - 2, (q +- 1)/2, q's top limb
    less one) over the four operands"""
    pr, text = _dev("a")
    q = _q(text)
    D = Dom(q, LIMBS["a"])
    T = targets(q, D.N)
    wb = pr.g1_len // 2
    E = T[:8]
    items = [(a0, a1, b0, b1) for a0 in E for a1 in E for b0 in E for b1 in E]
    rnd = random.Random(41)
    for t in T:
        items += [(t, t, t, t), (t, q - 1, q - 1, q - 1), (q - 1, t, q - 1, q - 1), (q - 1, q - 1, t, 1),
                  (t, rnd.randrange(q), rnd.randrange(q), t)]
    W = [tuple(D.wire(t) for t in it) for it in items]
    reached = 0
    for op, (wa, wbn, wo) in sorted(A_SLOT_OPS.items()):
        A = b"".join(_enc(w[:wa], wb) for w in W)
        B = b"".join(_enc(w[2:2 + wbn], wb) for w in W)
        got = _dec(pr.fp_op(op, A, B, len(W), widths=(wa, wbn, wo)), wb)
        bad = []
        for i, w in enumerate(W):
            want = _a_slot_want(op, w[0], w[1], w[2], w[3], q, D.R)
            if got[i * wo:(i + 1) * wo] != want:
                bad.append((i, [hex(t) for t in items[i]]))
        assert not bad, "type a op %d: %d of %d wrong, first (item, internal operands) %s" % (op, len(bad), len(W), bad[:3])
        if op == 9:
            reached = sum(1 for it in items if it[0] * it[2] + it[1] * it[3] >= q * D.R)
    assert reached > 0, "no item drives A0 B0 + A1 B1 to q R"


# ---- 5. the shipped type F final exponentiation (tower op 6: k_f_finalexp_s) ---------------------

def test_f_shipped_final_exponentiation_on_chosen_inputs():
    """k_f_finalexp_s, the kernel every type F pairing ends in, against the oracle's f_tateexp on internal
    extremes, 1 and -1, elements of the subfields F_q^6 (x^0, x^2, x^4 only) and F_q^4 (x^0, x^3 only) --
    (q^6 - 1)(q^2 + 1) takes those to 1, so the hard part runs on the identity -- and random elements.
    Zero is left out: the reference divides by it."""
    pr, text = _dev("f")
    orc = O.pairing_from_param(text)
    q = orc.q
    D = Dom(q, LIMBS["small"])
    fwd, inv, _, _ = _f_basis(pr, q)
    F12 = orc.Fq12
    ref = lambda d: inv(tuple((D.wire(c[0]), D.wire(c[1])) for c in d))
    rnd = random.Random(53)
    rc = lambda: (rnd.randrange(q), rnd.randrange(q))
    zero = (0, 0)
    P = [p for p in _f_patterns(q) if p != zero]
    elems = [ref(tuple([p] * 6)) for p in P]
    elems += [ref((p,) + tuple([P[(k + j) % len(P)] for j in range(5)])) for k, p in enumerate(P[:4])]
    one = F12.one
    elems += [one, F12.neg(one)]
    sub6 = [tuple(rc() if j % 2 == 0 else zero for j in range(6)) for _ in range(3)]
    sub4 = [tuple(rc() if j % 3 == 0 else zero for j in range(6)) for _ in range(3)]
    elems += sub6 + sub4
    elems += [tuple(rc() for _ in range(6)) for _ in range(3)]
    got = pr.tower_op(6, b"".join(F12.to_bytes(e) for e in elems), None, len(elems))
    L = pr.gt_len
    for i, e in enumerate(elems):
        want = orc.final_exp(e)
        if e in sub6 or e in sub4 or e == one or e == F12.neg(one):
            assert want == one
        assert got[i * L:(i + 1) * L] == F12.to_bytes(want), "element %d" % i


def test_f_shipped_final_exponentiation_hook_refuses_the_reference_basis():
    from pbc_b200.pairing import PairingError
    pr, _ = _dev("f", "b200_reference_basis 1\n")
    with pytest.raises(PairingError, match="tower_op 6"):
        pr.tower_op(6, b"\0" * pr.gt_len, None, 1)

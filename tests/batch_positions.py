"""Large batches whose every position has an exact expected value, for tests/test_gpu_batch_positions.py.

Everything comes from one reference output and bilinearity.  With P0, Q0 the first fixture pair and
e0 = e(P0, Q0) its reference output, position i of a batch pairs uP0 with wQ0, u = 1 + i mod L1 and
w = 1 + i mod L2, and e(uP0, wQ0) = e0^(uw) exactly, wire bytes included.  The multiples uP0, wQ0 and
the powers e0^m are built by repeated addition / multiplication on the host (the oracle's group laws;
type e: tests/type_e_model.py), never by a pairing.

L1 and L2 are distinct primes above the SM count of any current GPU, so no stride the library cuts a
batch at -- thread blocks of 64, 128 and 256, the batch-inversion chain stride T = SMs * 128 or 256,
the host pipeline's chunks of 2^18 / k outputs, a device's slice -- is a multiple of either period: an
output that reads a neighbour's data at such a stride gets a different value, not an equal one.
"""
from __future__ import annotations

import functools
import json
import os

import numpy as np

from oracle import pbc_oracle as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

L1, L2 = 139, 137          # periods of the first and the second argument
LP = 7                     # period of the second argument inside products: k * L1 * LP stays below L1 * L2
CHUNK = 1 << 18            # outputs per host pipeline chunk (divided by k for products)
# the strides an output could be confused at, for a 132-SM H100: blocks, inversion chains (A1 / E, A),
# a chunk, a chunk of k = 16 products
STRIDES = (64, 128, 256, 132 * 128, 132 * 256, CHUNK, CHUNK // 16)

# every shipped parameter set: the five golden files of tests/conftest.py, type e and the wide type d sets
WIDE_D = ("d175", "d190", "d196", "d201", "d224")
NAMES = ("a", "a1", "e", "f", "d159", "g149") + WIDE_D


def load(name):
    """(golden fixtures, parameter text) of a parameter set"""
    fname = "d_wide_" + name if name in WIDE_D else name
    with open(os.path.join(ROOT, "tests", "golden", fname + ".json")) as f:
        g = json.load(f)
    if "param_text" in g:
        return g, g["param_text"]
    from pbc_b200.params import PARAMS
    return g, PARAMS[name]


def chains_per_sm(kind):
    """independent batch-inversion chains per SM (engine.cu inv_threads): 256 for type a, 128 for a1 and e;
    types f, d and g invert nothing in a batch, 256 only sizes their batches alike"""
    return 128 if kind in ("a1", "e") else 256


class _Group:
    """multiples j * X0 of one point, j = 0 .. m, grown on demand by repeated addition"""

    def __init__(self, add, neg, enc, zero_bytes, X0):
        self._add, self._neg, self._enc = add, neg, enc
        self._zero = zero_bytes
        self._pts = [None, X0]

    def _grow(self, m):
        while len(self._pts) <= m:
            self._pts.append(self._add(self._pts[-1], self._pts[1]))

    def table(self, m, negate=False):
        """uint8 array (m + 1, len): row j = the wire bytes of j * X0 (or -j * X0); row 0 = O, all zero bytes"""
        self._grow(m)
        rows = [self._zero] + [self._enc(self._neg(p) if negate else p) for p in self._pts[1:m + 1]]
        return np.frombuffer(b"".join(rows), dtype=np.uint8).reshape(m + 1, -1)


class _Powers:
    """powers e^j, j = 0 .. m, of one GT element, grown on demand by repeated multiplication"""

    def __init__(self, mul, enc, one, e):
        self._mul, self._enc = mul, enc
        self._vals = [one, e]

    def _grow(self, m):
        while len(self._vals) <= m:
            self._vals.append(self._mul(self._vals[-1], self._vals[1]))

    def table(self, m):
        self._grow(m)
        return np.frombuffer(b"".join(self._enc(v) for v in self._vals[:m + 1]), dtype=np.uint8).reshape(m + 1, -1)


class Family:
    """one parameter set: its fixtures, lengths, group laws and the tables of multiples and powers"""

    def __init__(self, name):
        self.name = name
        self.g, self.text = load(name)
        self.kind = O.parse_param(self.text)["type"]       # a, a1, e, f, d or g
        L = self.g["lengths"]
        self.g1_len, self.g2_len, self.gt_len, self.zr_len = L["g1"], L["g2"], L["gt"], L["zr"]
        pr = self.g["pairing"]
        self.P0b, self.Q0b, self.e0b = (bytes.fromhex(pr[k][0]) for k in ("P", "Q", "e"))
        off = self.g["offcurve"]
        self.badP, self.badQ = bytes.fromhex(off["badP"]), bytes.fromhex(off["badQ"])
        self.identity = bytes.fromhex(off["identity"])
        self.has_hash = "hash" in self.g
        if self.kind == "e":
            from tests import type_e_model as M
            p = M.parse_param(self.text)
            q, a, self.r = p["q"], p["a"] % p["q"], p["r"]
            wb = self.g1_len // 2
            dec = lambda b: (int.from_bytes(b[:wb], "big"), int.from_bytes(b[wb:], "big"))
            enc = lambda P: P[0].to_bytes(wb, "big") + P[1].to_bytes(wb, "big")
            add = lambda P, Q: M.add(P, Q, a, q)
            neg = lambda P: (P[0], -P[1] % q)
            self.oracle = None
            g1 = g2 = (add, neg, enc, dec)
            gt = (lambda x, y: x * y % q, lambda x: x.to_bytes(wb, "big"), 1,
                  int.from_bytes(self.e0b, "big"), lambda x: pow(x, -1, q))
        else:
            orc = self.oracle = O.pairing_from_param(self.text)
            self.r = orc.r
            g1 = (orc.G1.add, orc.G1.neg, orc.G1.to_bytes, orc.G1.from_bytes)
            g2 = (orc.G2.add, orc.G2.neg, orc.G2.to_bytes, orc.G2.from_bytes)
            gt = (orc.GT.mul, orc.GT.to_bytes, orc.GT.one, orc.GT.from_bytes(self.e0b), orc.GT.inv)
        add, neg, enc, dec = g1
        self.P = _Group(add, neg, enc, bytes(self.g1_len), dec(self.P0b))
        add, neg, enc, dec = g2
        self.Q = _Group(add, neg, enc, bytes(self.g2_len), dec(self.Q0b))
        mul, genc, one, e0, inv = gt
        self.E = _Powers(mul, genc, one, e0)
        self.Einv = _Powers(mul, genc, one, inv(e0))

    @functools.cached_property
    def q0_has_order_r(self):
        """whether r Q0 = O.  Not so for the G2 fixtures of types f, d and g: the reference's random G2 points keep
        a cofactor part, which the pairing ignores but a power by r - v does not"""
        if self.oracle is None:
            return True                                # type e: Q0 is a G1 point
        return self.oracle.G2.mul(self.r, self.oracle.G2.from_bytes(self.Q0b)) is None

    def compress(self, rows):
        """element_to_bytes_compressed of the rows of a (n, g1_len) array: x || (y mod 2)"""
        wb = self.g1_len // 2
        return np.concatenate([rows[:, :wb], rows[:, -1:] & 1], axis=1)


@functools.lru_cache(maxsize=None)
def family(name) -> Family:
    return Family(name)


# ---- layouts -----------------------------------------------------------------------------------------
def uw(n, wper=L2):
    """multipliers u = 1 + i mod L1 and w = 1 + i mod wper of positions i < n"""
    i = np.arange(n, dtype=np.int64)
    return 1 + i % L1, 1 + i % wper


def chain_positions(n, T, chunk=CHUNK):
    """positions where the batch inversion of a chunk is most easily spoilt by a zero: the first and the last
    element of a chain, two consecutive elements of one chain, the first and the last slot of 64-, 128- and
    256-thread blocks, the first and the last position of each chunk (chains are local to a chunk)"""
    pos = set()
    for lo in range(0, n, chunk):
        m = min(chunk, n - lo)
        t = min(T, m)
        # chunk ends; the first element of chain 3; two last elements of chains (both at or above m - t)
        pos |= {lo, lo + m - 1, lo + 3, lo + m - 1 - 2 * t // 3}
        if m > t + 1000:
            pos |= {lo + 1000, lo + 1000 + t}          # consecutive elements of the chain 1000 mod t
        if m > 2 * 256 * 9:
            pos |= {lo + 64 * 7, lo + 64 * 7 + 63, lo + 256 * 9, lo + 256 * 9 + 255}
    return sorted(p for p in pos if 0 <= p < n)


def pairs(fam, n, bad=()):
    """(in1, in2, want) of n plain pairings at the (u, w) layout; badP / badQ alternate at `bad`, whose outputs are 1"""
    u, w = uw(n)
    in1 = fam.P.table(L1)[u]
    in2 = fam.Q.table(L2)[w]
    want = fam.E.table(L1 * L2)[u * w]
    for t, i in enumerate(bad):
        if t % 2:
            in2[i] = np.frombuffer(fam.badQ, dtype=np.uint8)
        else:
            in1[i] = np.frombuffer(fam.badP, dtype=np.uint8)
        want[i] = np.frombuffer(fam.identity, dtype=np.uint8)
    return in1, in2, want


def products(fam, k, n_out, poison=()):
    """(in1, in2, want) of n_out products of k pairings: pair p is (uP0, wQ0) with u = 1 + p mod L1, w = 1 + p mod LP;
    output o = e0^(sum of its uw).  For o in `poison` one input of the product is made invalid: that output is 1."""
    u, w = uw(n_out * k, wper=LP)
    in1 = fam.P.table(L1)[u]
    in2 = fam.Q.table(LP)[w]
    ex = (u * w).reshape(n_out, k).sum(axis=1)
    want = fam.E.table(L1 * L2)[ex]
    for t, o in enumerate(poison):
        j = o * k + (t * 5) % k                       # a different slot of the product each time
        if t % 2:
            in2[j] = np.frombuffer(fam.badQ, dtype=np.uint8)
        else:
            in1[j] = np.frombuffer(fam.badP, dtype=np.uint8)
        want[o] = np.frombuffer(fam.identity, dtype=np.uint8)
    return in1, in2, want


def fixed_first(fam, c, n):
    """(in1 = cP0, in2, want) of n pairings with a fixed first argument: e(cP0, wQ0) = e0^(cw)"""
    _, w = uw(n)
    return fam.P.table(c)[c].copy(), fam.Q.table(L2)[w], fam.E.table(c * L2)[c * w]


def scalars(fam, n, zero_at, negative=True):
    """(v, sign, Zr bytes) of n scalars: v = 1 + i mod L2 drawn as v, r - v or v + r (where that fits the Zr width) by
    i mod 7; 0 and r alternate at `zero_at`.  The scalar is congruent to sign * v mod r (sign 0 at zero_at).
    negative=False draws v in place of r - v: for points outside the subgroup of order r, (r - v) X != -v X."""
    i = np.arange(n, dtype=np.int64)
    v = 1 + i % L2
    pick = (i % 7) % 3
    r, zl = fam.r, fam.zr_len
    if r + L2 >= 1 << (8 * zl):
        pick[pick == 2] = 0
    if not negative:
        pick[pick == 1] = 0
    sign = np.where(pick == 1, -1, 1)
    zero = set(zero_at)
    vals = [0] * n
    for t in range(n):
        vals[t] = (r - int(v[t])) if pick[t] == 1 else (int(v[t]) + (r if pick[t] == 2 else 0))
    for t, p in enumerate(sorted(zero)):
        vals[p] = 0 if t % 2 == 0 else r
        sign[p] = 0
    raw = np.frombuffer(b"".join(x.to_bytes(zl, "big") for x in vals), dtype=np.uint8).reshape(n, zl)
    return v, sign, raw


def expected_points(grp, u, v, sign):
    """rows of (sign * u * v) * X0 from a group's tables (all-zero bytes where sign is 0)"""
    m = L1 * L2
    pos, neg = grp.table(m), grp.table(m, negate=True)
    ex = u * v
    out = np.where((sign < 0)[:, None], neg[ex], pos[ex])
    out[sign == 0] = 0
    return out


def expected_gt_powers(fam, u, v, sign):
    """rows of e0^(sign * u * v) (1 where sign is 0)"""
    m = L1 * L2
    ex = u * v
    out = np.where((sign < 0)[:, None], fam.Einv.table(m)[ex], fam.E.table(m)[ex])
    out[sign == 0] = fam.E.table(0)[0]
    return out


# ---- checking ----------------------------------------------------------------------------------------
def mismatches(got, want):
    """positions whose rows differ; `got` is bytes or a uint8 array, `want` a (n, len) uint8 array"""
    g = np.frombuffer(got, dtype=np.uint8) if isinstance(got, (bytes, bytearray)) else np.asarray(got, dtype=np.uint8)
    g = g.reshape(want.shape)
    return np.nonzero((g != want).any(axis=1))[0]


def describe(bad, n, strides=STRIDES):
    """how many positions differ, the first of them, and which of the kernels' strides they share"""
    if len(bad) == 0:
        return "all %d positions exact" % n
    first = ", ".join(str(int(b)) for b in bad[:12])
    common = [s for s in strides if len(bad) > 1 and np.all((bad - bad[0]) % s == 0)]
    return "%d of %d positions differ (first: %s%s)" % (
        len(bad), n, first, "; all congruent modulo %s" % common if common else "")


def differ_fraction(want, s):
    """fraction of positions i < n - s whose expected output differs from that of position i + s"""
    a, b = want[:-s], want[s:]
    return float((a != b).any(axis=1).mean())

"""Inputs for comparing the library with the compiled reference at test time (oracle/_ref/libpbcref.so,
bound by oracle/ref.py), for every shipped parameter set.  No test functions: the GPU comparisons are
tests/test_gpu_live_reference.py, the checks that every generator makes what it claims are
tests/test_live_reference_inputs.py.

Each generator draws from its own seeded random.Random (and reseeds the reference's own generator
before reference draws), so a run repeats exactly.  The classes are the ones the fixtures do not
reach: independent random pairs at batch scale, points of E(F_q) outside the order-r subgroup,
non-canonical coordinates (v + q), GT-field elements outside GT, scalars across the whole Zr wire
width, hash data around the width of q and with a chosen number of halvings, and the edges of
point decompression."""
from __future__ import annotations

import contextlib
import json
import os

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_LIB = os.path.join(ROOT, "oracle", "_ref", "libpbcref.so")
SETS = ("a", "a1", "e", "f", "d159", "g149", "d175", "d190", "d196", "d201", "d224")
WIDE_D = ("d175", "d190", "d196", "d201", "d224")


def param_text(name):
    if name in WIDE_D:
        with open(os.path.join(ROOT, "tests", "golden", "d_wide_%s.json" % name)) as f:
            return json.load(f)["param_text"]
    from pbc_b200.params import PARAMS
    return PARAMS[name]


def _tab(text):
    toks = [t for line in text.splitlines() for t in line.split("#")[0].split()]
    return dict(zip(toks[::2], toks[1::2]))


class SetInfo:
    """The numbers of one parameter set that the generators need: the base field q, the group order r
    (n for a1, whose Zr is mod n), the curve y^2 = x^3 + a x + b of G1 and how many points of E(F_q)
    lie outside G1 (cofactor > 1)."""

    def __init__(self, name):
        self.name = name
        self.text = param_text(name)
        t = _tab(self.text)
        self.type = t["type"]
        if self.type == "a1":
            self.q, self.r = int(t["p"]), int(t["n"])
            self.a, self.b, self.cofactor = 1, 0, int(t["l"])
        elif self.type == "a":
            self.q, self.r = int(t["q"]), int(t["r"])
            self.a, self.b, self.cofactor = 1, 0, int(t["h"])
        elif self.type == "f":
            self.q, self.r = int(t["q"]), int(t["r"])
            self.a, self.b, self.cofactor = 0, int(t["b"]), 1     # #E(F_q) = r
        else:                                                     # e, d, g
            self.q, self.r = int(t["q"]), int(t["r"])
            self.a, self.b, self.cofactor = int(t["a"]) % self.q, int(t["b"]) % self.q, int(t["h"])
        self.wb = (self.q.bit_length() + 7) // 8                  # bytes of one F_q coordinate
        self.count = self.wb                                      # pbc_mpz_from_hash's buffer length
        self.zlen = (self.r.bit_length() + 7) // 8

    def rhs(self, x):
        return (x * x * x + self.a * x + self.b) % self.q

    def legendre(self, v):
        v %= self.q
        return 0 if v == 0 else (1 if pow(v, (self.q - 1) // 2, self.q) == 1 else -1)

    def fits_plus_q(self, v):
        """v + q still fits the wire width and is not the non-canonical form of 0"""
        return v % self.q != 0 and v + self.q < 1 << (8 * self.wb)

    def be(self, v):
        return v.to_bytes(self.wb, "big")

    def coords(self, elem):
        return [int.from_bytes(elem[i:i + self.wb], "big") for i in range(0, len(elem), self.wb)]

    def from_coords(self, cs):
        return b"".join(self.be(c) for c in cs)


# ---- the reference -----------------------------------------------------------------------------

def ref_missing_message():
    return ("oracle/_ref/libpbcref.so is missing: run `python __graft_entry__.py` where the reference "
            "sources are")


@contextlib.contextmanager
def open_ref(name, seed):
    """one reference pairing_t for the set, its random generator seeded; cleared on exit"""
    from oracle.ref import RefPairing
    ref = RefPairing(param_text(name))
    RefPairing.seed(seed)
    try:
        yield ref
    finally:
        ref.close()


def split(buf, width):
    return [buf[i:i + width] for i in range(0, len(buf), width)]


def infinity_as_zero(out, width, inf):
    """the reference's output with each element flagged as the point at infinity replaced by zero
    bytes, the library's encoding of it (include/pbc_b200.h, powers in G1 and G2): the reference leaves
    stale coordinates behind its infinity flag, which can decode to a point on the curve, so the flag
    comes from the caller"""
    return b"".join(bytes(width) if f else e for e, f in zip(split(out, width), inf))


# ---- generators ----------------------------------------------------------------------------------

def random_pairs(ref, n):
    """n independent element_random draws from G1 and from G2"""
    from oracle.ref import G1, G2
    return ref.random(G1, n), ref.random(G2, n)


def curve_x_with_point(info, rnd, n):
    """n random x below q whose right-hand side is a nonzero square (y = 0 excluded)"""
    xs = []
    while len(xs) < n:
        x = rnd.randrange(info.q)
        if info.legendre(info.rhs(x)) == 1:
            xs.append(x)
    return xs


def off_subgroup_points(info, ref, rnd, n):
    """points of E(F_q) (G1's curve) outside the order-r subgroup: the reference's decompression of random
    x (element_from_bytes_compressed takes any x with a point, not only G1's) with r P != O; [] when
    the cofactor is 1 and E(F_q) is G1.  Type e builds them on the host (tests/type_e_model.py): the library only
    takes them as second arguments."""
    from tests.type_e_model import mul, sqrt_mod
    if info.cofactor == 1:
        return []
    out = []
    while len(out) < n:
        x = curve_x_with_point(info, rnd, 1)[0]
        if info.type == "e":
            p = info.be(x) + info.be(sqrt_mod(info.rhs(x), info.q))
        else:
            from oracle.ref import G1
            p = ref.decompress(G1, info.be(x) + bytes([rnd.randrange(2)]), 1)
        if mul(info.r, tuple(info.coords(p)), info.a, info.q) is not None:     # one in `cofactor` is in G1
            out.append(p)
    return out


def non_canonical(info, elem):
    """the same element with every coordinate v replaced by v + q where that fits the width (never for
    v = 0 mod q); None if no coordinate can be replaced"""
    cs = info.coords(elem)
    out = [c + info.q if info.fits_plus_q(c) else c for c in cs]
    return None if out == cs else info.from_coords(out)


def non_canonical_many(info, elems, n):
    """up to n non-canonical encodings from a list of elements"""
    out = []
    for e in elems:
        v = non_canonical(info, e)
        if v is not None:
            out.append(v)
            if len(out) == n:
                break
    return out


def gt_field_elements(info, rnd, k_coords, n):
    """random F_q^k elements (all coordinates below q, almost surely outside GT), then the zero element,
    the identity and non-canonical encodings of random ones (v + q where it fits, never for v = 0)"""
    out = [info.from_coords([rnd.randrange(info.q) for _ in range(k_coords)]) for _ in range(n)]
    out.append(bytes(k_coords * info.wb))
    out.append(info.from_coords([1] + [0] * (k_coords - 1)))
    room = (1 << (8 * info.wb)) - info.q
    for _ in range(max(2, n // 4)):
        cs = [rnd.randrange(1, min(info.q, room)) + info.q if rnd.randrange(2) else rnd.randrange(1, info.q)
              for _ in range(k_coords)]
        if all(c < info.q for c in cs):
            cs[0] = rnd.randrange(1, min(info.q, room)) + info.q
        out.append(info.from_coords(cs))
    return out


def special_scalars(info):
    """r - 1, r, r + 1, the largest multiple of r below 2^(8 zlen), 2^(8 zlen) - 1 and 0 (n for a1)"""
    top = (1 << (8 * info.zlen)) - 1
    return [info.r - 1, info.r, info.r + 1, top // info.r * info.r, top, 0]


def scalars(info, rnd, n):
    """n random values across all 8 zlen bits, then the special ones: as integers"""
    return [rnd.getrandbits(8 * info.zlen) for _ in range(n)] + special_scalars(info)


def scalar_bytes(info, ks):
    return b"".join(k.to_bytes(info.zlen, "big") for k in ks)


def mpz_from_hash(q, data):
    """pbc_mpz_from_hash (x from the hash, and how many halvings it took)"""
    count = (q.bit_length() + 7) // 8
    buf, counter = b"", 0
    while True:
        if len(data) >= count - len(buf):
            buf += data[:count - len(buf)]
            break
        buf += data
        buf += bytes([counter])
        counter = (counter + 1) & 0xFF
        if len(buf) == count:
            break
    z, halvings = int.from_bytes(buf, "big"), 0
    while z > q:
        z >>= 1
        halvings += 1
    return z, halvings


def hash_is_infinity(info, data):
    """whether element_from_hash on G1 gives the point at infinity (curve_from_hash, ecc/curve.c:455-482:
    x from the hash, x <- x^2 + 1 until x^3 + a x + b is a square, then the cofactor multiple, which is O
    where the point's order divides the cofactor -- x = 1 on type a, for one)"""
    from tests.type_e_model import mul, sqrt_mod
    x = mpz_from_hash(info.q, data)[0] % info.q
    while info.legendre(info.rhs(x)) < 0:
        x = (x * x + 1) % info.q
    t = info.rhs(x)
    return mul(info.cofactor, (x, sqrt_mod(t, info.q) if t else 0), info.a, info.q) is None


def max_halvings(info):
    return mpz_from_hash(info.q, b"\xff" * info.count)[1]


def hash_data_by_length(info, rnd, per_length):
    """{length: per_length random hashes of that length, back to back} for every length 1 .. 2 count + 2"""
    return {L: bytes(rnd.getrandbits(8) for _ in range(L * per_length)) for L in range(1, 2 * info.count + 3)}


def hash_data_by_value(info, rnd):
    """hashes of `count + 3` bytes whose first count bytes read as 0, 1, q - 1, q, q + 1 and all ones
    (the bytes after them do not enter the value): (label, data)"""
    top = (1 << (8 * info.count)) - 1
    vals = [("0", 0), ("1", 1), ("q-1", info.q - 1), ("q", info.q), ("q+1", info.q + 1), ("ones", top)]
    return [(lab, v.to_bytes(info.count, "big") + bytes(rnd.getrandbits(8) for _ in range(3)))
            for lab, v in vals if v <= top]


def hash_data_by_halvings(info, rnd, per_j=2):
    """for each j = 0 .. max, hashes of count bytes whose value takes exactly j halvings: j = 0 is a
    value <= q, j >= 1 lies in [(q + 1) 2^(j-1), (q + 1) 2^j) below 2^(8 count).  (j, data)"""
    top = 1 << (8 * info.count)
    out = []
    for j in range(max_halvings(info) + 1):
        lo, hi = (0, info.q + 1) if j == 0 else ((info.q + 1) << (j - 1), min((info.q + 1) << j, top))
        for i in range(per_j):
            v = hi - 1 if i == 0 and j else lo + rnd.randrange(hi - lo)
            out.append((j, v.to_bytes(info.count, "big")))
    return out


def decompression_inputs(info, rnd, n):
    """(label, x || sign byte): random x with both sign bytes; x = 0, 1 and q - 1; non-canonical x;
    sign bytes 2 and 0xFF.  An x with no point, or whose point has y = 0, is dropped (no point: the
    library writes zero bytes, tested elsewhere; y = 0: defined differently by include/pbc_b200.h)."""
    keep = lambda x: info.legendre(info.rhs(x)) == 1
    out = []
    for x in curve_x_with_point(info, rnd, n):
        out.append(("random", info.be(x) + bytes([rnd.randrange(2)])))
    for lab, x in (("0", 0), ("1", 1), ("q-1", info.q - 1)):
        if keep(x):
            out += [(lab, info.be(x) + b"\0"), (lab, info.be(x) + b"\1")]
    room = (1 << (8 * info.wb)) - info.q
    nc = [x for x in (1, 2, 3, 5, info.q - 1) if x < room and keep(x)]
    nc += [x for x in curve_x_with_point(info, rnd, 4 * n) if x < room][:n]
    for x in nc:
        out.append(("x+q", info.be(x + info.q) + bytes([rnd.randrange(2)])))
    for x in curve_x_with_point(info, rnd, 4):
        for s in (2, 0xFF):
            out.append(("sign%d" % s, info.be(x) + bytes([s])))
    return out

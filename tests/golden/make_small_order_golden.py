"""Generate tests/golden/small_order.json: element_pow_zn on curve points whose order is not r, expected
bytes from the compiled, unmodified reference (oracle/_ref), seeded.

Run next to the reference sources:  make -C oracle && python tests/golden/make_small_order_golden.py

The power kernels run a Jacobian double-and-add whose mixed addition meets V = O, V = P and V = -P
only when the order of P is not r; these fixtures reach those branches on purpose.
  * G1 of a, d159, e and the five wide type D sets, G2 (the twist) of f, d159, g149 and the wide D sets:
    for each prime-power factor m <= MAX_M (of a prime below SMALL_P) of the group order, a point of
    exact order m (a random curve point times order / m; y = 0 points are skipped, the library decodes
    them as O).  Type a also gets the composite orders 4, 6 and 12.  Factors left out, and sets without
    any, are recorded under "uncovered".
  * a1_composite: a type a1 set with n = p1 p2 (two 512-bit primes, l the least multiple of 4 with
    p = l n - 1 prime, as pbc_param_init_a1_gen builds it): P1 of order p1, P2 of order p2, G of order n,
    their powers, and pairings among them.
Fixture per point: its order m and, as "multiples_sha256", the SHA-256 of the reference's
element_pow_zn(P, j) for j = 0 .. m - 1 (every multiple of P; O written as zero bytes, since the
reference leaves stale coordinates behind its infinity flag, ecc/curve.c:603-609).  Every multiple is
checked against the exact affine multiple of oracle/pbc_oracle.py's Curve, and the reference's powers
at the scalars the test uses (1 .. 2m + 1, j m +- 1, j m +- 2, r - 1, r, r + 5, all-ones) against the
table.  For a1_composite the digest covers the powers at a1_scalars(), and the pairings are stored.
"""
import hashlib
import json
import os
import random
import sys

from sympy import isprime, nextprime

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle import ref as R  # noqa: E402
from oracle import pbc_oracle as O  # noqa: E402
from pbc_b200.params import PARAMS  # noqa: E402
from tests.small_order_points import random_point  # noqa: E402

SEED = 20261016
SMALL_P = 100           # primes below this count as small factors
MAX_M = 64              # largest point order enumerated
WIDE = ("d175", "d190", "d196", "d201", "d224")


def small_factors(N, bound):
    f = {}
    for p in range(2, bound):
        while N % p == 0:
            f[p] = f.get(p, 0) + 1
            N //= p
    return f


def primes_of(m):
    return [p for p in range(2, m + 1) if m % p == 0 and all(p % d for d in range(2, p))]


def trace_power(t, q, k):
    """trace of Frobenius of E over F_(q^k): t_k = t t_(k-1) - q t_(k-2), t_0 = 2"""
    a, b = 2, t
    for _ in range(k - 1):
        a, b = b, t * b - q * a
    return b


def twist_order(E, q, t, k, cands, rnd):
    """the candidate group order of the twist E(F_(q^k)) that kills random points"""
    pts = [random_point(E, q ** k, rnd) for _ in range(2)]
    good = [N for N in cands if all(E.mul(N, P) is None for P in pts)]
    assert len(good) == 1, (len(good), k)
    return good[0]


def find_point(E, N, m, size, rnd):
    """a point of exact order m with y != 0, or None.  Per prime power p^j of m: a random point times
    N / p^e (p^e the full power in N) lies in the p-part, which need not be cyclic; if its order p^a
    has a >= j, p^(a - j) times it has order p^j.  The sum over the primes of m has order m."""
    for _ in range(32):
        acc = None
        for p in primes_of(m):
            j = e = 0
            while m % p ** (j + 1) == 0:
                j += 1
            while N % p ** (e + 1) == 0:
                e += 1
            X = E.mul(N // p ** e, random_point(E, size, rnd))
            a, Y = 0, X
            while Y is not None:
                Y = E.mul(p, Y)
                a += 1
            if a < j:
                break
            acc = E.add(acc, E.mul(p ** (a - j), X))
        else:
            if acc is not None and not E.K.eq(acc[1], E.K.zero):
                return acc
    return None


def exact_order_points(E, N, size, rnd, extra=()):
    """per prime p < SMALL_P dividing N: a point of exact order p^j, j as large as the group and MAX_M
    allow; then one per m in extra.  What is left out goes to the `uncovered` notes."""
    pts, uncovered = [], []
    for p, e in sorted(small_factors(N, SMALL_P).items()):
        j = e
        while p ** j > MAX_M:
            j -= 1
        P = None
        while j > 0 and P is None:
            P = find_point(E, N, p ** j, size, rnd)
            if P is None:
                j -= 1
        if P is None:
            uncovered.append("%d^%d: no point of order %d with y != 0" % (p, e, p))
            continue
        if j < e:
            uncovered.append("%d^%d: exact order %d^%d taken" % (p, e, p, j))
        pts.append((p ** j, P))
    for m in extra:
        if N % m == 0 and m not in [o for o, _ in pts]:
            P = find_point(E, N, m, size, rnd)
            assert P is not None, m
            pts.append((m, P))
    big = sorted(p for p in small_factors(N, 10 ** 4) if p >= SMALL_P)
    if big:
        uncovered.append("prime factors %s are above the enumeration bound %d" % (big, SMALL_P))
    if not pts:
        uncovered.append("no factor below %d: every point of the group has order 1 or a large one" % SMALL_P)
    return pts, uncovered


def small_scalars(m, r, zlen):
    """the scalars tests/test_gpu_small_order_powers.py raises a point of order m to"""
    ks = list(range(1, 2 * m + 2)) + [j * m + d for j in (3, 7, 20) for d in (-2, -1, 1, 2)]
    return ks + [r - 1, r, r + 5, (1 << (8 * zlen)) - 1]


def a1_scalars(p1, p2, zlen):
    n = p1 * p2
    ks = [1, 2, 3]
    for p in (p1, p2):
        ks += [p - 1, p, p + 1, p + 2, 2 * p + 1, 2 * p + 3, n - p + 1]
    return ks + [n - 1, n, n + 5, (1 << (8 * zlen)) - 1]


def powers(rp, group, E, P, ks, r):
    """reference element_pow_zn of P at ks, O as zero bytes, each checked against the exact multiple"""
    pb, zlen, out = E.to_bytes(P), rp.zr_len, []
    got = rp.pow_zn(group, pb * len(ks), b"".join(k.to_bytes(zlen, "big") for k in ks), len(ks))
    for i, k in enumerate(ks):
        w = E.mul(k % r, P)
        out.append(bytes(len(pb)) if w is None else got[i * len(pb):(i + 1) * len(pb)])
        assert w is None or out[-1] == E.to_bytes(w), k
    return out


def block(rp, group, E, N, size, r, rnd, extra=()):
    pts, uncovered = exact_order_points(E, N, size, rnd, extra)
    doc = {"group_order": str(N), "points": [], "uncovered": uncovered}
    for m, P in pts:
        table = powers(rp, group, E, P, list(range(m)), r)
        ks = small_scalars(m, r, rp.zr_len)
        assert powers(rp, group, E, P, ks, r) == [table[k % r % m] for k in ks]
        doc["points"].append({"order": m, "P": E.to_bytes(P).hex(),
                              "multiples_sha256": hashlib.sha256(b"".join(table)).hexdigest()})
    return doc


def a1_composite(rnd):
    def prime512():
        return nextprime(rnd.getrandbits(512) | (1 << 511))
    p1, p2 = prime512(), prime512()
    n = p1 * p2
    l = 4
    while not isprime(l * n - 1):
        l += 4
    p = l * n - 1
    text = "type a1\np %d\nn %d\nl %d\n" % (p, n, l)
    rp = R.RefPairing(text)
    E = O.pairing_from_param(text).E
    G = None
    while G is None or E.mul(p1, G) is None or E.mul(p2, G) is None:
        G = E.mul(l, random_point(E, p, rnd))
    P1, P2 = E.mul(p2, G), E.mul(p1, G)
    doc = {"param_text": text, "p1": str(p1), "p2": str(p2), "points": []}
    ks = a1_scalars(p1, p2, rp.zr_len)
    for label, P in (("P1", P1), ("P2", P2), ("G", G)):
        digest = hashlib.sha256(b"".join(powers(rp, R.G1, E, P, ks, n))).hexdigest()
        doc["points"].append({"label": label, "P": E.to_bytes(P).hex(), "powers_sha256": digest})
    b1, b2, bg = E.to_bytes(P1), E.to_bytes(P2), E.to_bytes(G)
    PP, QQ = [b1, b1, bg], [b2, bg, b2]
    doc["pairing"] = {"P": [x.hex() for x in PP], "Q": [x.hex() for x in QQ],
                      "e": [rp.pairing(a, b, 1).hex() for a, b in zip(PP, QQ)]}
    assert rp.is_identity(R.GT, bytes.fromhex(doc["pairing"]["e"][0]))
    PP, QQ = [b1, b2, bg, b1], [bg, bg, b2, b2]
    doc["prod"] = {"k": 4, "P": [x.hex() for x in PP], "Q": [x.hex() for x in QQ],
                   "e": rp.prod_pairing(b"".join(PP), b"".join(QQ), 4, 1).hex()}
    QQ = [bg, b2, E.to_bytes(E.mul(2, G)), b1]
    e = rp.pp_pairing(b1, b"".join(QQ), len(QQ))
    doc["pp"] = {"P": b1.hex(), "Q": [x.hex() for x in QQ],
                 "e": [e[i * rp.gt_len:(i + 1) * rp.gt_len].hex() for i in range(len(QQ))]}
    return doc


def main():
    rnd = random.Random(SEED)
    R.RefPairing.seed(SEED)
    doc = {"source": "oracle/_ref/libpbcref.so (unmodified reference), tests/golden/make_small_order_golden.py, seed %d" % SEED,
           "sets": {}}
    texts = {name: PARAMS[name] for name in ("a", "d159", "e", "f", "g149")}
    for name in WIDE:
        with open(os.path.join(ROOT, "tests", "golden", "d_wide_%s.json" % name)) as f:
            texts[name] = json.load(f)["param_text"]
    for name, text in texts.items():
        prm = O.parse_param(text)
        rp = R.RefPairing(text)
        q, r = prm["q"], prm["r"]
        entry = {"param": name if name in PARAMS else None, "param_file": None if name in PARAMS else "d_wide_%s.json" % name}
        if prm["type"] == "e":
            E = O.Curve(O.PrimeField(q), prm["a"] % q, prm["b"] % q)
            N = prm["h"] * r
        else:
            orc = O.pairing_from_param(text)
            E = orc.E
            N = {"a": q + 1, "d": prm.get("n"), "g": prm.get("n"), "f": r}[prm["type"]]
        assert E.mul(N, random_point(E, q, rnd)) is None
        if name != "f":
            entry["g1"] = block(rp, R.G1, E, N, q, r, rnd, extra=(4, 6, 12) if name == "a" else ())
        else:
            entry["g1"] = {"group_order": str(N), "points": [], "uncovered": ["G1 of type f has prime order r"]}
        if prm["type"] in "dfg":
            Et = orc.Et
            t = q + 1 - N
            if prm["type"] == "d":
                cands = [q ** 3 + 1 + trace_power(t, q, 3)]
                k = 3
            elif prm["type"] == "g":
                cands = [q ** 5 + 1 + trace_power(t, q, 5)]
                k = 5
            else:
                import math
                t2 = trace_power(t, q, 2)
                f2 = (4 * q * q - t2 * t2) // 3
                fs = math.isqrt(f2)
                assert fs * fs == f2
                cands = [q * q + 1 - c for c in (t2, -t2, (t2 + 3 * fs) // 2, (t2 - 3 * fs) // 2,
                                                  (-t2 + 3 * fs) // 2, (-t2 - 3 * fs) // 2)]
                k = 2
            N2 = twist_order(Et, q, t, k, cands, rnd)
            assert N2 % r == 0
            entry["g2"] = block(rp, R.G2, Et, N2, q ** k, r, rnd)
        doc["sets"][name] = entry
        print(name, {g: ([p["order"] for p in entry[g]["points"]], entry[g]["uncovered"]) for g in ("g1", "g2") if g in entry},
              flush=True)
    doc["a1_composite"] = a1_composite(rnd)
    path = os.path.join(ROOT, "tests", "golden", "small_order.json")
    with open(path, "w") as f:
        json.dump(doc, f, indent=1)
    print("wrote", path)


if __name__ == "__main__":
    main()

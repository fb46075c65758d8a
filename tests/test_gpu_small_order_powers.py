"""element_pow_zn on curve points whose order is not r: points of small order on G1 of a, d159, e and
the wide type D sets and on the twists (G2) of d159, g149 and the wide D sets, and the subgroup
elements of a type a1 group of composite order n = p1 p2 (BGN-style).  The running multiple of the
double-and-add meets O, P and -P there, which a point of order r never does below r.

Expected values: tests/golden/small_order.json (digests of the compiled reference's element_pow_zn,
O written as zero bytes; see tests/golden/make_small_order_golden.py) and the exact affine multiples of
oracle/pbc_oracle.py (tests/type_e_model.py for e).  Ids that start with d_wide run on the eight-limb
type D instance."""
import hashlib
import json
import os
import random

import pytest

from oracle import pbc_oracle as O
from pbc_b200.params import PARAMS
from tests import type_e_model as EM

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
with open(os.path.join(ROOT, "tests", "golden", "small_order.json")) as _f:
    G = json.load(_f)
SETS = G["sets"]
A1C = G["a1_composite"]


def _cat(xs):
    return b"".join(bytes.fromhex(x) for x in xs)


def _golden(name):
    with open(os.path.join(ROOT, "tests", "golden", SETS[name]["param_file"] or name + ".json")) as f:
        return json.load(f)


def _text(name):
    return PARAMS[name] if SETS[name]["param"] else _golden(name)["param_text"]


def small_scalars(m, r, zlen):
    """1 .. 2m + 1, j m +- 1, j m +- 2, r - 1, r, r + 5 and the all-ones Zr string (as the generator)"""
    ks = list(range(1, 2 * m + 2)) + [j * m + d for j in (3, 7, 20) for d in (-2, -1, 1, 2)]
    return ks + [r - 1, r, r + 5, (1 << (8 * zlen)) - 1]


def a1_scalars(p1, p2, zlen):
    n = p1 * p2
    ks = [1, 2, 3]
    for p in (p1, p2):
        ks += [p - 1, p, p + 1, p + 2, 2 * p + 1, 2 * p + 3, n - p + 1]
    return ks + [n - 1, n, n + 5, (1 << (8 * zlen)) - 1]


_pairings = {}


def _dev(text):
    from pbc_b200.pairing import Pairing
    if text not in _pairings:
        _pairings[text] = Pairing(text)
    return _pairings[text]


@pytest.fixture(scope="module", autouse=True)
def _release():
    yield
    for pr in _pairings.values():
        pr.clear()
    _pairings.clear()


def _curve(name, group):
    """(oracle curve, multiply(k, P), Zr modulus) of a set's G1 or G2"""
    prm = O.parse_param(_text(name))
    if prm["type"] == "e":
        q, a = prm["q"], prm["a"] % prm["q"]
        return O.Curve(O.PrimeField(q), a, prm["b"] % q), (lambda k, P: EM.mul(k, P, a, q) if k else None), prm["r"]
    orc = O.pairing_from_param(_text(name))
    E = orc.E if group == "g1" else orc.Et
    return E, E.mul, orc.r


CASES = [pytest.param(n, g, id="%s%s-%s" % ("" if SETS[n]["param"] else "d_wide_", n, g))
         for n in SETS for g in ("g1", "g2") if g in SETS[n] and SETS[n][g]["points"]]


def _pow(d, group):
    return d.g1_pow_zn if group == "g1" else d.g2_pow_zn


@pytest.mark.parametrize("name,group", CASES)
def test_powers_of_small_order_points_match_reference_fixtures(name, group):
    """per point of order m, one launch: P^j for j < m against the reference's digest, then the
    scalars of small_scalars against that table"""
    d = _dev(_text(name))
    r = O.parse_param(_text(name))["r"]
    pts = SETS[name][group]["points"]
    items = [(p, j) for p in pts for j in range(p["order"])] + [(p, k) for p in pts for k in small_scalars(p["order"], r, d.zr_len)]
    got = _pow(d, group)(b"".join(bytes.fromhex(p["P"]) for p, _ in items),
                         b"".join(k.to_bytes(d.zr_len, "big") for _, k in items), len(items))
    L = len(bytes.fromhex(pts[0]["P"]))
    out = [got[i * L:(i + 1) * L] for i in range(len(items))]
    tables, i = {}, 0
    for p in pts:
        tables[p["P"]] = out[i:i + p["order"]]
        i += p["order"]
        assert hashlib.sha256(b"".join(tables[p["P"]])).hexdigest() == p["multiples_sha256"], p["order"]
    bad = [(p["order"], k) for (p, k), o in zip(items[i:], out[i:]) if o != tables[p["P"]][k % r % p["order"]]]
    assert not bad, "%d of %d wrong, (order, k): %s" % (len(bad), len(items) - i, bad[:12])


@pytest.mark.parametrize("name,group", CASES)
def test_mixed_batch_of_small_order_and_order_r_points_against_the_oracle(name, group):
    """one launch of 400 powers, small-order points interleaved with order-r fixture points so that
    threads on the exceptional branches share warps with threads that are not; seeded scalars"""
    E, mul, r = _curve(name, group)
    d = _dev(_text(name))
    small = [(p["order"], E.from_bytes(bytes.fromhex(p["P"]))) for p in SETS[name][group]["points"]]
    big = [(r, E.from_bytes(bytes.fromhex(x))) for x in _golden(name)["pairing"]["P" if group == "g1" else "Q"]]
    zlen = d.zr_len
    rnd = random.Random("%s-%s" % (name, group))
    items = []
    for i in range(400):
        m, P = small[i % len(small)] if i % 3 != 1 else big[i % len(big)]
        k = rnd.choice([rnd.randrange(1, 3 * m + 3) if m < r else rnd.randrange(1, 64), rnd.randrange(r),
                        rnd.randrange(1, 4) * m + rnd.choice((-2, -1, 0, 1, 2))]) % (1 << (8 * zlen))
        items.append((P, k))
    got = _pow(d, group)(b"".join(E.to_bytes(P) for P, _ in items), b"".join(k.to_bytes(zlen, "big") for _, k in items),
                         len(items))
    L = E.nbytes
    bad = []
    for i, (P, k) in enumerate(items):
        w = mul(k % r, P)
        if got[i * L:(i + 1) * L] != (bytes(L) if w is None else E.to_bytes(w)):
            bad.append((i, k))
    assert not bad, "%d of %d wrong: %s" % (len(bad), len(items), bad[:12])


# ---- type a1 with composite n = p1 p2 ------------------------------------------------------------

@pytest.fixture(scope="module")
def a1c():
    return _dev(A1C["param_text"]), O.pairing_from_param(A1C["param_text"])


def test_a1_composite_subgroup_powers(a1c):
    """P1, P2 (orders p1, p2) and G (order n) at the scalars around p1, p2 and n: the reference's
    digest and the oracle; p1 + 2 and 2 p1 + 1 on P1 give 2 P1 and P1, not O"""
    d, orc = a1c
    p1, p2 = int(A1C["p1"]), int(A1C["p2"])
    ks = a1_scalars(p1, p2, d.zr_len)
    E, L = orc.E, d.g1_len
    for pt in A1C["points"]:
        got = d.g1_pow_zn(bytes.fromhex(pt["P"]) * len(ks), b"".join(k.to_bytes(d.zr_len, "big") for k in ks), len(ks))
        P = E.from_bytes(bytes.fromhex(pt["P"]))
        bad = [k for i, k in enumerate(ks)
               if got[i * L:(i + 1) * L] != (lambda w: bytes(L) if w is None else E.to_bytes(w))(E.mul(k % orc.r, P))]
        assert not bad, (pt["label"], bad)
        assert hashlib.sha256(got).hexdigest() == pt["powers_sha256"], pt["label"]
        if pt["label"] == "P1":
            assert got[ks.index(p1 + 2) * L:][:L] == E.to_bytes(E.dbl(P))
            assert got[ks.index(2 * p1 + 1) * L:][:L] == bytes.fromhex(pt["P"])


def test_a1_composite_pairings_match_reference_fixtures(a1c):
    d, orc = a1c
    pg = A1C["pairing"]
    got = d.apply(_cat(pg["P"]), _cat(pg["Q"]), len(pg["e"]))
    assert got == _cat(pg["e"])
    assert got[:d.gt_len] == orc.GT.to_bytes(orc.GT.one)             # e(P1, P2) = 1
    pr = A1C["prod"]
    assert d.prod_apply(_cat(pr["P"]), _cat(pr["Q"]), pr["k"], 1) == bytes.fromhex(pr["e"])
    pp = A1C["pp"]
    h = d.pp_init(bytes.fromhex(pp["P"]))
    try:
        assert h.apply(_cat(pp["Q"]), len(pp["Q"])) == _cat(pp["e"])
    finally:
        h.clear()


def test_a1_composite_power_then_pair_is_bilinear_on_device(a1c):
    """e(P1^(p1 + 2), Q) == e(P1, Q)^2, both sides on the device"""
    d, _ = a1c
    P1 = bytes.fromhex(A1C["points"][0]["P"])
    Qs = [bytes.fromhex(p["P"]) for p in A1C["points"][1:]]
    n = len(Qs)
    aP = d.g1_pow_zn(P1 * n, (int(A1C["p1"]) + 2).to_bytes(d.zr_len, "big") * n, n)
    assert aP[:d.g1_len] != bytes(d.g1_len)
    rhs = d.gt_pow_zn(d.apply(P1 * n, b"".join(Qs), n), (2).to_bytes(d.zr_len, "big") * n, n)
    assert d.apply(aP, b"".join(Qs), n) == rhs


def test_device_pointer_power_of_small_order_points():
    """g1_pow_zn_device (torch tensors in device memory) on the type a points against the host entry"""
    torch = pytest.importorskip("torch")
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    d = _dev(PARAMS["a"])
    r = O.parse_param(PARAMS["a"])["r"]
    pts = SETS["a"]["g1"]["points"]
    items = [(p["P"], k) for p in pts for k in small_scalars(p["order"], r, d.zr_len)]
    P = b"".join(bytes.fromhex(x) for x, _ in items)
    K = b"".join(k.to_bytes(d.zr_len, "big") for _, k in items)
    dP = torch.frombuffer(bytearray(P), dtype=torch.uint8).cuda()
    dK = torch.frombuffer(bytearray(K), dtype=torch.uint8).cuda()
    out = torch.empty(len(P), dtype=torch.uint8, device="cuda")
    d.g1_pow_zn_device(out.data_ptr(), dP.data_ptr(), dK.data_ptr(), len(items), torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    assert bytes(out.cpu().numpy().tobytes()) == d.g1_pow_zn(P, K, len(items))

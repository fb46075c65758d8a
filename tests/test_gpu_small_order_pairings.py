"""Pairings, products, fixed-argument pairings and is_almost_coddh on the inputs where the Miller walk
meets degenerate geometry, against the compiled reference (oracle/_ref/libpbcref.so) at test time:

  - first arguments of small order (tests/golden/small_order.json; not type e, whose value for a first
    argument outside G1 is undefined): the running multiple V reaches O, P or -P, chords turn
    vertical and line values can be 0;
  - second arguments of small order: points of E(F_q) for a and e, twist points for d and g;
  - twist points drawn without cofactor multiplication (almost surely outside G2) for f, d and g;
  - twist points with y = 0, wherever the twist has them (x a root of x^3 + a x + b), and the points of
    E(F_q) with y = 0;
  - the subgroup elements of a type a1 group of composite order n = p1 p2: e(P1, P2) = 1.

Where the reference's own computation divides by zero (_kind) the reference's bytes are a by-product of
that, or it exits with "division by zero"; it is not called there, and the library's value is the one
include/pbc_b200.h defines:
  - "inf": a point of E(F_q) with y = 0 decodes as O: the pairing is 1, and so is a product holding it;
  - "one": type a, the walk over P reaches O or its last chord joins V to itself; type g, the Miller
    value lies in F_q^5 (the Lucas step would divide by P^2 - 4 = 0): the pairing is 1; a type a
    product holding such a pair is 1, a type g product is the product of the others;
  - "zero": types f, d, g, the walk over P reaches O: the Miller value is 0 and so is the output (the
    zero of F_q^k, outside GT), for pairings, pp and any product holding such a pair.
Every other case is bit-identical to the reference.  DEGENERATE pins how many cases of each kind
every set has, so that a shift in the classification is noticed.

Degenerate pairs are interleaved with regular ones inside one warp and one block.  The five wide type D
sets run on the eight-limb type D instance.  PBC_LIVE_REFERENCE_REDUCED=1 shrinks the batches, for
the CPU simulator of the library (tests/test_live_reference_inputs.py)."""
import json
import os
import random

import pytest

from oracle import pbc_oracle as O
from tests import live_reference as L
from tests import small_order_points as S
from tests.test_gpu_live_reference import _torch_device_call

pytestmark = pytest.mark.gpu
REDUCED = bool(os.environ.get("PBC_LIVE_REFERENCE_REDUCED"))
N_REGULAR = 8 if REDUCED else 40
PROD_KS = (1, 2, 3) if REDUCED else (1, 2, 3, 17)
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
with open(os.path.join(ROOT, "tests", "golden", "small_order.json")) as _f:
    SO = json.load(_f)
SETS = tuple(s for s in L.SETS if s != "a1")          # a1: the composite-order set below
EXT_DEGREE = {"f": 2, "d": 3, "g": 5}
# {set: {kind: number of cases}} for the cases of _cases at full size
DEGENERATE = {"a": {"inf": 2, "one": 5}, "e": {}, "f": {}, "g149": {"one": 1}, "d159": {"zero": 1},
              "d175": {}, "d190": {"zero": 2}, "d196": {"zero": 1}, "d201": {"zero": 1},
              "d224": {}}


def _identity(info, gt_len):
    return b"\0" * (info.wb - 1) + b"\1" + bytes(gt_len - info.wb)


@pytest.fixture(scope="module", params=SETS, ids=["%s_set" % s for s in SETS])
def live(request):
    """(info, library handle, reference handle, oracle or None for type e)"""
    from pbc_b200.pairing import Pairing
    assert os.path.exists(L.REF_LIB), L.ref_missing_message()
    name = request.param
    info = L.SetInfo(name)
    with L.open_ref(name, 4000 + L.SETS.index(name)) as ref:
        yield info, Pairing(info.text), ref, (None if info.type == "e" else O.pairing_from_param(info.text))


def _walk_meets_o(info, orc, P):
    """whether the reference's walk over the multiples of P reaches O: type a doubles V = P exp2 times
    (a_pairing_proj); f, d and g scan the bits of r with a doubling and, on set bits, an addition of P
    (cc_miller_no_denom, the oracle's _cc_miller_affine)"""
    E, V = orc.E, orc.E.from_bytes(P)
    if info.type == "a":
        for _ in range(orc.exp2):
            V = E.dbl(V)
            if V is None:
                return True
        return False
    m = orc.r.bit_length() - 2
    while m > 0:
        V = E.dbl(V)
        if V is not None and (orc.r >> m) & 1:
            V = E.add(V, E.from_bytes(P))
        if V is None:
            return True
        m -= 1
    return False


def _a_last_chord_joins_v_to_itself(orc, P):
    """type a: the last line of the walk is the chord through V = 2^exp2 P and V1 = +-2^exp1 P; where
    V = V1 its coefficients are all 0 and so is the Miller value"""
    E, V = orc.E, orc.E.from_bytes(P)
    for i in range(orc.exp2):
        if i == orc.exp1:
            V1 = E.neg(V) if orc.sign1 < 0 else V
        V = E.dbl(V)
    return V == V1


class _LucasInput(Exception):
    pass


_LUCAS = {}


def _g_lucas_divides_by_zero(orc, P, Q):
    """type g: tatepower10's Lucas step divides by P^2 - 4, which is 0 where its input (the Miller
    value to the power (q^5 - 1)(q + 1)) is +-1, i.e. has a zero odd half"""
    if (P, Q) not in _LUCAS:
        def capture(inn):
            raise _LucasInput(inn)
        orc._lucas_even = capture
        try:
            orc.tatepower(orc.miller(orc.G1.from_bytes(P), orc.G2.from_bytes(Q)))
            raise AssertionError("tatepower did not reach the Lucas step")
        except _LucasInput as e:
            _LUCAS[P, Q] = not any(e.args[0][1])
        finally:
            del orc._lucas_even
    return _LUCAS[P, Q]


def _kind(info, orc, P, Q, special_q=()):
    """None where the reference divides by no zero (its bytes are expected), else "inf", "one" or
    "zero" (module docstring).  Type g's Lucas input is only examined for the second arguments in
    special_q: a Q in G2 with P in G1 gives a Miller value outside F_q^5."""
    if orc is None:
        return None
    Pt, Qt = orc.G1.from_bytes(P), orc.G2.from_bytes(Q)
    assert Pt is not None and Qt is not None
    if Pt[1] == 0 or (info.type == "a" and Qt[1] == 0):
        return "inf"
    if _walk_meets_o(info, orc, P):
        return "one" if info.type == "a" else "zero"
    if info.type == "a" and _a_last_chord_joins_v_to_itself(orc, P):
        return "one"
    if info.type == "g" and Q in special_q and _g_lucas_divides_by_zero(orc, P, Q):
        return "one"
    return None


def _cases(info, pr, ref, orc):
    """(label, P, Q): the degenerate pairs of the set, each with a random partner from the reference"""
    rnd = random.Random("small-order-pairings/%s" % info.name)
    ent = SO["sets"].get(info.name, {})
    Pr, Qr = (L.split(b, w) for b, w in zip(L.random_pairs(ref, 4), (pr.g1_len, pr.g2_len)))
    out = []
    if info.type != "e":
        # "neither library defines the value for a first argument outside G1" (include/pbc_b200.h, type E)
        out += [("P order %d" % p["order"], bytes.fromhex(p["P"]), Qr[i % 4])
                for i, p in enumerate(ent.get("g1", {}).get("points", []))]
        out += [("P with y = 0", orc.E.to_bytes(T), Qr[i % 4]) for i, T in enumerate(S.two_torsion(orc.E, info.q, rnd))]
    if info.type in ("a", "e"):                              # G2 is E(F_q)
        out += [("Q order %d" % p["order"], Pr[i % 4], bytes.fromhex(p["P"]))
                for i, p in enumerate(ent["g1"]["points"])]
        if info.type == "a":
            out += [("Q with y = 0", Pr[i % 4], orc.E.to_bytes(T)) for i, T in enumerate(S.two_torsion(orc.E, info.q, rnd))]
    else:
        out += [("twist Q order %d" % p["order"], Pr[i % 4], bytes.fromhex(p["P"]))
                for i, p in enumerate(ent.get("g2", {}).get("points", []))]
        size = info.q ** EXT_DEGREE[info.type]
        out += [("twist Q outside G2", Pr[i % 4], orc.Et.to_bytes(S.random_point(orc.Et, size, rnd)))
                for i in range(1 if REDUCED or info.type in ("f", "g") else 3)]
        out += [("twist Q with y = 0", Pr[i % 4], orc.Et.to_bytes(T))
                for i, T in enumerate(S.two_torsion(orc.Et, size, rnd))]
    return out


def _special_q(cases):
    return {q for lab, _, q in cases if not lab.startswith("P ")}


def test_degenerate_cases_per_set(live):
    """the number of cases of each kind is the one pinned in DEGENERATE"""
    info, pr, ref, orc = live
    cases = _cases(info, pr, ref, orc)
    sq = _special_q(cases)
    kinds = {}
    for _, P, Q in cases:
        k = _kind(info, orc, P, Q, sq)
        if k:
            kinds[k] = kinds.get(k, 0) + 1
    assert kinds == DEGENERATE[info.name], (info.name, kinds)


def _value(info, pr, kind):
    return {"inf": _identity(info, pr.gt_len), "one": _identity(info, pr.gt_len), "zero": bytes(pr.gt_len)}[kind]


def _expected(info, pr, ref, orc, pairs, special_q):
    """the expected pairing of every (P, Q), and the kinds: the reference's where it divides by no zero,
    the header's value where it does"""
    kinds = [_kind(info, orc, P, Q, special_q) for P, Q in pairs]
    reg = [i for i, k in enumerate(kinds) if k is None]
    want = [None if k is None else _value(info, pr, k) for k in kinds]
    if reg:
        got = ref.pairing(b"".join(pairs[i][0] for i in reg), b"".join(pairs[i][1] for i in reg), len(reg))
        for j, i in enumerate(reg):
            want[i] = got[j * pr.gt_len:(j + 1) * pr.gt_len]
    return want, kinds


def _batch(info, pr, ref, cases):
    """N_REGULAR random pairs with the degenerate ones at odd positions of the first warp (and the
    last position), so that they share a warp and a block with regular pairs"""
    P, Q = (L.split(b, w) for b, w in zip(L.random_pairs(ref, N_REGULAR), (pr.g1_len, pr.g2_len)))
    pairs = list(zip(P, Q))
    spots = [2 * i + 1 for i in range(len(cases) - 1)] + [10 ** 9]
    for s, (_, p, q) in sorted(zip(spots, cases), key=lambda t: t[0], reverse=True):
        pairs.insert(min(s, len(pairs)), (p, q))
    return pairs


def test_pairings_host_and_device(live):
    info, pr, ref, orc = live
    cases = _cases(info, pr, ref, orc)
    assert cases, info.name
    pairs = _batch(info, pr, ref, cases)
    n, g = len(pairs), pr.gt_len
    Pb, Qb = b"".join(p for p, _ in pairs), b"".join(q for _, q in pairs)
    want, kinds = _expected(info, pr, ref, orc, pairs, _special_q(cases))
    got = pr.apply(Pb, Qb, n)
    out = L.split(got, g)
    bad = [i for i in range(n) if out[i] != want[i]]
    assert not bad, (info.name, [(i, kinds[i]) for i in bad])
    dev = _torch_device_call(lambda o, a, b: pr.apply_device(o, a, b, n), n * g, Pb, Qb)
    assert dev in (got, None), info.name


def _product_expected(info, pr, ref, orc, pairs, special_q):
    """expected product of `pairs`: 1 if one input decodes as O (or, for type a, one pair is
    degenerate: the Miller product is 0 or the walk reaches O), 0 if one pair's Miller value is 0,
    else the reference's product of the regular pairs (type g: the "one" pairs contribute 1)"""
    kinds = [_kind(info, orc, P, Q, special_q) for P, Q in pairs]
    one = _identity(info, pr.gt_len)
    if "inf" in kinds or (info.type == "a" and "one" in kinds):
        return one
    if "zero" in kinds:
        return bytes(pr.gt_len)
    reg = [p for p, k in zip(pairs, kinds) if k is None]
    return ref.prod_pairing(b"".join(p for p, _ in reg), b"".join(q for _, q in reg), len(reg), 1) if reg else one


def _check_products(info, pr, ref, orc, cases, device):
    sq = _special_q(cases)
    P, Q = (L.split(b, w) for b, w in zip(L.random_pairs(ref, 3 * max(PROD_KS)), (pr.g1_len, pr.g2_len)))
    for k in PROD_KS:
        # output j carries one degenerate pair at the first, a middle or the last position
        outs = []
        for j, pos in enumerate((0, k // 2, k - 1)):
            row = list(zip(P[j * k:(j + 1) * k], Q[j * k:(j + 1) * k]))
            c = cases[(k + j) % len(cases)]
            row[pos] = (c[1], c[2])
            outs.append(row)
        outs.append([(c[1], c[2]) for c in (cases * k)[:k]])            # every pair degenerate
        Pb = b"".join(p for row in outs for p, _ in row)
        Qb = b"".join(q for row in outs for _, q in row)
        want = b"".join(_product_expected(info, pr, ref, orc, row, sq) for row in outs)
        assert pr.prod_apply(Pb, Qb, k, len(outs)) == want, (info.name, k)
        if device and k in (3, max(PROD_KS)):
            got = _torch_device_call(lambda o, a, b: pr.prod_apply_device(o, a, b, k, len(outs)),
                                     len(outs) * pr.gt_len, Pb, Qb)
            assert got in (want, None), (info.name, k, "device")


def test_products_with_degenerate_pairs_first_middle_last_and_all(live):
    info, pr, ref, orc = live
    _check_products(info, pr, ref, orc, _cases(info, pr, ref, orc), device=True)


@pytest.mark.parametrize("share", (2, 3))
def test_type_a_products_sharing_an_accumulator_with_a_degenerate_pair(share):
    """k_a_miller9_shared (forced through the parameter key): a degenerate pair shares its Miller
    accumulator with regular ones, so its zero or its O reaches theirs"""
    from pbc_b200.pairing import Pairing
    assert os.path.exists(L.REF_LIB), L.ref_missing_message()
    info = L.SetInfo("a")
    pr = Pairing(info.text + "\nb200_prod_share %d\n" % share)
    orc = O.pairing_from_param(info.text)
    with L.open_ref("a", 4100 + share) as ref:
        cases = _cases(info, pr, ref, orc)
        sq = _special_q(cases)
        for k in (2 * share, 3 * share):
            P, Q = (L.split(b, w) for b, w in zip(L.random_pairs(ref, 3 * k), (pr.g1_len, pr.g2_len)))
            outs = []
            for j, pos in enumerate((0, share - 1, k - 1)):
                row = list(zip(P[j * k:(j + 1) * k], Q[j * k:(j + 1) * k]))
                c = cases[(share + j) % len(cases)]
                row[pos] = (c[1], c[2])
                outs.append(row)
            Pb = b"".join(p for row in outs for p, _ in row)
            Qb = b"".join(q for row in outs for _, q in row)
            want = b"".join(_product_expected(info, pr, ref, orc, row, sq) for row in outs)
            assert pr.prod_apply(Pb, Qb, k, len(outs)) == want, (share, k)


def test_pp_degenerate_table_and_degenerate_second_arguments(live):
    """pp one-shot and through a handle: a small-order fixed first argument (the table is built from a
    degenerate walk) against regular and degenerate second arguments, and a regular first argument
    against the degenerate second arguments"""
    info, pr, ref, orc = live
    cases = _cases(info, pr, ref, orc)
    P0, Qr = L.random_pairs(ref, N_REGULAR)
    Qs = L.split(Qr, pr.g2_len)
    firsts = [P0[:pr.g1_len]] + [p for lab, p, _ in cases if lab.startswith("P ")]
    seconds = [q for lab, _, q in cases if not lab.startswith("P ")]
    for P in firsts:
        Q = [q for pair in zip(Qs, seconds + [None] * len(Qs)) for q in pair if q is not None]
        n, Qb = len(Q), b"".join(Q)
        want, _ = _expected(info, pr, ref, orc, [(P, q) for q in Q], _special_q(cases))
        one_shot = pr.pp_apply(P, Qb, n)
        h = pr.pp_init(P)
        try:
            for got in (one_shot, h.apply(Qb, n)):
                out = L.split(got, pr.gt_len)
                bad = [i for i in range(n) if out[i] != want[i]]
                assert not bad, (info.name, bad)
            half = n // 2
            assert h.apply(Qb[half * pr.g2_len:], n - half) == one_shot[half * pr.gt_len:], info.name
            dev = _torch_device_call(lambda o, b: h.apply_device(o, b, n), n * pr.gt_len, Qb)
            assert dev in (one_shot, None), info.name
            dev = _torch_device_call(lambda o, a, b: pr.pp_apply_device(o, a, b, n), n * pr.gt_len, P, Qb)
            assert dev in (one_shot, None), info.name
        finally:
            h.clear()


def test_is_almost_coddh_on_degenerate_tuples(live):
    """(a, b, c, d) with a, b or c, d degenerate: the expected flag from the expected pairings"""
    info, pr, ref, orc = live
    from oracle.ref import GT
    cases = _cases(info, pr, ref, orc)
    A, C = (L.split(b, w) for b, w in zip(L.random_pairs(ref, 2 * len(cases)), (pr.g1_len, pr.g2_len)))
    tuples = []
    for i, (lab, p, q) in enumerate(cases):
        if lab.startswith("P "):
            tuples += [(p, p, C[i], C[i]), (p, A[i], C[i], C[len(cases) + i])]
        else:
            tuples += [(A[i], A[i], q, q), (A[i], A[len(cases) + i], C[i], q)]
    n = len(tuples)
    sq = _special_q(cases)
    e1, _ = _expected(info, pr, ref, orc, [(a, d) for a, _, _, d in tuples], sq)
    e2, _ = _expected(info, pr, ref, orc, [(b, c) for _, b, c, _ in tuples], sq)
    prod = L.split(ref.mul(GT, b"".join(e1), b"".join(e2), n), pr.gt_len)
    want = bytes(int(x == y or ref.is_identity(GT, z)) for x, y, z in zip(e1, e2, prod))
    got = pr.is_almost_coddh(*(b"".join(t[j] for t in tuples) for j in range(4)), n)
    assert got == want, info.name


# ---- type a1 with composite n = p1 p2 ------------------------------------------------------------

def test_a1_composite_subgroups_against_the_reference():
    """P1, P2 (orders p1, p2) and G (order n) in every combination, as pairings, products and pp:
    e(P1, P2) = 1 (orthogonal subgroups), and every value equals the reference's"""
    from pbc_b200.pairing import Pairing
    from oracle.ref import GT, RefPairing
    assert os.path.exists(L.REF_LIB), L.ref_missing_message()
    A1C = SO["a1_composite"]
    pr = Pairing(A1C["param_text"])
    ref = RefPairing(A1C["param_text"])
    try:
        pts = [bytes.fromhex(p["P"]) for p in A1C["points"]]
        combos = [(a, b) for a in pts for b in pts][:4 if REDUCED else 9]
        P, Q = b"".join(a for a, _ in combos), b"".join(b for _, b in combos)
        want = ref.pairing(P, Q, len(combos))
        assert pr.apply(P, Q, len(combos)) == want
        assert ref.is_identity(GT, want[pr.gt_len:2 * pr.gt_len]) and combos[1] == (pts[0], pts[1])
        got = _torch_device_call(lambda o, a, b: pr.apply_device(o, a, b, len(combos)), len(want), P, Q)
        assert got in (want, None)
        k = 2
        assert pr.prod_apply(P[:2 * k * pr.g1_len], Q[:2 * k * pr.g2_len], k, 2) == \
            ref.prod_pairing(P[:2 * k * pr.g1_len], Q[:2 * k * pr.g2_len], k, 2)
        h = pr.pp_init(pts[0])
        try:
            Qs = b"".join(pts)
            assert h.apply(Qs, 3) == ref.pp_pairing(pts[0], Qs, 3) == pr.pp_apply(pts[0], Qs, 3)
        finally:
            h.clear()
    finally:
        ref.close()

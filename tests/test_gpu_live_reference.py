"""Every entry point against the compiled reference itself (oracle/_ref/libpbcref.so), called at test
time on inputs no fixture holds, for all eleven shipped parameter sets: independent random pairs at
batch scale, points of E(F_q) outside G1, non-canonical coordinates, GT-field elements outside GT,
scalars across the whole Zr wire width, hash data around the width of q and with every possible
number of halvings, products over many pairs, decompression edges (tests/live_reference.py makes the
inputs).  PBC_LIVE_REFERENCE_REDUCED=1 shrinks the batches, for the CPU simulator of the library
(tests/test_live_reference_inputs.py)."""
import os
import random

import pytest

from tests import live_reference as L

pytestmark = pytest.mark.gpu
REDUCED = bool(os.environ.get("PBC_LIVE_REFERENCE_REDUCED"))
# batches span at least two blocks of every kernel a call launches (blocks of at most 256 threads)
N_PAIRS = 12 if REDUCED else 300
PROD_KS = (1, 2, 3) if REDUCED else (1, 2, 3, 5, 8, 17, 64)
PROD_OUTPUTS = 1 if REDUCED else 2
BIG_K = 9 if REDUCED else 300
N_POW = 2 if REDUCED else 24
N_PP = 3 if REDUCED else 64


@pytest.fixture(scope="module", params=L.SETS, ids=["%s_set" % s for s in L.SETS])
def live(request):
    """(info, library handle, reference handle) of one set; the reference is cleared afterwards"""
    from pbc_b200.pairing import Pairing
    # oracle/_ref travels with the build: without it nothing below compares anything, a failure
    assert os.path.exists(L.REF_LIB), L.ref_missing_message()
    name = request.param
    info = L.SetInfo(name)
    with L.open_ref(name, 1000 + L.SETS.index(name)) as ref:
        yield info, Pairing(info.text), ref


def _rnd(info, salt):
    return random.Random("%s/%s" % (info.name, salt))


def _identity(pr):
    wb = pr.g1_len // 2
    return b"\0" * (wb - 1) + b"\1" + bytes(pr.gt_len - wb)


def _torch_device_call(fn, out_len, *bufs):
    """run a _device entry point on torch.cuda buffers holding `bufs`; returns the output bytes, or None
    on the CPU simulator of the library, which cannot read device memory (whether or not torch sees a
    GPU)"""
    from pbc_b200 import _lib
    if _lib.IS_SIMULATOR:
        return None
    import torch
    dev = [torch.frombuffer(bytearray(b), dtype=torch.uint8).cuda() for b in bufs]
    out = torch.zeros(max(1, out_len), dtype=torch.uint8, device="cuda")
    fn(out.data_ptr(), *[d.data_ptr() for d in dev])
    torch.cuda.synchronize()
    return bytes(out.cpu().numpy().tobytes())[:out_len]


def _pair_batch(info, pr, ref):
    """N_PAIRS independent random pairs with the special ones (off-subgroup first or second arguments,
    non-canonical coordinates) at the ends of 32-element blocks"""
    rnd = _rnd(info, "pairs")
    P, Q = (L.split(b, w) for b, w in zip(L.random_pairs(ref, N_PAIRS), (pr.g1_len, pr.g2_len)))
    special = []
    off = L.off_subgroup_points(info, ref, rnd, 6)
    if info.type != "e":
        # type e: "neither library defines the value for a first argument outside G1" (include/pbc_b200.h)
        special += [(o, Q[i]) for i, o in enumerate(off[:3])]
    if info.type in ("a", "a1", "e"):                 # G2 is E(F_q) as well
        special += [(P[i], o) for i, o in enumerate(off[3:])]
    for i in range(6):
        p2, q2 = L.non_canonical(info, P[i]), L.non_canonical(info, Q[i])
        if p2 or q2:
            special.append((p2 or P[i], q2 or Q[i]))
    spots = sorted({b + d for b in range(32, N_PAIRS, 32) for d in (-1, 0)} | {N_PAIRS - 1})
    for (p, q), s in zip(special, spots if not REDUCED else range(N_PAIRS)):
        P[s], Q[s] = p, q
    return b"".join(P), b"".join(Q), len(special)


def test_pairings_random_off_subgroup_and_non_canonical(live):
    info, pr, ref = live
    P, Q, nspecial = _pair_batch(info, pr, ref)
    want = ref.pairing(P, Q, N_PAIRS)
    assert nspecial > 0
    got = pr.apply(P, Q, N_PAIRS)
    bad = [i for i in range(N_PAIRS) if got[i * pr.gt_len:(i + 1) * pr.gt_len] != want[i * pr.gt_len:(i + 1) * pr.gt_len]]
    assert not bad, (info.name, bad)
    got = _torch_device_call(lambda o, a, b: pr.apply_device(o, a, b, N_PAIRS), N_PAIRS * pr.gt_len, P, Q)
    assert got in (want, None), info.name


def _mix_specials(info, pr, ref, rnd, P, Q):
    """the same pairs with some replaced by non-canonical encodings and off-subgroup points (first
    arguments outside type e, second arguments where G2 is E(F_q)), spread over the batch"""
    P, Q = L.split(P, pr.g1_len), L.split(Q, pr.g2_len)
    n = len(P)
    spots = [1, n // 3, n // 2, n - 2]
    for i in spots:
        P[i] = L.non_canonical(info, P[i]) or P[i]
        Q[i + 1] = L.non_canonical(info, Q[i + 1]) or Q[i + 1]
    off = L.off_subgroup_points(info, ref, rnd, 2)
    if off and info.type != "e":
        P[n // 4] = off[0]
    if off and info.type in ("a", "a1", "e"):
        Q[3 * n // 4] = off[1]
    return b"".join(P), b"".join(Q)


def test_products_against_the_reference(live):
    info, pr, ref = live
    rnd = _rnd(info, "prod")
    for k in PROD_KS + (BIG_K,):
        n_out = 1 if k == BIG_K else PROD_OUTPUTS
        P, Q = L.random_pairs(ref, k * n_out)
        if k >= 9:
            P, Q = _mix_specials(info, pr, ref, rnd, P, Q)
        want = ref.prod_pairing(P, Q, k, n_out)
        assert pr.prod_apply(P, Q, k, n_out) == want, (info.name, k)
        if k in (3, BIG_K):
            got = _torch_device_call(lambda o, a, b: pr.prod_apply_device(o, a, b, k, n_out), n_out * pr.gt_len, P, Q)
            assert got in (want, None), (info.name, k, "device")


def test_off_curve_pair_poisons_only_its_own_product(live):
    info, pr, ref = live
    k, n_out = 5, 3
    P, Q = (L.split(b, w) for b, w in zip(L.random_pairs(ref, k * n_out), (pr.g1_len, pr.g2_len)))
    cs = info.coords(P[k + 2])
    P[k + 2] = info.from_coords([cs[0], (cs[1] + 1) % info.q])          # off the curve: the point at infinity
    P, Q = b"".join(P), b"".join(Q)
    want = ref.prod_pairing(P, Q, k, n_out)
    got = pr.prod_apply(P, Q, k, n_out)
    assert got == want, info.name
    gt = pr.gt_len
    assert got[gt:2 * gt] == _identity(pr) and got[:gt] != _identity(pr) and got[2 * gt:] != _identity(pr)


@pytest.mark.parametrize("share", (2, 3, 4))
def test_type_a_products_with_forced_accumulator_sharing(share):
    """k_a_miller9_shared: pairs per thread sharing one Miller accumulator, forced through the parameter
    key, at odd and even k (the largest divisor of k not above the setting, 1 for a prime k)"""
    from pbc_b200.pairing import Pairing
    assert os.path.exists(L.REF_LIB), L.ref_missing_message()
    info = L.SetInfo("a")
    pr = Pairing(info.text + "\nb200_prod_share %d\n" % share)
    with L.open_ref("a", 77 + share) as ref:
        for k in ((3, 4) if REDUCED else (3, 4, 5, 6, 8, 9, 12, 300)):
            n_out = 1 if k == 300 or REDUCED else 3
            P, Q = L.random_pairs(ref, k * n_out)
            assert pr.prod_apply(P, Q, k, n_out) == ref.prod_pairing(P, Q, k, n_out), (share, k)


def test_pp_one_shot_and_handle(live):
    info, pr, ref = live
    P1, Q = L.random_pairs(ref, N_PP)
    firsts = [P1[:pr.g1_len]]
    firsts += L.non_canonical_many(info, L.split(P1, pr.g1_len), 1)
    if info.type != "e":
        firsts += L.off_subgroup_points(info, ref, _rnd(info, "pp"), 1)
    for P in firsts:
        want = ref.pp_pairing(P, Q, N_PP)
        assert pr.pp_apply(P, Q, N_PP) == want, info.name
        h = pr.pp_init(P)
        try:
            assert h.apply(Q, N_PP) == want, info.name
            half = N_PP // 2
            assert h.apply(Q[half * pr.g2_len:], N_PP - half) == want[half * pr.gt_len:], info.name
        finally:
            h.clear()


def _check_pow(info, pr, ref, group, elems, width, lib_call, lib_device):
    from oracle.ref import GT
    rnd = _rnd(info, "pow%d" % group)
    ks = L.scalars(info, rnd, N_POW)
    E, K = [], []
    for e in elems:                                    # every element with every special scalar and a random one
        for k in ks[N_POW:] + [ks[rnd.randrange(N_POW)]]:
            E.append(e)
            K.append(k)
    E += [elems[i % len(elems)] for i in range(N_POW)]
    K += ks[:N_POW]
    n = len(E)
    Eb, Kb = b"".join(E), L.scalar_bytes(info, K)
    want = ref.pow_zn(group, Eb, Kb, n)
    if group != GT:
        want = L.infinity_as_zero(want, width, [k % info.r == 0 for k in K])
    got = lib_call(Eb, Kb, n)
    bad = [i for i in range(n) if got[i * width:(i + 1) * width] != want[i * width:(i + 1) * width]]
    assert not bad, (info.name, group, [(i, K[i]) for i in bad[:8]])
    got = _torch_device_call(lambda o, a, b: lib_device(o, a, b, n), n * width, Eb, Kb)
    assert got in (want, None), (info.name, group, "device")


def test_g1_powers(live):
    info, pr, ref = live
    from oracle.ref import G1
    rnd = _rnd(info, "g1")
    pts = L.split(ref.random(G1, 4), pr.g1_len)
    pts += L.non_canonical_many(info, pts, 2)
    pts += L.off_subgroup_points(info, ref, rnd, 3)
    _check_pow(info, pr, ref, G1, pts, pr.g1_len, pr.g1_pow_zn, pr.g1_pow_zn_device)


def test_g2_powers(live):
    info, pr, ref = live
    from oracle.ref import G2
    rnd = _rnd(info, "g2")
    pts = L.split(ref.random(G2, 4), pr.g2_len)
    pts += L.non_canonical_many(info, pts, 2)
    if info.type in ("a", "a1", "e"):                 # G2 is E(F_q)
        pts += L.off_subgroup_points(info, ref, rnd, 3)
    _check_pow(info, pr, ref, G2, pts, pr.g2_len, pr.g2_pow_zn, pr.g2_pow_zn_device)


def test_gt_powers_on_gt_field_elements(live):
    info, pr, ref = live
    from oracle.ref import GT
    rnd = _rnd(info, "gt")
    elems = L.split(ref.random(GT, 3), pr.gt_len)
    elems += L.gt_field_elements(info, rnd, pr.gt_len // info.wb, 4)
    _check_pow(info, pr, ref, GT, elems, pr.gt_len, pr.gt_pow_zn, pr.gt_pow_zn_device)


def test_gt_mul_on_gt_field_elements(live):
    info, pr, ref = live
    from oracle.ref import GT
    rnd = _rnd(info, "gtmul")
    k = pr.gt_len // info.wb
    a = L.gt_field_elements(info, rnd, k, 16) + L.split(ref.random(GT, 2), pr.gt_len)
    b = L.gt_field_elements(info, rnd, k, 16) + L.split(ref.random(GT, 2), pr.gt_len)
    n = min(len(a), len(b))
    a, b = b"".join(a[:n]), b"".join(b[::-1][:n])
    assert pr.gt_mul(a, b, n) == ref.mul(GT, a, b, n), info.name


def test_is_almost_coddh(live):
    """true tuples (a, u a, c, u c), "almost" ones (d = -u c) and false ones (d random); the expected flag
    from reference pairings and the reference's GT product"""
    info, pr, ref = live
    from oracle.ref import G1, G2, GT, ZR
    n = 4 if REDUCED else 12
    A, C = L.random_pairs(ref, n)
    u = L.split(ref.random(ZR, n), info.zlen)
    neg_u = [(info.r - int.from_bytes(x, "big")).to_bytes(info.zlen, "big") for x in u]
    B = ref.pow_zn(G1, A, b"".join(u), n)
    Du = L.split(ref.pow_zn(G2, C, b"".join(u), n), pr.g2_len)
    Dn = L.split(ref.pow_zn(G2, C, b"".join(neg_u), n), pr.g2_len)
    Dr = L.split(ref.random(G2, n), pr.g2_len)
    D = b"".join((Du, Dn, Dr)[i % 3][i] for i in range(n))
    e1, e2 = ref.pairing(A, D, n), ref.pairing(B, C, n)
    prod = ref.mul(GT, e1, e2, n)
    g = pr.gt_len
    want = bytes(int(e1[i * g:(i + 1) * g] == e2[i * g:(i + 1) * g] or ref.is_identity(GT, prod[i * g:(i + 1) * g]))
                 for i in range(n))
    assert want == bytes(i % 3 != 2 for i in range(n))
    assert pr.is_almost_coddh(A, B, C, D, n) == want, info.name


def _hash_check(info, pr, ref, length, data, n, device=False):
    from oracle.ref import G1
    want = L.infinity_as_zero(ref.from_hash(G1, data, length, n), pr.g1_len,
                              [L.hash_is_infinity(info, data[i * length:(i + 1) * length]) for i in range(n)])
    got = pr.g1_from_hash(data, length, n)
    bad = [i for i in range(n) if got[i * pr.g1_len:(i + 1) * pr.g1_len] != want[i * pr.g1_len:(i + 1) * pr.g1_len]]
    assert not bad, (info.name, length, [data[i * length:(i + 1) * length].hex() for i in bad[:2]])
    if device:
        got = _torch_device_call(lambda o, d: pr.g1_from_hash_device(o, d, length, n), n * pr.g1_len, data)
        assert got in (want, None), (info.name, length, "device")


def test_hash_every_length_around_the_width_of_q(live):
    info, pr, ref = live
    if info.type == "e":
        pytest.skip("type e has no element_from_hash here (include/pbc_b200.h)")
    per = 2
    rnd = _rnd(info, "hashlen")
    lengths = L.hash_data_by_length(info, rnd, per)
    if REDUCED:
        keep = {1, info.count - 1, info.count, info.count + 1, 2 * info.count + 2}
        lengths = {k: v for k, v in lengths.items() if k in keep}
    for length, data in lengths.items():
        _hash_check(info, pr, ref, length, data, per,
                    device=length in (info.count - 1, info.count, info.count + 1) and not REDUCED)


def test_hash_values_and_halvings(live):
    info, pr, ref = live
    if info.type == "e":
        pytest.skip("type e has no element_from_hash here (include/pbc_b200.h)")
    rnd = _rnd(info, "hashval")
    vals = L.hash_data_by_value(info, rnd)
    length = info.count + 3
    _hash_check(info, pr, ref, length, b"".join(d for _, d in vals), len(vals))
    halv = L.hash_data_by_halvings(info, rnd)
    _hash_check(info, pr, ref, info.count, b"".join(d for _, d in halv), len(halv), device=not REDUCED)


def test_decompression_edges_and_compression(live):
    info, pr, ref = live
    from oracle.ref import G1
    if info.type == "e":
        pytest.skip("type e has no compressed points here (include/pbc_b200.h)")
    rnd = _rnd(info, "dec")
    items = L.decompression_inputs(info, rnd, 4 if REDUCED else 24)
    data = b"".join(d for _, d in items)
    want = ref.decompress(G1, data, len(items))
    got = pr.g1_decompress(data, len(items))
    w = pr.g1_len
    bad = [items[i][0] for i in range(len(items)) if got[i * w:(i + 1) * w] != want[i * w:(i + 1) * w]]
    assert not bad, (info.name, bad)
    pts = ref.random(G1, 8) + b"".join(L.off_subgroup_points(info, ref, rnd, 4))
    n = len(pts) // w
    assert pr.g1_compress(pts, n) == ref.compress(G1, pts, n), info.name


def test_type_e_power_of_the_zero_gt_element_is_zero():
    """GT of type e is F_q^*, and the reference's F_q power (fp_pow_mpz, arith/montfp.c:379-396) leaves a
    zero base at 0 for every exponent, 0 and multiples of r included; k_e_gt_pow once wrote 1 there"""
    from pbc_b200.pairing import Pairing
    info = L.SetInfo("e")
    pr = Pairing(info.text)
    top = (1 << (8 * info.zlen)) - 1
    ks = [0, info.r, top // info.r * info.r, 1, info.r + 1, top]
    got = pr.gt_pow_zn(bytes(pr.gt_len * len(ks)), L.scalar_bytes(info, ks), len(ks))
    assert got == bytes(pr.gt_len * len(ks))
    one = (1).to_bytes(info.wb, "big")
    assert pr.gt_pow_zn(one + one, L.scalar_bytes(info, [0, info.r]), 2) == one + one


@pytest.mark.parametrize("name", ("d159", "d175", "d190", "d196", "d201", "a1"))
def test_first_argument_outside_g1_with_r_either_side_mod_4(name):
    """the Miller walk takes the signed digits of r - 1 where the curve has points outside E[r]
    (host_naf.hpp, miller_naf_digits): a walk over the digits of r evaluates f_{r+1,P} instead of the
    reference's f_{r-1,P} where r = 3 mod 4 (d190, d196), which agree only for r P = O"""
    from pbc_b200.pairing import Pairing
    assert os.path.exists(L.REF_LIB), L.ref_missing_message()
    info = L.SetInfo(name)
    pr = Pairing(info.text)
    n = 3 if REDUCED else 8
    with L.open_ref(name, 31) as ref:
        P = b"".join(L.off_subgroup_points(info, ref, _rnd(info, "outside"), n))
        Q = L.random_pairs(ref, n)[1]
        assert pr.apply(P, Q, n) == ref.pairing(P, Q, n)
        assert pr.pp_apply(P[:pr.g1_len], Q, n) == ref.pp_pairing(P[:pr.g1_len], Q, n)
        k = n // 2
        assert pr.prod_apply(P[:2 * k * pr.g1_len], Q[:2 * k * pr.g2_len], k, 2) == \
            ref.prod_pairing(P[:2 * k * pr.g1_len], Q[:2 * k * pr.g2_len], k, 2)

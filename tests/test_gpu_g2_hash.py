"""element_from_hash and element_from_bytes_compressed on G2 (pbc_b200_g2_from_hash, _device,
pbc_b200_g2_from_bytes_compressed; Pairing.g2_compress on the host) against the compiled reference at test
time and against tests/golden/g2_hash.json, for every shipped parameter set: every hash length around the
width of q, hash values with every number of halvings (both halves for type f), the reference-basis
variants of f and d159, decompression of random, non-canonical and y = 0 points and of every sign byte,
x with no point, pairings and BLS signatures in G2 built on the hashes, and batches that span several
blocks.  Types a and a1 (G2 = G1) give the bytes of the G1 calls; type e fails.
PBC_LIVE_REFERENCE_REDUCED=1 shrinks the batches (tests/test_g2_hash_on_cpu_sim.py)."""
import json
import os
import random

import pytest

from tests import live_reference as L
from tests import small_order_points as S

pytestmark = pytest.mark.gpu
REDUCED = bool(os.environ.get("PBC_LIVE_REFERENCE_REDUCED"))
EXT_DEGREE = {"f": 2, "d": 3, "g": 5}
BLOCK = 128                     # threads per block of the G2 kernels
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "g2_hash.json")


@pytest.fixture(scope="module", params=L.SETS, ids=["%s_set" % s for s in L.SETS])
def live(request):
    """(info, library handle, reference handle, oracle or None) of one set"""
    from pbc_b200.pairing import Pairing
    from oracle import pbc_oracle as O
    assert os.path.exists(L.REF_LIB), L.ref_missing_message()
    name = request.param
    info = L.SetInfo(name)
    orc = O.pairing_from_param(info.text) if info.type in EXT_DEGREE else None
    with L.open_ref(name, 2000 + L.SETS.index(name)) as ref:
        yield info, Pairing(info.text), ref, orc


def _rnd(info, salt):
    return random.Random("g2/%s/%s" % (info.name, salt))


def _lengths(info):
    wb = info.count
    return sorted({1, 2, 3, wb - 1, wb, wb + 1, 2 * wb, 2 * wb + 1, 70})


def _twist(pr):
    return pr.type in EXT_DEGREE


def _skip_e(info, pr):
    if info.type == "e":
        from pbc_b200.pairing import PairingError
        with pytest.raises(PairingError, match="type e"):
            pr.g2_from_hash(b"abc", 3, 1)
        with pytest.raises(PairingError, match="type e"):
            pr.g2_decompress(bytes(pr.g2_len // 2 + 1), 1)
        with pytest.raises(PairingError, match="type e"):
            pr.g2_compress(bytes(pr.g2_len), 1)
        pytest.skip("type e has no element_from_hash or compressed points (checked that it fails)")


def _torch_device_call(fn, out_len, data):
    from pbc_b200 import _lib
    if _lib.IS_SIMULATOR:
        return None
    import torch
    d = torch.frombuffer(bytearray(data), dtype=torch.uint8).cuda()
    out = torch.zeros(max(1, out_len), dtype=torch.uint8, device="cuda")
    fn(out.data_ptr(), d.data_ptr())
    torch.cuda.synchronize()
    return bytes(out.cpu().numpy().tobytes())[:out_len]


def _want_hash(info, pr, ref, data, length, n):
    """the reference's G2 hashes; for a and a1 (G2 = G1) the library's G1 call"""
    from oracle.ref import G2
    if _twist(pr):
        return ref.from_hash(G2, data, length, n)
    return pr.g1_from_hash(data, length, n)


def _check_hash(info, pr, ref, data, length, n, device=False):
    want = _want_hash(info, pr, ref, data, length, n)
    got = pr.g2_from_hash(data, length, n)
    w = pr.g2_len
    bad = [i for i in range(n) if got[i * w:(i + 1) * w] != want[i * w:(i + 1) * w]]
    assert not bad, (info.name, length, [data[i * length:(i + 1) * length].hex() for i in bad[:2]])
    if device:
        got = _torch_device_call(lambda o, d: pr.g2_from_hash_device(o, d, length, n), n * w, data)
        assert got in (want, None), (info.name, length, "device")


def test_hash_every_length(live):
    info, pr, ref, _ = live
    _skip_e(info, pr)
    rnd = _rnd(info, "len")
    per = 2
    for length in _lengths(info):
        data = bytes(rnd.getrandbits(8) for _ in range(per * length))
        _check_hash(info, pr, ref, data, length, per, device=length in (32, info.count) or length == 70)


def test_hash_values_and_halvings(live):
    """values 0, 1, q - 1, q, q + 1, all ones, and every number of halvings; type f in either half, with
    even and odd lengths (x0 takes len/2 bytes, x1 the rest)"""
    info, pr, ref, _ = live
    _skip_e(info, pr)
    rnd = _rnd(info, "val")
    vals = [d[:info.count] for _, d in L.hash_data_by_value(info, rnd)]
    vals += [d for _, d in L.hash_data_by_halvings(info, rnd, 1)]
    c = info.count
    if info.type == "f":
        other = [bytes(rnd.getrandbits(8) for _ in range(c + 1)) for _ in vals]
        for first in (True, False):
            even = b"".join((v + o[:c]) if first else (o[:c] + v) for v, o in zip(vals, other))
            _check_hash(info, pr, ref, even, 2 * c, len(vals))
            # odd length 2c + 1: x0 takes c bytes, x1 the c + 1 after them.  x1 = v || one byte reads as v:
            # pbc_mpz_from_hash fills its count = c byte buffer from the first c bytes of the data
            assert all(L.mpz_from_hash(info.q, v + o[c:c + 1]) == L.mpz_from_hash(info.q, v) for v, o in zip(vals, other))
            odd = b"".join((v + o) if first else (o[:c] + v + o[c:c + 1]) for v, o in zip(vals, other))
            _check_hash(info, pr, ref, odd, 2 * c + 1, len(vals))
    else:
        _check_hash(info, pr, ref, b"".join(vals), c, len(vals), device=not REDUCED)


@pytest.mark.parametrize("name", ("f", "d159"))
def test_reference_basis_variants(name):
    """b200_reference_basis 1 computes in the reference's basis: the same bytes"""
    from pbc_b200.pairing import Pairing
    from oracle.ref import G2
    info = L.SetInfo(name)
    pr, pr_ref = Pairing(info.text), Pairing(info.text + "\nb200_reference_basis 1\n")
    rnd = _rnd(info, "basis")
    n = 4 if REDUCED else 32
    with L.open_ref(name, 77) as ref:
        for length in (1, info.count + 1, 2 * info.count + 1):
            data = bytes(rnd.getrandbits(8) for _ in range(n * length))
            want = ref.from_hash(G2, data, length, n)
            assert pr.g2_from_hash(data, length, n) == want
            assert pr_ref.g2_from_hash(data, length, n) == want
        pts = ref.random(G2, n)
        comp = ref.compress(G2, pts, n)
        assert pr.g2_decompress(comp, n) == pts
        assert pr_ref.g2_decompress(comp, n) == pts
        assert pr_ref.g2_compress(pts, n) == comp


def _flip(comp, clen, to):
    return b"".join(comp[i:i + clen - 1] + bytes([to(comp[i + clen - 1])]) for i in range(0, len(comp), clen))


def test_decompression_and_compression(live):
    """random points, each sign byte (0, 1, 2, 255) and x + q, against the reference's own decompression"""
    info, pr, ref, _ = live
    from oracle.ref import G2
    _skip_e(info, pr)
    n = 4 if REDUCED else 48
    pts = ref.random(G2, n)
    comp = ref.compress(G2, pts, n)
    assert pr.g2_compress(pts, n) == comp, info.name
    assert pr.g2_decompress(comp, n) == pts, info.name
    clen = len(comp) // n
    for to in (lambda s: 1 - s, lambda s: 2 * s, lambda s: 255 * s, lambda s: 0):
        c2 = _flip(comp, clen, to)
        assert pr.g2_decompress(c2, n) == ref.decompress(G2, c2, n), info.name
    # coordinate 0 of x non-canonical (v + q), where the wire width has room
    nc = []
    for i in range(n):
        c = comp[i * clen:(i + 1) * clen]
        v = int.from_bytes(c[:info.wb], "big")
        if v + info.q < 1 << (8 * info.wb):
            nc.append(info.be(v + info.q) + c[info.wb:])
    if nc:
        data = b"".join(nc)
        assert pr.g2_decompress(data, len(nc)) == ref.decompress(G2, data, len(nc)), info.name


def _rhs(E, x):
    K = E.K
    return K.add(K.mul(K.add(K.sqr(x), E.a), x), E.b)


def _x_without_point(orc, size, rnd, n):
    """x in K whose x^3 + a'x + b' is not a square (checked here; never handed to the reference, whose
    polymod_sqrt does not return on a non-square)"""
    E, K, out = orc.Et, orc.Et.K, []
    while len(out) < n:
        x = S.rand_el(K, rnd)
        t = _rhs(E, x)
        if not K.eq(t, K.zero) and not K.eq(S.kpow(K, t, (size - 1) // 2), K.one):
            out.append(x)
    return out


def test_no_point_and_y_zero(live):
    """an x with no point gives zero bytes; a root of x^3 + a'x + b' gives (x, 0) for either sign byte"""
    info, pr, ref, orc = live
    _skip_e(info, pr)
    if not _twist(pr):
        pytest.skip("G2 = G1: test_gpu_group_ops.py covers G1")
    rnd = _rnd(info, "edge")
    size = info.q ** EXT_DEGREE[info.type]
    K = orc.Et.K
    xs = _x_without_point(orc, size, rnd, 2 if REDUCED else 6)
    data = b"".join(K.to_bytes(x) + bytes([i & 1]) for i, x in enumerate(xs))
    assert pr.g2_decompress(data, len(xs)) == bytes(pr.g2_len * len(xs)), info.name
    roots = S.two_torsion(orc.Et, size, rnd)
    for T in roots:
        for s in (0, 1):
            assert pr.g2_decompress(K.to_bytes(T[0]) + bytes([s]), 1) == orc.Et.to_bytes(T), (info.name, s)


def test_pairing_with_hashed_second_argument(live):
    """e(P, H2(m)) equals the reference's pairing of its own H2(m)"""
    info, pr, ref, _ = live
    from oracle.ref import G1, G2
    _skip_e(info, pr)
    n = 2 if REDUCED else 16
    rnd = _rnd(info, "pair")
    msgs = bytes(rnd.getrandbits(8) for _ in range(32 * n))
    P = ref.random(G1, n)
    H = pr.g2_from_hash(msgs, 32, n)
    assert pr.apply(P, H, n) == ref.pairing(P, ref.from_hash(G2, msgs, 32, n), n), info.name


def test_bls_signatures_in_g2(live):
    """BLS with short public keys: pk = sk g, sig = sk H2(m), e(g, sig) == e(pk, H2(m)); a forged key fails"""
    info, pr, ref, _ = live
    from oracle.ref import G1
    _skip_e(info, pr)
    n = 2 if REDUCED else 8
    rnd = _rnd(info, "bls")
    g = ref.random(G1, 1) * n
    sk = L.scalar_bytes(info, [rnd.randrange(1, info.r) for _ in range(n)])
    forged = L.scalar_bytes(info, [rnd.randrange(1, info.r) for _ in range(n)])
    msgs = bytes(rnd.getrandbits(8) for _ in range(32 * n))
    pk, pk_bad = pr.g1_pow_zn(g, sk, n), pr.g1_pow_zn(g, forged, n)
    H = pr.g2_from_hash(msgs, 32, n)
    sig = pr.g2_pow_zn(H, sk, n)
    assert pr.apply(g, sig, n) == pr.apply(pk, H, n), info.name
    lhs, bad = pr.apply(g, sig, n), pr.apply(pk_bad, H, n)
    w = pr.gt_len
    assert all(lhs[i * w:(i + 1) * w] != bad[i * w:(i + 1) * w] for i in range(n)), info.name


def test_batches_across_blocks(live):
    """hashes and decompressions over several blocks, with the special inputs at the block ends"""
    info, pr, ref, orc = live
    from oracle.ref import G2
    _skip_e(info, pr)
    rnd = _rnd(info, "batch")
    n = BLOCK + 2 if REDUCED else 3 * BLOCK + 5
    ends = [BLOCK - 1, BLOCK] + ([] if REDUCED else [2 * BLOCK - 1, 2 * BLOCK, 3 * BLOCK - 1, 3 * BLOCK, n - 1])
    c = info.count
    items = [bytes(rnd.getrandbits(8) for _ in range(c + 3)) for _ in range(n)]
    special = [d for _, d in L.hash_data_by_value(info, rnd)]
    for j, i in enumerate(ends):
        items[i] = special[j % len(special)]
    data = b"".join(items)
    _check_hash(info, pr, ref, data, c + 3, n)
    if not _twist(pr):
        return
    pts = ref.random(G2, n)
    comp = bytearray(ref.compress(G2, pts, n))
    clen, w = len(comp) // n, pr.g2_len
    want = bytearray(pts)
    size = info.q ** EXT_DEGREE[info.type]
    K = orc.Et.K
    edges = [(K.to_bytes(x), bytes(w)) for x in _x_without_point(orc, size, rnd, 2)]
    edges += [(K.to_bytes(T[0]), orc.Et.to_bytes(T)) for T in S.two_torsion(orc.Et, size, rnd)]
    for j, i in enumerate(ends):
        x, out = edges[j % len(edges)]
        comp[i * clen:(i + 1) * clen] = x + bytes([j & 1])
        want[i * w:(i + 1) * w] = out
    assert pr.g2_decompress(bytes(comp), n) == bytes(want), info.name


def test_golden_fixture(live):
    """tests/golden/g2_hash.json, made by tests/golden/make_g2_hash_golden.py from the reference"""
    info, pr, _, _ = live
    _skip_e(info, pr)
    g = json.load(open(GOLDEN))["sets"].get(info.name)
    if g is None:
        pytest.skip("no fixture entry for %s" % info.name)
    cat = lambda xs: b"".join(bytes.fromhex(x) for x in xs)
    from pbc_b200._lib import lib
    assert lib.pbc_b200_pairing_length_in_bytes_compressed_G2(pr.handle) == g["compressed_len"]
    for length, blk in g["hash"].items():
        assert pr.g2_from_hash(cat(blk["data"]), int(length), len(blk["data"])) == cat(blk["G2"]), (info.name, length)
    comp = g["compressed"]
    n = len(comp["G2"])
    assert pr.g2_compress(cat(comp["points"]), n) == cat(comp["G2"])
    assert pr.g2_decompress(cat(comp["G2"]), n) == cat(comp["points"])
    assert pr.g2_decompress(cat(comp["G2_flipped_sign"]), n) == cat(comp["points_flipped"])
    for p in g.get("y_zero", []):
        assert pr.g2_decompress(bytes.fromhex(p["compressed"]), 1) == bytes.fromhex(p["point"])

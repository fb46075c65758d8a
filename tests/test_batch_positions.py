"""The expected values of tests/test_gpu_batch_positions.py, checked without a GPU: they differ between
positions the kernels could confuse (so a kernel that reads its neighbour's data at one of their
strides fails), and the tables they come from agree with the oracle's pairing."""
import numpy as np
import pytest

from oracle import pbc_oracle as O
from tests import batch_positions as B


def _strides_below(n):
    return [s for s in B.STRIDES if s < n]


@pytest.mark.parametrize("name", B.NAMES)
def test_expected_outputs_differ_at_every_kernel_stride(name):
    fam = B.family(name)
    T = 132 * B.chains_per_sm(fam.kind)
    n = B.CHUNK + T + 1001
    _, _, want = B.pairs(fam, n)
    for s in _strides_below(n):
        assert B.differ_fraction(want, s) >= 0.99, ("apply", s)
    for k in (3, 16):
        n_out = B.CHUNK // k + 1001
        _, _, want = B.products(fam, k, n_out)
        for s in _strides_below(n_out):
            assert B.differ_fraction(want, s) >= 0.99, ("prod_apply", k, s)
    _, _, want = B.fixed_first(fam, 3, B.CHUNK + 1001)
    for s in _strides_below(B.CHUNK + 1001):
        assert B.differ_fraction(want, s) >= 0.99, ("pp_apply", s)
    n = 3 * T + 17
    u = 1 + np.arange(n, dtype=np.int64) % B.L1
    v, sign, _ = B.scalars(fam, n, B.chain_positions(n, T, chunk=n))
    for what, want in (("g1_pow_zn", B.expected_points(fam.P, u, v, sign)),
                       ("gt_pow_zn", B.expected_gt_powers(fam, u, v, sign))):
        for s in _strides_below(n):
            assert B.differ_fraction(want, s) >= 0.99, (what, s)


def test_type_a_products_of_16_differ_at_every_kernel_stride():
    fam = B.family("a")
    n_out = (1 << 16) + 3
    _, _, want = B.products(fam, 16, n_out)
    for s in _strides_below(n_out):
        assert B.differ_fraction(want, s) >= 0.99, s


@pytest.mark.parametrize("name", B.NAMES)
def test_tables_agree_with_the_oracle_pairing(name):
    """e0 is the reference output; e(uP0, wQ0) = e0^(uw) and e(-uP0, wQ0) = e0^(-uw) by the oracle's pairing (type e:
    the restatement tests/type_e_model.py) for a few (u, w); the scalars are congruent to what the layout says"""
    fam = B.family(name)
    E, Einv = fam.E.table(35), fam.Einv.table(35)
    assert bytes(E[1]) == fam.e0b
    if fam.kind == "e":
        from tests import type_e_model as M
        model = M.PairingE(fam.text, M.any_r(fam.text))
        pairing = model.pairing
    else:
        pairing = lambda P, Q: O.pairing_bytes(fam.oracle, P, Q)
    for u, w in ((2, 3), (5, 7)):
        assert pairing(bytes(fam.P.table(u)[u]), bytes(fam.Q.table(w)[w])) == bytes(E[u * w]), (u, w)
    assert pairing(bytes(fam.P.table(2, negate=True)[2]), bytes(fam.Q.table(3)[3])) == bytes(Einv[6])
    assert pairing(fam.badP, fam.Q0b) == fam.identity
    n = 40
    v, sign, raw = B.scalars(fam, n, (0, 9))
    ks = [int.from_bytes(bytes(row), "big") for row in raw]
    assert all(k % fam.r == (int(s) * int(x)) % fam.r for k, s, x in zip(ks, sign, v))
    assert ks[0] == 0 and ks[9] == fam.r


@pytest.mark.parametrize("name", [n for n in B.NAMES if n != "e"])
def test_oracle_hash_agrees_with_the_reference(name):
    """the oracle's element_from_hash, which gives the expected points of the hashing test, against the reference"""
    fam = B.family(name)
    blk = fam.g["hash"]["32"]
    P = O.g1_from_hash(fam.oracle, bytes.fromhex(blk["data"][0]))
    assert fam.oracle.G1.to_bytes(P) == bytes.fromhex(blk["G1"][0])


def test_chain_positions_cover_both_chunks():
    T = 132 * 256
    n = B.CHUNK + T + 1001
    pos = B.chain_positions(n, T)
    assert {0, B.CHUNK - 1, B.CHUNK, n - 1} <= set(pos)
    assert {1000, 1000 + T, B.CHUNK + 1000, B.CHUNK + 1000 + T} <= set(pos)
    assert {64 * 7, 64 * 7 + 63, 256 * 9, 256 * 9 + 255} <= set(pos)
    assert any(n - T <= p < n - 1 for p in pos) and any(B.CHUNK - T <= p < B.CHUNK - 1 for p in pos)

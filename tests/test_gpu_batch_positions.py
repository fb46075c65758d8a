"""Every position of large batches against exact values, with inputs that repeat at no stride the library
uses (tests/batch_positions.py builds them: position i pairs uP0 with wQ0, u = 1 + i mod 139,
w = 1 + i mod 137, and expects e0^(uw) from tables grown by repeated multiplication).

Tiled fixtures repeat with periods of 8 to 24, which divide the thread blocks, the pipeline chunks and
the batch-inversion chain stride T = SMs * 128 or 256: an output that took its neighbour's data at such
a stride would still be right.  Here it is not, so these tests see a batch inversion that multiplies by
the wrong element of its chain, a chunk that reads another chunk's inputs, a block that reads another
block's slots.  Invalid inputs and zero scalars sit where a chain is easiest to spoil: its first and
last elements, two consecutive elements, the ends of blocks and of chunks."""
import hashlib

import numpy as np
import pytest

from tests import batch_positions as B

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module", params=B.NAMES)
def case(request):
    import torch
    from pbc_b200.pairing import Pairing
    fam = B.family(request.param)
    pr = Pairing(fam.text)
    sms = torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count
    yield fam, pr, sms * B.chains_per_sm(fam.kind)
    pr.clear()


def _check(got, want, what):
    bad = B.mismatches(got, want)
    assert len(bad) == 0, "%s: %s" % (what, B.describe(bad, len(want)))


def _flat(a):
    return np.ascontiguousarray(a).reshape(-1)


def _cuda(a):
    import torch
    return torch.from_numpy(_flat(a).copy()).cuda()


def _empty(nbytes):
    import torch
    return torch.empty(max(1, nbytes), dtype=torch.uint8, device="cuda")


def _back(t, nbytes):
    import torch
    torch.cuda.synchronize()
    return t[:nbytes].cpu().numpy()


def _stream():
    import torch
    return torch.cuda.current_stream().cuda_stream


# ---- 1, 2: plain pairings, host pipeline (two chunks) and one device launch ----------------------------
def test_apply_every_position_across_chunks_and_chains(case):
    """n = 2^18 + T + 1001: the second chunk is longer than one inversion stride, so both chunks have chains of
    two or more elements; invalid inputs at the chain, block and chunk ends give 1, every other output is exact"""
    fam, pr, T = case
    n = B.CHUNK + T + 1001
    bad = B.chain_positions(n, T)
    in1, in2, want = B.pairs(fam, n, bad)
    _check(pr.apply(_flat(in1), _flat(in2), n), want, "apply")


def test_apply_device_every_position_in_one_launch(case):
    fam, pr, T = case
    n = B.CHUNK + T + 1001
    bad = B.chain_positions(n, T, chunk=n)
    in1, in2, want = B.pairs(fam, n, bad)
    out, d1, d2 = _empty(n * pr.gt_len), _cuda(in1), _cuda(in2)    # kept alive until the call has finished
    pr.apply_device(out.data_ptr(), d1.data_ptr(), d2.data_ptr(), n, _stream())
    _check(_back(out, n * pr.gt_len), want, "apply_device")


# ---- 3: products across the chunk boundary -----------------------------------------------------------------
@pytest.mark.parametrize("k", [3, 16])
def test_products_across_the_chunk_boundary(case, k):
    """2^18 / k + 1001 products of k: two chunks; one invalid input poisons exactly one output of each chunk"""
    fam, pr, T = case
    per = B.CHUNK // k
    n_out = per + 1001
    poison = (17, per + 5)
    in1, in2, want = B.products(fam, k, n_out, poison)
    _check(pr.prod_apply(_flat(in1), _flat(in2), k, n_out), want, "prod_apply k=%d" % k)


def test_type_a_products_on_the_default_shared_accumulator():
    """prod_apply_device, k = 16, 2^16 + 3 outputs, as bench.py's prod16 runs it.  A type a product shares one
    Miller accumulator between c pairs per thread, c the largest divisor of k not above the handle's setting
    (default 2), once the m = n_out * k pairs leave m / c >= 4 * SMs * 3 * 128 threads: here, on an H100,
    k_a_miller9_shared runs with c = 2"""
    import torch
    from pbc_b200.pairing import Pairing
    fam = B.family("a")
    sms = torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count
    k, n_out = 16, (1 << 16) + 3
    assert n_out * k // 2 >= 4 * sms * 3 * 128, "this device has too many SMs for the shared path at this size"
    pr = Pairing(fam.text)
    poison = (0, 4099, n_out - 1)
    in1, in2, want = B.products(fam, k, n_out, poison)
    out, d1, d2 = _empty(n_out * pr.gt_len), _cuda(in1), _cuda(in2)
    pr.prod_apply_device(out.data_ptr(), d1.data_ptr(), d2.data_ptr(), k, n_out, _stream())
    _check(_back(out, n_out * pr.gt_len), want, "prod_apply_device k=16 (shared accumulator)")
    pr.clear()


# ---- 4: fixed first argument ------------------------------------------------------------------------------
def test_fixed_first_argument_one_shot_and_handle(case):
    """P = 3 P0 against 2^18 + 1001 second arguments: e(3P0, wQ0) = e0^(3w); invalid second arguments give 1"""
    fam, pr, T = case
    n = B.CHUNK + 1001
    in1, in2, want = B.fixed_first(fam, 3, n)
    for i in B.chain_positions(n, T):
        in2[i] = np.frombuffer(fam.badQ, dtype=np.uint8)
        want[i] = np.frombuffer(fam.identity, dtype=np.uint8)
    _check(pr.pp_apply(_flat(in1), _flat(in2), n), want, "pp_apply")
    h = pr.pp_init(_flat(in1))
    try:
        _check(h.apply(_flat(in2), n), want, "pp_init handle")
    finally:
        h.clear()


# ---- 5: powers on G1, G2 and GT ----------------------------------------------------------------------------
@pytest.mark.parametrize("which", ["g1", "g2", "gt"])
def test_powers_every_position(case, which):
    """n = 3T + 17 powers: element u at position i, scalar v, r - v or v + r (v = 1 + i mod 137); the scalars 0 and r
    at the chain ends and at two consecutive elements of a chain.  Host buffers and device pointers.  The G2 fixtures
    of types f, d and g have a cofactor part, so their scalars are v and v + r only (both reduce to v)."""
    fam, pr, T = case
    n = 3 * T + 17
    u = 1 + np.arange(n, dtype=np.int64) % B.L1
    negative = which != "g2" or fam.q0_has_order_r
    v, sign, raw = B.scalars(fam, n, B.chain_positions(n, T, chunk=n), negative)
    if which == "gt":
        elems = fam.E.table(B.L1)[u]
        want = B.expected_gt_powers(fam, u, v, sign)
        host, device = pr.gt_pow_zn, pr.gt_pow_zn_device
    else:
        grp = fam.P if which == "g1" else fam.Q
        elems = grp.table(B.L1)[u]
        want = B.expected_points(grp, u, v, sign)
        host, device = (pr.g1_pow_zn, pr.g1_pow_zn_device) if which == "g1" else (pr.g2_pow_zn, pr.g2_pow_zn_device)
    L = elems.shape[1]
    _check(host(_flat(elems), _flat(raw), n), want, "%s_pow_zn" % which)
    out, d_elems, d_raw = _empty(n * L), _cuda(elems), _cuda(raw)
    device(out.data_ptr(), d_elems.data_ptr(), d_raw.data_ptr(), n, _stream())
    _check(_back(out, n * L), want, "%s_pow_zn_device" % which)


# ---- 6: decompression, GT product and comparison, co-DDH ------------------------------------------------
def test_decompress_every_position(case):
    fam, pr, T = case
    if fam.kind == "e":
        pytest.skip("type e has no element_from_bytes_compressed")
    n = T + 1001
    u = 1 + np.arange(n, dtype=np.int64) % B.L1
    want = fam.P.table(B.L1)[u]
    _check(pr.g1_decompress(_flat(fam.compress(want)), n), want, "g1_decompress")


def test_gt_mul_and_cmp_every_position(case):
    fam, pr, T = case
    n = T + 1001
    u, w = B.uw(n)
    E = fam.E.table(2 * B.L1)
    _check(pr.gt_mul(_flat(E[u]), _flat(E[w]), n), E[u + w], "gt_mul")
    i = np.arange(n)
    b = np.where(i % 11 < 4, u, u + w)                # equal at i = 0..3 mod 11
    want = (b != u).astype(np.uint8)[:, None]
    _check(pr.gt_cmp(_flat(E[u]), _flat(E[b]), n), want, "gt_cmp")


def test_is_almost_coddh_every_position(case):
    """(a, b, c, d) = (uP0, wP0, c, wQ0): e(a, d) = e0^(uw).  c = uQ0 (true), -uQ0 (true: the inverse is allowed)
    or (u + 1)Q0 (false), in a pattern of period 13"""
    fam, pr, T = case
    n = T + 1001
    u, w = B.uw(n)
    t = np.arange(n) % 13
    Pt, Qt, Qn = fam.P.table(B.L1 + 1), fam.Q.table(B.L1 + 1), fam.Q.table(B.L1 + 1, negate=True)
    c = np.where((t < 5)[:, None], Qt[u], np.where((t < 9)[:, None], Qn[u], Qt[u + 1]))
    want = (t < 9).astype(np.uint8)[:, None]
    got = pr.is_almost_coddh(_flat(Pt[u]), _flat(Pt[w]), _flat(c), _flat(fam.Q.table(B.L2)[w]), n)
    _check(got, want, "is_almost_coddh")


# ---- 7: hashing to G1 ----------------------------------------------------------------------------------
def test_g1_from_hash_every_position(case):
    """a prime period of distinct messages (139; 13 for a1, whose oracle cofactor multiplication is slow), each
    expected point computed once by the oracle, tiled past T"""
    from oracle import pbc_oracle as O
    fam, pr, T = case
    if not fam.has_hash:
        pytest.skip("type e has no element_from_hash")
    per = 13 if fam.kind == "a1" else B.L1
    msgs = [hashlib.sha256(b"position-%d" % j).digest() for j in range(per)]
    pts = np.frombuffer(b"".join(fam.oracle.G1.to_bytes(O.g1_from_hash(fam.oracle, m)) for m in msgs),
                        dtype=np.uint8).reshape(per, -1)
    data = np.frombuffer(b"".join(msgs), dtype=np.uint8).reshape(per, -1)
    n = T + 1001
    j = np.arange(n) % per
    _check(pr.g1_from_hash(_flat(data[j]), 32, n), pts[j], "g1_from_hash")


# ---- 8: two devices ------------------------------------------------------------------------------------------
def test_two_devices_every_position(case):
    """set_devices(2): each device takes ceil(n / 2) outputs and runs them through its own two-chunk pipeline"""
    import torch
    from pbc_b200.pairing import Pairing
    if torch.cuda.device_count() < 2:
        pytest.skip("one GPU visible: multi-device slicing needs two")
    fam, _, T = case
    pr = Pairing(fam.text)
    try:
        pr.set_devices(2)
        n = 2 * (B.CHUNK + 1001) + 1                  # slices of 2^18 + 1002 and 2^18 + 1000
        in1, in2, want = B.pairs(fam, n, B.chain_positions(n, T))
        _check(pr.apply(_flat(in1), _flat(in2), n), want, "apply on two devices")
        k = 3
        n_out = 2 * (B.CHUNK // k + 501) + 1
        in1, in2, want = B.products(fam, k, n_out, (17, n_out // 2 + 3, n_out - 1))
        _check(pr.prod_apply(_flat(in1), _flat(in2), k, n_out), want, "prod_apply on two devices")
        in1, in2, want = B.fixed_first(fam, 3, n)
        _check(pr.pp_apply(_flat(in1), _flat(in2), n), want, "pp_apply on two devices")
    finally:
        pr.clear()

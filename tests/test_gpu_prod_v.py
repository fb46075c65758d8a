"""Products of pairings with a pair count per output (Pairing.prod_apply_v, pbc_b200_prod_pairings_apply_v):
every output must be byte-identical to the uniform product (prod_apply with k = its length) of its
pairs, and to the compiled reference (oracle/_ref/libpbcref.so) wherever the reference divides by no
zero.  The segmented product multiplies runs of at most 16 values per pass (pbc_b200/csrc/prod_v.cuh);
the lengths below sit around the boundaries of one, two, three and four passes.  Pairs are drawn from a
pool of independent random pairs, reused at a stride (a prime) that matches no run length.
PBC_PROD_V_REDUCED=1 shrinks the batches, for the CPU simulator of the library (tests/test_prod_v_cpu.py), and
shrinks them further for the 34-limb types a1 and e, whose simulated Miller loops take 0.4 to 2 s each."""
import json
import os
import random

import pytest

from tests import live_reference as L
from tests.test_gpu_live_reference import _torch_device_call

pytestmark = pytest.mark.gpu
REDUCED = bool(os.environ.get("PBC_PROD_V_REDUCED"))
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
POOL = 13 if REDUCED else 97
TYPES = ("a", "a1", "e", "f", "d159", "g149", "d201")
with open(os.path.join(ROOT, "tests", "golden", "small_order.json")) as _f:
    SO = json.load(_f)


def _tiny(name):
    """the reduced batches of the simulator, at their smallest"""
    return REDUCED and name in ("a1", "e")


@pytest.fixture(scope="module")
def handles():
    """per set: (info, library handle, reference handle, pool of pairs); references cleared at the end"""
    import contextlib
    from pbc_b200.pairing import Pairing
    assert os.path.exists(L.REF_LIB), L.ref_missing_message()
    cache, stack = {}, contextlib.ExitStack()

    def get(name):
        if name not in cache:
            info = L.SetInfo(name)
            ref = stack.enter_context(L.open_ref(name, 7000 + L.SETS.index(name)))
            pr = Pairing(info.text)
            P, Q = L.random_pairs(ref, POOL)
            cache[name] = (info, pr, ref, L.split(P, pr.g1_len), L.split(Q, pr.g2_len))
        return cache[name]
    with stack:
        yield get


def _identity(pr):
    wb = pr.g1_len // 2
    return b"\0" * (wb - 1) + b"\1" + bytes(pr.gt_len - wb)


def _offsets(lengths):
    off = [0]
    for n in lengths:
        off.append(off[-1] + n)
    return off


def _pool_pairs(P, Q, m, start=0):
    return [(P[(start + j) % len(P)], Q[(start + j) % len(Q)]) for j in range(m)]


def _grouped(pr, pairs, off):
    """the outputs of one uniform prod_apply call per distinct length, scattered back to order"""
    segs = [pairs[off[i]:off[i + 1]] for i in range(len(off) - 1)]
    out = [None] * len(segs)
    for k in sorted({len(s) for s in segs}):
        idx = [i for i, s in enumerate(segs) if len(s) == k]
        P = b"".join(p for i in idx for p, _ in segs[i])
        Q = b"".join(q for i in idx for _, q in segs[i])
        got = L.split(pr.prod_apply(P, Q, k, len(idx)), pr.gt_len)
        for i, g in zip(idx, got):
            out[i] = g
    return out


def _ragged(pr, pairs, off):
    return L.split(pr.prod_apply_v(b"".join(p for p, _ in pairs), b"".join(q for _, q in pairs), off), pr.gt_len)


def _off_curve(info, P):
    cs = info.coords(P)
    return info.from_coords([cs[0], (cs[1] + 1) % info.q])


def _negate(info, P):
    x, y = info.coords(P)
    return info.from_coords([x, (info.q - y) % info.q])


# ---- against the compiled reference, every shipped set --------------------------------------------

def _specials(info, pr, ref, rnd):
    """(P, Q, small-order) pairs the uniform tests use: non-canonical coordinates, first arguments
    outside G1 (not type e), second arguments outside G2 where G2 is E(F_q), off-curve first arguments,
    and the small-order points of tests/golden/small_order.json"""
    P, Q = L.split(L.random_pairs(ref, 8)[0], pr.g1_len), L.split(L.random_pairs(ref, 8)[1], pr.g2_len)
    out = []
    for i in range(3):
        out.append((L.non_canonical(info, P[i]) or P[i], L.non_canonical(info, Q[i]) or Q[i], False))
    off = L.off_subgroup_points(info, ref, rnd, 2)
    if off and info.type != "e":
        out.append((off[0], Q[3], False))
    if off and info.type in ("a", "a1", "e"):
        out.append((P[4], off[1], False))
    out.append((_off_curve(info, P[5]), Q[5], False))
    ent = SO["sets"].get(info.name, {})
    if info.type != "e":
        out += [(bytes.fromhex(p["P"]), Q[6], True) for p in ent.get("g1", {}).get("points", [])[:2]]
    if info.type in ("a", "e"):
        out += [(P[7], bytes.fromhex(p["P"]), True) for p in ent.get("g1", {}).get("points", [])[:2]]
    elif info.type != "a1":
        out += [(P[7], bytes.fromhex(p["P"]), True) for p in ent.get("g2", {}).get("points", [])[:2]]
    return out


@pytest.mark.parametrize("name", L.SETS, ids=["%s_set" % s for s in L.SETS])
def test_random_lengths_with_special_inputs_against_the_reference(handles, name):
    info, pr, ref, P, Q = handles(name)
    rnd = random.Random("prod_v/%s" % name)
    lengths = [rnd.randint(1, 5 if REDUCED else 40) for _ in range((3 if _tiny(name) else 6) if REDUCED else 24)]
    off = _offsets(lengths)
    pairs = _pool_pairs(P, Q, off[-1], rnd.randrange(POOL))
    small = set()
    for s, (p, q, so) in enumerate(_specials(info, pr, ref, rnd)):
        seg = (2 * s + 1) % len(lengths)
        j = off[seg] + rnd.randrange(lengths[seg])
        pairs[j] = (p, q)
        if so:
            small.add(seg)
    got = _ragged(pr, pairs, off)
    uni = _grouped(pr, pairs, off)
    for i in range(len(lengths)):
        seg = pairs[off[i]:off[i + 1]]
        if i in small:             # where the reference may divide by zero, the uniform product's value
            want = uni[i]
        else:
            want = ref.prod_pairing(b"".join(p for p, _ in seg), b"".join(q for _, q in seg), len(seg), 1)
        assert got[i] == want, (name, i, lengths[i])
        assert got[i] == uni[i], (name, i, lengths[i])


# ---- pass structure -------------------------------------------------------------------------------

LENGTHS = [1, 2, 3, 15, 16, 17, 31, 32, 33, 257] if REDUCED else \
    (list(range(1, 41)) + [255, 256, 257, 1023, 1024, 1025, 4095, 4096, 4097])


@pytest.mark.parametrize("name", TYPES)
def test_lengths_around_every_pass_boundary_in_one_call(handles, name):
    info, pr, ref, P, Q = handles(name)
    lengths = [1, 2, 17] if _tiny(name) else list(LENGTHS)
    random.Random(name).shuffle(lengths)
    off = _offsets(lengths)
    pairs = _pool_pairs(P, Q, off[-1])
    got = _ragged(pr, pairs, off)
    assert got == _grouped(pr, pairs, off), name
    for i, n in enumerate(lengths):
        if n == 1:
            p, q = pairs[off[i]]
            assert got[i] == pr.apply(p, q, 1), name


@pytest.mark.parametrize("name", TYPES)
def test_bad_input_turns_only_its_own_product_into_one(handles, name):
    """segment i of S segments of length S carries an O or off-curve first argument at position i:
    half of them per call, so that every segment is checked bad and clean"""
    info, pr, ref, P, Q = handles(name)
    S = (3 if _tiny(name) else 17) if REDUCED else 40
    off = _offsets([S] * S)
    clean = _pool_pairs(P, Q, S * S)
    uni = _grouped(pr, clean, off)
    for parity in (0, 1):
        pairs = list(clean)
        for i in range(parity, S, 2):
            p, q = pairs[off[i] + i]
            pairs[off[i] + i] = (bytes(len(p)) if i % 4 < 2 else _off_curve(info, p), q)
        got = _ragged(pr, pairs, off)
        for i in range(S):
            assert got[i] == (_identity(pr) if i % 2 == parity else uni[i]), (name, parity, i)
        assert got[1 - parity] != _identity(pr)


# ---- scale --------------------------------------------------------------------------------------

@pytest.mark.parametrize("name", TYPES)
def test_many_random_lengths_equal_grouped_uniform_calls(handles, name):
    info, pr, ref, P, Q = handles(name)
    rnd = random.Random("scale/" + name)
    n_out, top = ((4, 4) if _tiny(name) else (24, 40)) if REDUCED else (1 << 14, 64)
    off = _offsets([rnd.randint(1, top) for _ in range(n_out)])
    pairs = _pool_pairs(P, Q, off[-1], 5)
    assert _ragged(pr, pairs, off) == _grouped(pr, pairs, off), name


@pytest.mark.parametrize("name", ("a", "f", "d159", "g149"))
def test_one_long_product_of_cancelling_pairs(handles, name):
    """(P_j, Q_j), (-P_j, Q_j) over 2^18 pairs: the GT identity; one unmatched pair more: its pairing"""
    info, pr, ref, P, Q = handles(name)
    m = 1 << (8 if REDUCED else 18)
    half = _pool_pairs(P, Q, m // 2)
    neg = {p: _negate(info, p) for p in set(P)}
    pairs = [x for p, q in half for x in ((p, q), (neg[p], q))]
    assert _ragged(pr, pairs, [0, m]) == [_identity(pr)], name
    extra = (P[3], Q[4])
    assert _ragged(pr, pairs + [extra], [0, m + 1]) == [pr.apply(extra[0], extra[1], 1)], name


@pytest.mark.skipif(REDUCED, reason="sized for the GPU")
@pytest.mark.parametrize("name", ("a", "f"))
def test_host_chunks_of_whole_outputs(handles, name):
    """host batches whose pair count crosses the library's chunk (2^18 pairs), among them one output
    longer than a chunk"""
    info, pr, ref, P, Q = handles(name)
    lengths = [1 + (i * 7) % 64 for i in range(9000)]
    lengths.insert(4500, (1 << 18) + 5)
    off = _offsets(lengths)
    assert off[-1] > 2 * (1 << 18)
    pairs = _pool_pairs(P, Q, off[-1], 11)
    assert _ragged(pr, pairs, off) == _grouped(pr, pairs, off), name


# ---- device path, streams, devices --------------------------------------------------------------------

@pytest.mark.parametrize("name", TYPES)
def test_device_form_equals_host_form(handles, name):
    from pbc_b200 import _lib
    if _lib.IS_SIMULATOR:
        pytest.skip("device buffers")
    info, pr, ref, P, Q = handles(name)
    rnd = random.Random("device/" + name)
    off = _offsets([rnd.randint(1, 40) for _ in range(6 if REDUCED else 300)])
    pairs = _pool_pairs(P, Q, off[-1], 2)
    Pb, Qb = b"".join(p for p, _ in pairs), b"".join(q for _, q in pairs)
    n_out = len(off) - 1
    host = pr.prod_apply_v(Pb, Qb, off)
    dev = _torch_device_call(lambda o, a, b: pr.prod_apply_v_device(o, a, b, off), n_out * pr.gt_len, Pb, Qb)
    assert dev in (host, None), name


def test_two_streams_share_one_handle(handles):
    from pbc_b200 import _lib
    if _lib.IS_SIMULATOR:
        pytest.skip("device buffers")
    import numpy as np
    import torch
    info, pr, ref, P, Q = handles("f")
    calls = []
    for seed in (1, 2):
        rnd = random.Random("streams/%d" % seed)
        off = _offsets([rnd.randint(1, 70) for _ in range(2000)])
        pairs = _pool_pairs(P, Q, off[-1], seed)
        Pb, Qb = b"".join(p for p, _ in pairs), b"".join(q for _, q in pairs)
        calls.append((off, pr.prod_apply_v(Pb, Qb, off), Pb, Qb))
    streams = [torch.cuda.Stream() for _ in calls]
    bufs = []
    for (off, _, Pb, Qb), s in zip(calls, streams):
        a = torch.frombuffer(bytearray(Pb), dtype=torch.uint8).cuda()
        b = torch.frombuffer(bytearray(Qb), dtype=torch.uint8).cuda()
        o = torch.zeros((len(off) - 1) * pr.gt_len, dtype=torch.uint8, device="cuda")
        bufs.append((a, b, o))
    torch.cuda.synchronize()
    for rep in range(3):
        for (off, _, _, _), (a, b, o), s in zip(calls, bufs, streams):
            pr.prod_apply_v_device(o.data_ptr(), a.data_ptr(), b.data_ptr(), np.array(off), s.cuda_stream)
    torch.cuda.synchronize()
    for (off, want, _, _), (_, _, o) in zip(calls, bufs):
        assert bytes(o.cpu().numpy().tobytes()) == want


def test_two_devices_equal_one():
    from pbc_b200 import _lib
    if _lib.IS_SIMULATOR:
        pytest.skip("one simulated device")
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("one GPU visible")
    from pbc_b200.pairing import Pairing
    info = L.SetInfo("f")
    with L.open_ref("f", 7100) as ref:
        Pp, Qp = L.random_pairs(ref, POOL)
    one, two = Pairing(info.text), Pairing(info.text)
    two.set_devices(2)
    rnd = random.Random("devices")
    off = _offsets([rnd.randint(1, 64) for _ in range(3000)] + [5000])
    pairs = _pool_pairs(L.split(Pp, one.g1_len), L.split(Qp, one.g2_len), off[-1])
    Pb, Qb = b"".join(p for p, _ in pairs), b"".join(q for _, q in pairs)
    assert two.prod_apply_v(Pb, Qb, off) == one.prod_apply_v(Pb, Qb, off)

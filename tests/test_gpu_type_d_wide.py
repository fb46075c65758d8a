"""Type D (MNT, k = 6) parameter sets with 160- to 255-bit q -- the eight-limb instance of the type D
kernels -- byte for byte against the reference fixtures tests/golden/d_wide_*.json (written by
tests/golden/make_d_wide_golden.py from the compiled reference)."""
import json
import os

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NAMES = ("d175", "d190", "d196", "d201", "d224")

pytestmark = pytest.mark.gpu


def _fix(name):
    with open(os.path.join(ROOT, "tests", "golden", "d_wide_%s.json" % name)) as f:
        return json.load(f)


def _cat(xs):
    return b"".join(bytes.fromhex(x) for x in xs)


@pytest.fixture(scope="module", params=NAMES)
def case(request):
    from pbc_b200.pairing import Pairing
    g = _fix(request.param)
    pr = Pairing(g["param_text"])
    yield g, pr


def _identity(pr):
    wb = pr.g1_len // 2
    return b"\0" * (wb - 1) + b"\1" + b"\0" * (pr.gt_len - wb)


def test_lengths(case):
    g, pr = case
    L = g["lengths"]
    assert (pr.g1_len, pr.g2_len, pr.gt_len, pr.zr_len) == (L["g1"], L["g2"], L["gt"], L["zr"])
    assert pr.type == "d"


def test_pairing(case):
    g, pr = case
    P, Q, E = g["pairing"]["P"], g["pairing"]["Q"], g["pairing"]["e"]
    assert pr.apply(_cat(P), _cat(Q), len(P)) == _cat(E)


def test_prod(case):
    g, pr = case
    k = g["prod"]["k"]
    n = len(g["prod"]["e"])
    assert pr.prod_apply(_cat(g["prod"]["P"]), _cat(g["prod"]["Q"]), k, n) == _cat(g["prod"]["e"])


def test_pp_one_shot_and_handle(case):
    g, pr = case
    P = bytes.fromhex(g["pp"]["P"])
    Q = g["pairing"]["Q"][:4]
    assert pr.pp_apply(P, _cat(Q), 4) == _cat(g["pp"]["e"])
    h = pr.pp_init(P)
    try:
        assert h.apply(_cat(Q), 4) == _cat(g["pp"]["e"])
        assert h.apply(_cat(Q[1:3]), 2) == _cat(g["pp"]["e"][1:3])
    finally:
        h.clear()


def test_group_powers(case):
    g, pr = case
    a = _cat(g["pow"]["a"])
    assert pr.g1_pow_zn(_cat(g["pairing"]["P"][:4]), a, 4) == _cat(g["pow"]["Pa"])
    assert pr.g2_pow_zn(_cat(g["pairing"]["Q"][:4]), a, 4) == _cat(g["pow"]["Qa"])
    assert pr.gt_pow_zn(_cat(g["pairing"]["e"][:4]), a, 4) == _cat(g["pow"]["ea"])
    # bilinearity through the library itself
    assert pr.apply(_cat(g["pow"]["Pa"]), _cat(g["pairing"]["Q"][:4]), 4) == _cat(g["pow"]["e_Pa_Q"])
    assert pr.apply(_cat(g["pow"]["Pa"]), _cat(g["pow"]["Qa"]), 4) == _cat(g["pow"]["e_Pa_Qa"])


def test_gt_ops_and_coddh(case):
    g, pr = case
    E = g["pairing"]["e"]
    assert pr.gt_mul(_cat(E[:4]), _cat(E[4:8]), 4) == _cat(g["gt_mul"]["e0_e4"])
    assert pr.gt_cmp(_cat(E[:2]), _cat([E[0], E[0]]), 2) == b"\0\1"
    P, Q, Pa, Qa = g["pairing"]["P"], g["pairing"]["Q"], g["pow"]["Pa"], g["pow"]["Qa"]
    # e(P, Q^a) == e(P^a, Q): co-DDH holds; with Q^a replaced by another Q it does not
    assert pr.is_almost_coddh(_cat(P[:2]), _cat(Pa[:2]), _cat(Q[:2]), _cat([Qa[0], Q[1]]), 2) == b"\1\0"


def test_hash_and_decompress(case):
    g, pr = case
    for ln, h in g["hash"].items():
        data = _cat(h["data"])
        assert pr.g1_from_hash(data, int(ln), len(h["data"])) == _cat(h["G1"]), ln
    c = g["compressed"]
    n = len(c["G1"])
    assert pr.g1_decompress(_cat(c["G1"]), n) == _cat(g["pairing"]["P"][:n])
    flipped = b"".join(bytes.fromhex(x)[:-1] + bytes([bytes.fromhex(x)[-1] ^ 1]) for x in c["G1"])
    assert pr.g1_decompress(flipped, n) == _cat(c["G1_flipped_sign"])


def test_offcurve_and_infinity(case):
    g, pr = case
    off = g["offcurve"]
    Q0, P0 = bytes.fromhex(g["pairing"]["Q"][0]), bytes.fromhex(g["pairing"]["P"][0])
    one = _identity(pr)
    assert bytes.fromhex(off["identity"]) == one
    assert pr.apply(bytes.fromhex(off["badP"]), Q0, 1) == one
    assert pr.apply(P0, bytes.fromhex(off["badQ"]), 1) == one
    O1, O2 = b"\0" * pr.g1_len, b"\0" * pr.g2_len
    assert pr.apply(O1 + P0, Q0 + O2, 2) == one + one
    # an O inside a product makes it 1
    k = g["prod"]["k"]
    PP, QQ = list(g["prod"]["P"][:k]), list(g["prod"]["Q"][:k])
    PP[1] = O1.hex()
    assert pr.prod_apply(_cat(PP), _cat(QQ), k, 1) == one


def test_device_pointers(case):
    torch = pytest.importorskip("torch")
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    g, pr = case
    P, Q, E = g["pairing"]["P"], g["pairing"]["Q"], g["pairing"]["e"]
    n = len(P)
    dP = torch.frombuffer(bytearray(_cat(P)), dtype=torch.uint8).cuda()
    dQ = torch.frombuffer(bytearray(_cat(Q)), dtype=torch.uint8).cuda()
    out = torch.empty(n * pr.gt_len, dtype=torch.uint8, device="cuda")
    pr.apply_device(out.data_ptr(), dP.data_ptr(), dQ.data_ptr(), n, torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    assert bytes(out.cpu().numpy().tobytes()) == _cat(E)


@pytest.mark.parametrize("name", ("d201", "d224"))
def test_large_batch_crosses_the_chunk_boundary(name):
    """2^18 + 37 pairings: two pipeline chunks on two streams, the fixture inputs repeated"""
    from pbc_b200.pairing import Pairing
    g = _fix(name)
    pr = Pairing(g["param_text"])
    P, Q, E = g["pairing"]["P"], g["pairing"]["Q"], g["pairing"]["e"]
    n = (1 << 18) + 37
    reps = (n + len(P) - 1) // len(P)
    idx = [i % len(P) for i in range(n)]
    got = pr.apply((_cat(P) * reps)[:n * pr.g1_len], (_cat(Q) * reps)[:n * pr.g2_len], n)
    L = pr.gt_len
    for i in (0, 1, (1 << 18) - 1, 1 << 18, n - 1):
        assert got[i * L:(i + 1) * L] == bytes.fromhex(E[idx[i]]), i
    assert got == b"".join(bytes.fromhex(E[i]) for i in idx)

"""Type E (k = 1, 34-limb field) on the GPU, byte for byte against the reference fixtures
tests/golden/e*.json (tests/golden/make_e_golden.py) and against the Python restatement
tests/type_e_model.py run with the library's own R."""
import json
import os
import random

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NAMES = ("e", "e_s510", "e_s513")

pytestmark = pytest.mark.gpu


def _fix(name):
    with open(os.path.join(ROOT, "tests", "golden", name + ".json")) as f:
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
    return b"\0" * (pr.gt_len - 1) + b"\1"


def test_lengths(case):
    g, pr = case
    L = g["lengths"]
    assert (pr.g1_len, pr.g2_len, pr.gt_len, pr.zr_len) == (L["g1"], L["g2"], L["gt"], L["zr"])
    assert pr.type == "e"


def test_field_ops_against_integers(case):
    g, pr = case
    from tests.type_e_model import parse_param
    q = parse_param(g["param_text"])["q"]
    wb = pr.gt_len
    rnd = random.Random(7)
    n = 64
    xs = [rnd.randrange(q) for _ in range(n)]
    ys = [rnd.randrange(1, q) for _ in range(n)]
    A = b"".join(x.to_bytes(wb, "big") for x in xs)
    B = b"".join(y.to_bytes(wb, "big") for y in ys)
    want = {0: lambda x, y: x * y % q, 1: lambda x, y: (x + y) % q, 2: lambda x, y: (x - y) % q,
            3: lambda x, y: pow(x, q - 2, q), 5: lambda x, y: -x % q, 6: lambda x, y: x * x % q}
    for op, f in want.items():
        got = pr.fp_op(op, A, B, n)
        assert got == b"".join(f(x, y).to_bytes(wb, "big") for x, y in zip(xs, ys)), op


def test_pairing(case):
    g, pr = case
    P, Q, E = g["pairing"]["P"], g["pairing"]["Q"], g["pairing"]["e"]
    assert pr.apply(_cat(P), _cat(Q), len(P)) == _cat(E)


def test_every_pair_across_blocks_against_the_restatement(case):
    """every (P_i, Q_j) of the fixture, repeated past several 128-thread blocks, against the Python
    restatement with the library's R"""
    g, pr = case
    from tests.type_e_model import PairingE
    wb = pr.gt_len
    R = pr.derived_constant("R", wb)
    model = PairingE(g["param_text"], tuple(R))
    Ps, Qs = g["pairing"]["P"][:4], g["pairing"]["Q"][:4]
    pairs = [(i, j) for i in range(4) for j in range(4)]
    want = {(i, j): model.pairing(bytes.fromhex(Ps[i]), bytes.fromhex(Qs[j])) for i, j in pairs}
    n = 3 * 128 + 5
    idx = [pairs[(7 * t) % len(pairs)] for t in range(n)]
    got = pr.apply(b"".join(bytes.fromhex(Ps[i]) for i, _ in idx), b"".join(bytes.fromhex(Qs[j]) for _, j in idx), n)
    assert got == b"".join(want[p] for p in idx)
    assert want[(0, 0)] == bytes.fromhex(g["pairing"]["e"][0])


def test_prod(case):
    g, pr = case
    k = g["prod"]["k"]
    n = len(g["prod"]["e"])
    assert pr.prod_apply(_cat(g["prod"]["P"]), _cat(g["prod"]["Q"]), k, n) == _cat(g["prod"]["e"])
    # k = 1 is the plain pairing
    assert pr.prod_apply(_cat(g["pairing"]["P"][:5]), _cat(g["pairing"]["Q"][:5]), 1, 5) == _cat(g["pairing"]["e"][:5])


def test_pp_one_shot_and_handle(case):
    g, pr = case
    P = bytes.fromhex(g["pp"]["P"])
    Q = g["pairing"]["Q"][:4]
    assert pr.pp_apply(P, _cat(Q), 4) == _cat(g["pp"]["e"])
    h = pr.pp_init(P)
    try:
        assert h.apply(_cat(Q), 4) == _cat(g["pp"]["e"])
        assert h.apply(_cat(Q[1:3]), 2) == _cat(g["pp"]["e"][1:3])
        assert h.apply(bytes.fromhex(g["offcurve"]["badQ"]) + _cat(Q[:1]), 2) == _identity(pr) + _cat(g["pp"]["e"][:1])
    finally:
        h.clear()
    bad = bytes.fromhex(g["offcurve"]["badP"])
    assert pr.pp_apply(bad, _cat(Q[:2]), 2) == _identity(pr) * 2
    h = pr.pp_init(bad)
    try:
        assert h.apply(_cat(Q[:2]), 2) == _identity(pr) * 2
    finally:
        h.clear()


def test_group_powers_and_bilinearity(case):
    g, pr = case
    a = _cat(g["pow"]["a"])
    assert pr.g1_pow_zn(_cat(g["pairing"]["P"][:4]), a, 4) == _cat(g["pow"]["Pa"])
    assert pr.g2_pow_zn(_cat(g["pairing"]["Q"][:4]), a, 4) == _cat(g["pow"]["Qa"])
    assert pr.gt_pow_zn(_cat(g["pairing"]["e"][:4]), a, 4) == _cat(g["pow"]["ea"])
    # e(aP, Q) = e(P, aQ) = e(P, Q)^a, through the library itself
    assert pr.apply(_cat(g["pow"]["Pa"]), _cat(g["pairing"]["Q"][:4]), 4) == _cat(g["pow"]["ea"])
    assert pr.apply(_cat(g["pairing"]["P"][:4]), _cat(g["pow"]["Qa"]), 4) == _cat(g["pow"]["ea"])
    assert pr.apply(_cat(g["pow"]["Pa"]), _cat(g["pow"]["Qa"]), 4) == _cat(g["pow"]["e_Pa_Qa"])


def test_gt_ops_and_coddh(case):
    g, pr = case
    E = g["pairing"]["e"]
    assert pr.gt_mul(_cat(E[:4]), _cat(E[4:8]), 4) == _cat(g["gt_mul"]["e0_e4"])
    assert pr.gt_cmp(_cat(E[:2]), _cat([E[0], E[0]]), 2) == b"\0\1"
    P, Q, Pa, Qa = g["pairing"]["P"], g["pairing"]["Q"], g["pow"]["Pa"], g["pow"]["Qa"]
    assert pr.is_almost_coddh(_cat(P[:2]), _cat(Pa[:2]), _cat(Q[:2]), _cat([Qa[0], Q[1]]), 2) == b"\1\0"


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
    k = g["prod"]["k"]
    PP, QQ = list(g["prod"]["P"][:2 * k]), list(g["prod"]["Q"][:2 * k])
    PP[1] = O1.hex()
    assert pr.prod_apply(_cat(PP), _cat(QQ), k, 2) == one + bytes.fromhex(g["prod"]["e"][1])


def test_hash_and_decompress_fail_cleanly(case):
    from pbc_b200.pairing import PairingError
    g, pr = case
    with pytest.raises(PairingError, match="type e"):
        pr.g1_from_hash(b"abc" * 4, 12, 1)
    with pytest.raises(PairingError, match="type e"):
        pr.g1_decompress(b"\0" * (pr.g1_len // 2 + 1), 1)


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
    stream = torch.cuda.current_stream().cuda_stream
    pr.apply_device(out.data_ptr(), dP.data_ptr(), dQ.data_ptr(), n, stream)
    torch.cuda.synchronize()
    assert bytes(out.cpu().numpy().tobytes()) == _cat(E)
    a = torch.frombuffer(bytearray(_cat(g["pow"]["a"])), dtype=torch.uint8).cuda()
    o1 = torch.empty(4 * pr.g1_len, dtype=torch.uint8, device="cuda")
    pr.g1_pow_zn_device(o1.data_ptr(), dP.data_ptr(), a.data_ptr(), 4, stream)
    torch.cuda.synchronize()
    assert bytes(o1.cpu().numpy().tobytes()) == _cat(g["pow"]["Pa"])


def test_type_e_and_a1_alternate_on_one_device():
    from pbc_b200.pairing import Pairing
    from pbc_b200.params import PARAMS
    ge, ga = _fix("e"), _fix("a1")
    pe, pa = Pairing(ge["param_text"]), Pairing(PARAMS["a1"])
    for _ in range(2):
        assert pe.apply(_cat(ge["pairing"]["P"][:2]), _cat(ge["pairing"]["Q"][:2]), 2) == _cat(ge["pairing"]["e"][:2])
        assert pa.apply(_cat(ga["pairing"]["P"][:2]), _cat(ga["pairing"]["Q"][:2]), 2) == _cat(ga["pairing"]["e"][:2])
    pe.clear()
    pa.clear()

"""Type E (k = 1) without a GPU: the Python restatement of the kernels' formulas
(tests/type_e_model.py) with an R of its own against the compiled reference's fixtures
tests/golden/e*.json, the host ABI of the library (lengths, type letter, the derived R, the
rejected parameter variants), and the type E kernels themselves on the CPU simulator of the library
(tests/host/make_host_sim.py: inline PTX through the PTX interpreter) against the fixtures."""
import json
import os
import shutil
import subprocess
import sys

import pytest

from tests import type_e_model as M

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NAMES = ("e", "e_s510", "e_s513")


def _fix(name):
    with open(os.path.join(ROOT, "tests", "golden", name + ".json")) as f:
        return json.load(f)


def _cat(xs):
    return b"".join(bytes.fromhex(x) for x in xs)


def test_fixtures_cover_every_sign_branch():
    signs = {(M.parse_param(_fix(n)["param_text"])["sign1"], M.parse_param(_fix(n)["param_text"])["sign0"]) for n in NAMES}
    assert signs == {(1, 1), (1, -1), (-1, -1)}
    assert M.parse_param(_fix("e_s513")["param_text"])["q"].bit_length() == 513


@pytest.mark.parametrize("name", NAMES)
def test_restatement_with_its_own_r_equals_the_reference(name):
    g = _fix(name)
    text = g["param_text"]
    pr = M.PairingE(text, M.any_r(text, start=7))
    n = 4 if name == "e" else 12
    assert pr.pairing_batch(_cat(g["pairing"]["P"][:n]), _cat(g["pairing"]["Q"][:n]), n) == _cat(g["pairing"]["e"][:n])
    # pp: the same P against the first four Q
    P0 = bytes.fromhex(g["pp"]["P"])
    assert b"".join(pr.pairing(P0, bytes.fromhex(x)) for x in g["pairing"]["Q"][:2]) == _cat(g["pp"]["e"][:2])
    # products: the reference multiplies in GT
    k = g["prod"]["k"]
    acc = 1
    for i in range(k):
        acc = acc * int.from_bytes(pr.pairing(bytes.fromhex(g["prod"]["P"][i]), bytes.fromhex(g["prod"]["Q"][i])), "big") % pr.q
    assert pr.gt_bytes(acc) == bytes.fromhex(g["prod"]["e"][0])
    # off-curve inputs
    one = pr.gt_bytes(1)
    assert pr.pairing(bytes.fromhex(g["offcurve"]["badP"]), bytes.fromhex(g["pairing"]["Q"][0])) == one


@pytest.fixture(scope="module")
def built():
    import __graft_entry__ as ge
    ge.build()
    from pbc_b200 import pairing
    return pairing


@pytest.mark.parametrize("name", NAMES)
def test_host_abi_lengths_and_r(built, name):
    g = _fix(name)
    p = built.Pairing(g["param_text"])
    L = g["lengths"]
    assert (p.type, p.g1_len, p.g2_len, p.gt_len, p.zr_len) == ("e", L["g1"], L["g2"], L["gt"], L["zr"])
    prm = M.parse_param(g["param_text"])
    q, r, a, b = prm["q"], prm["r"], prm["a"] % prm["q"], prm["b"] % prm["q"]
    x, y = p.derived_constant("R", p.gt_len)
    assert (y * y - (x * x * x + a * x + b)) % q == 0
    assert M.mul(r, (x, y), a, q) is not None                   # r R != O: R lies outside E[r]
    assert p.derived_constant("phikonr", p.gt_len) == [(q - 1) // r]
    p.clear()


def _variant(text, **kw):
    prm = M.parse_param(text)
    prm.update(kw)
    return "type e\n" + "".join("%s %s\n" % (k, prm[k]) for k in ("q", "r", "h", "a", "b", "exp2", "exp1", "sign1", "sign0"))


def test_q_width_bound(built):
    """q below 2^1087 (the 34-limb field): a 1087-bit q passes the width check (and fails on r here),
    a 1088-bit q does not"""
    text = _fix("e")["param_text"]
    with pytest.raises(built.PairingError, match="r does not divide q - 1"):
        built.Pairing(_variant(text, q=2 ** 1086 + 3))
    with pytest.raises(built.PairingError, match=r"below 2\^1087 \(got 1088 bits\)"):
        built.Pairing(_variant(text, q=2 ** 1087 + 3))


@pytest.mark.parametrize("change,message", [
    ({"sign0": -1}, "r != 2^exp2"),
    ({"exp1": 134}, "r != 2^exp2"),
    ({"sign1": 2}, "sign1 and sign0"),
    ({"sign0": 0}, "sign1 and sign0"),
])
def test_rejects_malformed_parameters(built, change, message):
    text = _variant(_fix("e")["param_text"], **change)
    with pytest.raises(built.PairingError, match=message.replace("^", r"\^")):
        built.Pairing(text)


def test_rejects_r_not_dividing_q_minus_1(built):
    prm = M.parse_param(_fix("e_s510")["param_text"])
    text = _variant(_fix("e_s510")["param_text"], q=prm["q"] + 2)
    with pytest.raises(built.PairingError, match="r does not divide q - 1"):
        built.Pairing(text)


def test_rejects_missing_key(built):
    text = "\n".join(l for l in _fix("e")["param_text"].splitlines() if not l.startswith("h "))
    with pytest.raises(built.PairingError, match="missing param"):
        built.Pairing(text)


# ---- the kernels on the CPU simulator against the reference fixtures -----------------------------

@pytest.fixture(scope="module")
def sim(tmp_path_factory):
    if not shutil.which("g++"):
        pytest.skip("no g++")
    tmp = tmp_path_factory.mktemp("esim")
    cpp, so = str(tmp / "host_sim.cpp"), str(tmp / "libpbc_b200_sim.so")
    subprocess.check_call([sys.executable, os.path.join(ROOT, "tests", "host", "make_host_sim.py"), cpp])
    subprocess.check_call(["g++", "-O1", "-std=c++17", "-shared", "-fPIC", "-Wno-unknown-pragmas", "-pthread",
                           "-o", so, cpp])
    return so


def _run(so, code, arg):
    env = dict(os.environ)
    env["PBC_B200_LIB"] = so
    env["PYTHONPATH"] = ROOT + os.pathsep + env.get("PYTHONPATH", "")
    out = subprocess.run([sys.executable, "-c", code, arg], env=env, capture_output=True, text=True, timeout=1800)
    assert out.returncode == 0, out.stderr[-3000:]
    return json.loads(out.stdout.strip().splitlines()[-1])


_ENTRY_CHECK = r'''
import json, sys
from pbc_b200.pairing import Pairing
cat = lambda xs: b"".join(bytes.fromhex(x) for x in xs)
g = json.load(open(sys.argv[1]))
pr = Pairing(g["param_text"])
ok = {}
if g["param"] == "e":
    # one pairing on the 1020-bit set
    ok["pairing"] = pr.apply(cat(g["pairing"]["P"][:1]), cat(g["pairing"]["Q"][:1]), 1) == cat(g["pairing"]["e"][:1])
else:
    ok["pairing"] = pr.apply(cat(g["pairing"]["P"][:3]), cat(g["pairing"]["Q"][:3]), 3) == cat(g["pairing"]["e"][:3])
    k = g["prod"]["k"]
    ok["prod"] = pr.prod_apply(cat(g["prod"]["P"][:k]), cat(g["prod"]["Q"][:k]), k, 1) == cat(g["prod"]["e"][:1])
    ok["pp_one_shot"] = pr.pp_apply(bytes.fromhex(g["pp"]["P"]), cat(g["pairing"]["Q"][:2]), 2) == cat(g["pp"]["e"][:2])
    h = pr.pp_init(bytes.fromhex(g["pp"]["P"]))
    ok["pp_handle"] = h.apply(cat(g["pairing"]["Q"][:2]), 2) == cat(g["pp"]["e"][:2])
    h.clear()
    ok["g1_pow"] = pr.g1_pow_zn(cat(g["pairing"]["P"][:1]), cat(g["pow"]["a"][:1]), 1) == cat(g["pow"]["Pa"][:1])
    ok["gt_pow"] = pr.gt_pow_zn(cat(g["pairing"]["e"][:1]), cat(g["pow"]["a"][:1]), 1) == cat(g["pow"]["ea"][:1])
    ok["gt_mul"] = pr.gt_mul(cat(g["pairing"]["e"][:1]), cat(g["pairing"]["e"][4:5]), 1) == cat(g["gt_mul"]["e0_e4"][:1])
    one = bytes(pr.gt_len - 1) + bytes([1])
    ok["offcurve"] = pr.apply(bytes.fromhex(g["offcurve"]["badP"]), cat(g["pairing"]["Q"][:1]), 1) == one
print(json.dumps(ok))
'''


@pytest.mark.parametrize("name", NAMES)
def test_entry_points_on_the_simulator(sim, name):
    ok = _run(sim, _ENTRY_CHECK, os.path.join(ROOT, "tests", "golden", name + ".json"))
    assert ok and all(ok.values()), ok

"""Type D with 160- to 255-bit q (the eight-limb instance, engine_d_wide.cu) without a GPU: the host ABI
(lengths, constants, the limits of the q range) and the kernels themselves on the CPU simulator of the
library with the eight-limb instance (tests/host/make_host_sim_d_wide.py: inline PTX through the PTX
interpreter), against Python integers and the reference fixtures tests/golden/d_wide_*.json."""
import json
import os
import shutil
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HOST = os.path.join(ROOT, "tests", "host")
NAMES = ("d175", "d190", "d196", "d201", "d224")


def _fix(name):
    with open(os.path.join(ROOT, "tests", "golden", "d_wide_%s.json" % name)) as f:
        return json.load(f)


def _params(text):
    tab = {}
    toks = [t for line in text.splitlines() for t in line.split("#")[0].split()]
    for k, v in zip(toks[::2], toks[1::2]):
        tab[k] = v
    return tab


# ---- host ABI (the product library or, without one, the simulator below) ------------------------

@pytest.fixture(scope="module")
def sim(tmp_path_factory):
    if not shutil.which("g++"):
        pytest.skip("no g++")
    tmp = tmp_path_factory.mktemp("dwsim")
    cpp, so = str(tmp / "host_sim.cpp"), str(tmp / "libpbc_b200_sim.so")
    subprocess.check_call([sys.executable, os.path.join(HOST, "make_host_sim_d_wide.py"), cpp])
    subprocess.check_call(["g++", "-O1", "-std=c++17", "-shared", "-fPIC", "-Wno-unknown-pragmas", "-pthread",
                           "-o", so, cpp])
    return so


def _run(so, code):
    env = dict(os.environ)
    env["PBC_B200_LIB"] = so
    env["PYTHONPATH"] = ROOT + os.pathsep + env.get("PYTHONPATH", "")
    out = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, timeout=1800)
    assert out.returncode == 0, out.stderr[-3000:]
    return json.loads(out.stdout.strip().splitlines()[-1])


_HOST_CHECK = r'''
import json, sys
from pbc_b200.pairing import Pairing, PairingError
g = json.load(open(sys.argv[1]))
res = {}
pr = Pairing(g["param_text"])
res["lengths"] = [pr.g1_len, pr.g2_len, pr.gt_len, pr.zr_len]
res["type"] = pr.type
names = ["phikonr", "xpwr3", "xpwr4", "xpowq", "xpowq2", "nqrinv"]
res["derived"] = {n: pr.derived_constant_n(n, 64, 3) for n in names}
try:
    res["basis_cubic"] = pr.derived_constant_n("basis_cubic", 64, 3)
except PairingError:
    res["basis_cubic"] = None
print(json.dumps(res))
'''


def _poly_mulmod(a, b, c, q):
    """a b mod x^3 + c2 x^2 + c1 x + c0 over F_q (coefficient lists, low first)"""
    d = [0] * 5
    for i in range(3):
        for j in range(3):
            d[i + j] = (d[i + j] + a[i] * b[j]) % q
    for k in (4, 3):
        t = d[k]
        d[k] = 0
        for i in range(3):
            d[k - 3 + i] = (d[k - 3 + i] - t * c[i]) % q
    return d[:3]


def _poly_pow(a, e, c, q):
    r = [1, 0, 0]
    while e:
        if e & 1:
            r = _poly_mulmod(r, a, c, q)
        a = _poly_mulmod(a, a, c, q)
        e >>= 1
    return r


@pytest.mark.parametrize("name", NAMES)
def test_host_abi_accepts_the_wide_sets(sim, name):
    g = _fix(name)
    t = _params(g["param_text"])
    q, r, nqr = int(t["q"]), int(t["r"]), int(t["nqr"])
    c = [int(t["coeff0"]) % q, int(t["coeff1"]) % q, int(t["coeff2"]) % q]
    res = _run(sim, _HOST_CHECK.replace("sys.argv[1]", repr(os.path.join(ROOT, "tests", "golden", "d_wide_%s.json" % name))))
    wb = (q.bit_length() + 7) // 8
    assert res["lengths"] == [2 * wb, 6 * wb, 6 * wb, (r.bit_length() + 7) // 8]
    L = g["lengths"]
    assert res["lengths"] == [L["g1"], L["g2"], L["gt"], L["zr"]]
    assert res["type"] == "d"
    D = res["derived"]
    assert D["phikonr"] == [(q * q - q + 1) // r] and (q * q - q + 1) % r == 0
    assert D["nqrinv"] == [pow(nqr, q - 2, q)]
    x = [0, 1, 0]
    assert D["xpwr3"] == _poly_pow(x, 3, c, q)
    assert D["xpwr4"] == _poly_pow(x, 4, c, q)
    xq = _poly_pow(x, q, c, q)
    assert D["xpowq"] == xq
    assert D["xpowq2"] == _poly_mulmod(xq, xq, c, q)
    # the internal cubic basis exists exactly where q = 2 mod 3 (d175, d190, d201 here; not d196, d224)
    assert (res["basis_cubic"] is not None) == (q % 3 == 2)
    if res["basis_cubic"] is not None:
        s0, lam, pc = res["basis_cubic"]
        assert s0 == c[2] * pow(3, q - 2, q) % q
        # x = lam w - s with w^3 + p w + 1 = 0: substitute w = (x + s) / lam into the cubic
        li = pow(lam, q - 2, q)
        w = [s0 * li % q, li, 0]
        w3 = _poly_mulmod(_poly_mulmod(w, w, c, q), w, c, q)
        assert [(w3[i] + pc * w[i] + (1 if i == 0 else 0)) % q for i in range(3)] == [0, 0, 0]


_RANGE_CHECK = r'''
import json, sys
from pbc_b200.pairing import Pairing, PairingError
text = sys.stdin.read()
try:
    Pairing(text)
    print(json.dumps("ok"))
except PairingError as e:
    print(json.dumps(str(e)))
'''


def _with_q(text, q):
    t = _params(text)
    return text.replace("q %s" % t["q"], "q %d" % q)


def _run_stdin(so, code, text):
    env = dict(os.environ)
    env["PBC_B200_LIB"] = so
    env["PYTHONPATH"] = ROOT + os.pathsep + env.get("PYTHONPATH", "")
    out = subprocess.run([sys.executable, "-c", code], input=text, env=env, capture_output=True, text=True, timeout=600)
    assert out.returncode == 0, out.stderr[-3000:]
    return json.loads(out.stdout.strip().splitlines()[-1])


def test_q_range_limits(sim):
    """q < 2^255 is the bound of the eight-limb code (engine.cu, next to init_type_d): a 255-bit q passes
    the width check, a 256-bit q and a 152-bit q do not"""
    text = _fix("d224")["param_text"]
    # d224's r does not divide q^2 - q + 1 for this q: the width check lets it through, the later checks refuse it
    msg = _run_stdin(sim, _RANGE_CHECK, _with_q(text, (1 << 254) + 3))
    assert "r does not divide" in msg, msg
    msg = _run_stdin(sim, _RANGE_CHECK, _with_q(text, (1 << 255) + 1))
    assert "160..255" in msg, msg
    msg = _run_stdin(sim, _RANGE_CHECK, _with_q(text, (1 << 151) + 1))
    assert "153..159" in msg, msg


# ---- the eight-limb field on the PTX interpreter, against Python integers -----------------------

_FP_CHECK = r'''
import json, random, sys
from pbc_b200.pairing import Pairing
g = json.load(open(sys.argv[1]))
pr = Pairing(g["param_text"])
q = int([l.split()[1] for l in g["param_text"].splitlines() if l.startswith("q ")][0])
wb = pr.g1_len // 2
rnd = random.Random(7)
xs = [rnd.randrange(q) for _ in range(12)] + [0, 1, q - 1, (1 << (8 * wb)) - 1 - q]
ys = [rnd.randrange(q) for _ in range(len(xs))]
enc = lambda v: b"".join(x.to_bytes(wb, "big") for x in v)
dec = lambda b: [int.from_bytes(b[i * wb:(i + 1) * wb], "big") for i in range(len(b) // wb)]
res = {}
for op in (0, 6, 9, 3, 1, 2, 4, 5):
    res[str(op)] = dec(pr.fp_op(op, enc(xs), enc(ys), len(xs)))
sq = [x * x % q for x in xs[:8]] + [rnd.randrange(q) for _ in range(8)]
res["8"] = dec(pr.fp_op(8, enc(sq), enc(sq), len(sq)))
print(json.dumps({"xs": xs, "ys": ys, "sq": sq, "q": q, "res": res}))
'''


@pytest.mark.parametrize("name", ("d175", "d190", "d224", "d201"))
def test_eight_limb_field_on_the_ptx_interpreter(sim, name):
    out = _run(sim, _FP_CHECK.replace("sys.argv[1]", repr(os.path.join(ROOT, "tests", "golden", "d_wide_%s.json" % name))))
    q, xs, ys, R = out["q"], out["xs"], out["ys"], out["res"]
    xs = [x % q for x in xs]                       # the wire reader reduces mod q, as the reference does
    assert R["0"] == [x * y % q for x, y in zip(xs, ys)]
    assert R["9"] == R["0"]                        # lazy double-width product + reduction
    assert R["6"] == [x * x % q for x in xs]
    assert R["3"] == [pow(x, q - 2, q) for x in xs]
    assert R["1"] == [(x + y) % q for x, y in zip(xs, ys)]
    assert R["2"] == [(x - y) % q for x, y in zip(xs, ys)]
    assert R["4"] == [x * pow(2, q - 2, q) % q for x in xs]
    assert R["5"] == [(-x) % q for x in xs]
    if q % 8 == 1:                                 # Tonelli-Shanks (d175, d190, d224: s = 4, 10, 4)
        for a, y in zip(out["sq"], R["8"]):
            if pow(a, (q - 1) // 2, q) in (0, 1):
                assert y * y % q == a
            else:
                assert y == 0


# ---- the kernels on the simulator against the reference fixtures -------------------------------

_ENTRY_CHECK = r'''
import json, sys
from pbc_b200.pairing import Pairing
cat = lambda xs: b"".join(bytes.fromhex(x) for x in xs)
g = json.load(open(sys.argv[1]))
pr = Pairing(g["param_text"])
ok = {}
ok["pairing"] = pr.apply(cat(g["pairing"]["P"][:3]), cat(g["pairing"]["Q"][:3]), 3) == cat(g["pairing"]["e"][:3])
k = g["prod"]["k"]
ok["prod"] = pr.prod_apply(cat(g["prod"]["P"][:k]), cat(g["prod"]["Q"][:k]), k, 1) == cat(g["prod"]["e"][:1])
h = pr.pp_init(bytes.fromhex(g["pp"]["P"]))
ok["pp_handle"] = h.apply(cat(g["pairing"]["Q"][:2]), 2) == cat(g["pp"]["e"][:2])
h.clear()
ok["hash"] = pr.g1_from_hash(cat(g["hash"]["32"]["data"][:2]), 32, 2) == cat(g["hash"]["32"]["G1"][:2])
ok["decompress"] = pr.g1_decompress(cat(g["compressed"]["G1"][:2]), 2) == cat(g["pairing"]["P"][:2])
ok["g2_pow"] = pr.g2_pow_zn(cat(g["pairing"]["Q"][:1]), cat(g["pow"]["a"][:1]), 1) == cat(g["pow"]["Qa"][:1])
ok["gt_pow"] = pr.gt_pow_zn(cat(g["pairing"]["e"][:1]), cat(g["pow"]["a"][:1]), 1) == cat(g["pow"]["ea"][:1])
print(json.dumps(ok))
'''


@pytest.mark.parametrize("name", NAMES)
def test_entry_points_on_the_simulator(sim, name):
    ok = _run(sim, _ENTRY_CHECK.replace("sys.argv[1]", repr(os.path.join(ROOT, "tests", "golden", "d_wide_%s.json" % name))))
    assert all(ok.values()), ok


def test_small_order_powers_on_the_simulator(sim):
    """the wide type D cases of tests/test_gpu_small_order_powers.py (G1 and G2 powers of points of
    small order, against the reference fixtures and the oracle), unchanged, on the eight-limb simulator"""
    env = dict(os.environ)
    env["PBC_B200_LIB"] = sim
    env["PYTHONPATH"] = ROOT + os.pathsep + env.get("PYTHONPATH", "")
    cmd = [sys.executable, "-m", "pytest", "-q", "-m", "gpu", "-p", "no:cacheprovider", "-k", "d_wide",
           os.path.join(ROOT, "tests", "test_gpu_small_order_powers.py")]
    out = subprocess.run(cmd, env=env, capture_output=True, text=True, timeout=1800, cwd=ROOT)
    assert out.returncode == 0, out.stdout[-3000:]
    tail = out.stdout.strip().splitlines()[-1]
    assert int(tail.split(" passed")[0].split()[-1]) >= 8, tail


def test_montgomery_extremes_on_the_simulator(sim):
    """the wide type D cases of tests/test_gpu_montgomery_extremes.py (field ops, square roots and the F_q^3 /
    F_q^6 tower on operands extreme in the Montgomery domain, both bases), unchanged, on the eight-limb
    simulator"""
    env = dict(os.environ)
    env["PBC_B200_LIB"] = sim
    env["PYTHONPATH"] = ROOT + os.pathsep + env.get("PYTHONPATH", "")
    cmd = [sys.executable, "-m", "pytest", "-q", "-m", "gpu", "-p", "no:cacheprovider", "-k", "d_wide",
           os.path.join(ROOT, "tests", "test_gpu_montgomery_extremes.py")]
    out = subprocess.run(cmd, env=env, capture_output=True, text=True, timeout=1800, cwd=ROOT)
    assert out.returncode == 0, out.stdout[-3000:]
    tail = out.stdout.strip().splitlines()[-1]
    assert int(tail.split(" passed")[0].split()[-1]) >= 18, tail

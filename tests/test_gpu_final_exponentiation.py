"""The final stages of types A, A1 and E -- k_batch_invert, then k_a_finalexp (the Lucas ladder over h),
k_a1_finalexp (a_lucas_final over l) or k_e_finalexp (the width-4 window over (q - 1)/r) -- on chosen
inputs, through pbc_b200_tower_op op 3: the same launches every pairing of these types ends in.

A Miller value is pseudo-random, so the pairing tests only ever feed these stages pseudo-random values.
Here the inputs are the ones a ladder or a window goes wrong on: elements of F_q^* and i F_q^* (N f0 f1 = 0,
the kernels' shortcut to 1), trace 0 (f = c (1 +- i)), torus elements of small order (the ladder's
P = trace of f^(q-1) then takes the values -1, 0 and 1, and V_k passes through 0 and +-2), r-th powers
(-> 1) and elements of order r (-> not 1), coordinates at Montgomery-domain extremes, and zero, which has
the documented value (include/pbc_b200.h).  Type e takes the numerator v and the denominator vd apart,
and b = NULL (vd = 1).  Wire coordinates at or above q are reduced mod q, as element_from_bytes does.

Expected values are plain Python integers: f^((q^2 - 1)/r) in F_q[i] (a), f^((p - 1) l) (a1),
(v / vd)^((q - 1)/r) in F_q (e); on a few random elements also the oracle's tateexp.  The batch-inversion
test runs one batch per family a little over three chains long (thread t of k_batch_invert owns elements
t, t + T, t + 2T, ..., T = multiprocessors x 256 or 128), with shortcut elements at chain heads and tails.

PBC_FINAL_EXP_REDUCED=1 shrinks the cases for the CPU simulator of the library
(tests/test_kernels_on_cpu_sim.py runs it, with PBC_SIM_SMS lowering the simulator's multiprocessor
count so that the chains are several elements long there too)."""
import functools
import os
import random

import pytest

from oracle import pbc_oracle as O
from tests.batch_positions import chains_per_sm
from tests.test_gpu_montgomery_extremes import FAMILY_LIMBS, LIMBS, Dom, _core, _param_text, targets

pytestmark = pytest.mark.gpu
REDUCED = bool(os.environ.get("PBC_FINAL_EXP_REDUCED"))
SETS = ("a", "a1", "a1_small", "e", "e_s510", "e_s513")
POOL = 61            # distinct non-shortcut elements of the chain batch: a prime, so no stride of 2^k 3^j 11 repeats it


def _sms():
    """multiprocessors of the device the library runs on (the simulator: PBC_SIM_SMS, default 132)"""
    import torch
    if torch.cuda.is_available():           # the library launches on the current device (engine.cu cur_sms)
        return torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count
    return int(os.environ.get("PBC_SIM_SMS", "132"))


class Fam:
    """one parameter set: the field, the exponent of its final stage, and the F_q^2 / F_q arithmetic"""

    def __init__(self, name):
        from pbc_b200.pairing import Pairing
        self.name = name
        self.text = _param_text(name)
        prm = O.parse_param(self.text)
        self.kind = prm["type"]
        self.pr = Pairing(self.text)
        if self.kind == "a1":
            self.q, self.r, self.cof = prm["p"], prm["n"], prm["l"]
            self.exp = (self.q - 1) * self.cof
        else:
            self.q, self.r, self.cof = prm["q"], prm["r"], prm["h"]
            self.exp = (self.q * self.q - 1) // self.r if self.kind == "a" else (self.q - 1) // self.r
        self.k = 1 if self.kind == "e" else 2
        self.wb = self.pr.gt_len // self.k
        self.dom = Dom(self.q, LIMBS[FAMILY_LIMBS[name]])

    # F_q[i], i^2 = -1
    def mul(self, x, y):
        q = self.q
        return ((x[0] * y[0] - x[1] * y[1]) % q, (x[0] * y[1] + x[1] * y[0]) % q)

    def pow(self, x, e):
        acc = (1, 0)
        while e:
            if e & 1:
                acc = self.mul(acc, x)
            x, e = self.mul(x, x), e >> 1
        return acc

    def rand2(self, rnd):
        return (rnd.randrange(1, self.q), rnd.randrange(1, self.q))

    def want(self, x):
        """the documented value of the final stage: x = (f0, f1) for a / a1, (v, vd) for e"""
        q = self.q
        x = tuple(c % q for c in x)       # wire values are reduced mod q, as element_from_bytes does
        if self.kind == "e":
            v, vd = x
            if vd % q == 0:
                return (1,)
            return (pow(v * pow(vd, q - 2, q) % q, self.exp, q),)
        if x[0] * x[1] % q == 0:
            return (1, 0)                 # N f0 f1 = 0: the shortcut (f = 0 included)
        return self.pow(x, self.exp)

    def enc(self, vals):
        return b"".join(v.to_bytes(self.wb, "big") for v in vals)

    def run(self, items):
        """the final stage on items (a, a1: (f0, f1); e: (v, vd)); the outputs as tuples of coordinates"""
        if self.kind == "e":
            a = self.enc(v for v, _ in items)
            b = self.enc(vd for _, vd in items)
        else:
            a = b"".join(self.enc(x) for x in items)
            b = None
        out = self.pr.tower_op(3, a, b, len(items))
        L, w = self.pr.gt_len, self.wb
        return [tuple(int.from_bytes(out[i * L + c * w:i * L + (c + 1) * w], "big") for c in range(self.k))
                for i in range(len(items))]


@functools.lru_cache(maxsize=None)
def fam(name):
    return Fam(name)


def _check(F, labelled):
    """run every (label, item) in one batch and name the classes that differ"""
    got = F.run([x for _, x in labelled])
    bad = [(lab, [hex(c) for c in x], [hex(c) for c in g]) for (lab, x), g in zip(labelled, got) if g != F.want(x)]
    assert not bad, "%s: %d of %d wrong; first (class, input, got): %s" % (F.name, len(bad), len(labelled), bad[:3])


def _exact_order(F, m, rnd, scale=False):
    """an element of F_q[i] of order exactly m on the norm-1 torus (m | q + 1), times c in F_q^* if scale"""
    q = F.q
    primes = [p for p in range(2, m + 1) if m % p == 0 and all(p % d for d in range(2, p))]
    while True:
        x = F.pow(F.rand2(rnd), (q * q - 1) // m)
        if all(F.pow(x, m // p) != (1, 0) for p in primes):
            break
    assert F.pow(x, m) == (1, 0)
    if scale:
        c = rnd.randrange(2, q)
        x = (x[0] * c % q, x[1] * c % q)
    return x


def _small_orders(F):
    """orders m | q + 1 the torus classes use: 3, 4, 6, 8, 12 for type a; the divisors of l for type a1"""
    if F.kind == "a":
        ms = [3, 4, 6, 8, 12]
        assert all((F.q + 1) % m == 0 for m in ms) and F.cof % 12 == 0
        return ms
    return [d for d in range(2, F.cof + 1) if F.cof % d == 0]


def _extremes(F, rnd):
    """coordinates whose Montgomery forms are the internal extremes (targets), f0 = +-f1 at extremes too"""
    T = targets(F.q, F.dom.N)
    C = _core(T, 12 if REDUCED else 24)
    W = [F.dom.wire(t) for t in C]
    out = [(a, b) for a in W[:8] for b in W[:8]] if not REDUCED else [(a, b) for a in W[:4] for b in W[:4]]
    out += [(a, rnd.choice(W)) for a in W]
    out += [(w, w) for w in W] + [(w, -w % F.q) for w in W]
    return out


def _golden_outputs(F):
    import json
    fn = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", F.name + ".json")
    with open(fn) as f:
        es = json.load(f)["pairing"]["e"]
    return [tuple(int.from_bytes(bytes.fromhex(e)[c * F.wb:(c + 1) * F.wb], "big") for c in range(F.k)) for e in es]


def _classes_k2(F, rnd):
    """(label, (f0, f1)) of every class, types a and a1"""
    q = F.q
    nr = 2 if REDUCED else 6
    L = []
    named = [1, q - 1, 2, q - 2] + [F.dom.wire(t) for t in targets(q, F.dom.N)[1:8]]
    for c in named + [rnd.randrange(1, q) for _ in range(nr)]:
        L += [("subfield F_q^*", (c, 0)), ("subfield i F_q^*", (0, c))]
    L.append(("zero", (0, 0)))
    for c in [1, q - 1, 2] + [rnd.randrange(1, q) for _ in range(nr)]:
        L += [("trace 0: c (1 + i)", (c, c)), ("trace 0: c (1 - i)", (c, -c % q))]
    for m in _small_orders(F):
        for s in range(1 if REDUCED else 2):
            L += [("order %d" % m, _exact_order(F, m, rnd)), ("order %d times c" % m, _exact_order(F, m, rnd, True))]
    for _ in range(nr):
        L.append(("r-th power", F.pow(F.rand2(rnd), F.r)))
        L.append(("order-r part", F.pow(F.rand2(rnd), (q * q - 1) // F.r)))
    L += [("Montgomery extremes", x) for x in _extremes(F, rnd)]
    L += [("random", F.rand2(rnd)) for _ in range(nr)]
    L += [("pairing output", x) for x in _golden_outputs(F)[:2 if REDUCED else None]]
    return L


def _classes_e(F, rnd):
    """(label, (v, vd)) of every class, type e"""
    q = F.q
    nr = 2 if REDUCED else 6
    rv = lambda: rnd.randrange(1, q)
    L = [("v = 1", (1, 1)), ("v = -1", (q - 1, 1)), ("v = 1, vd = -1", (1, q - 1)), ("v = -1, vd = -1", (q - 1, q - 1))]
    e = F.exp
    assert e % 2 == 0
    small = [m for m in range(2, 200) if e % m == 0][:4 if REDUCED else 12]
    for m in small:
        while True:
            x = pow(rv(), (q - 1) // m, q)
            if all(pow(x, m // p, q) != 1 for p in range(2, m + 1) if m % p == 0 and all(p % d for d in range(2, p))):
                break
        L += [("order %d" % m, (x, 1)), ("order %d over random vd" % m, (x * (c := rv()) % q, c))]
    for _ in range(nr):
        L.append(("r-th root of unity", (pow(rv(), (q - 1) // F.r, q), 1)))
        L.append(("r-th power", (pow(rv(), F.r, q), 1)))
        L.append(("r-th power over r-th power", (pow(rv(), F.r, q), pow(rv(), F.r, q))))
    L += [("v = 0", (0, 1)), ("v = 0, random vd", (0, rv())), ("vd = 0", (1, 0)), ("vd = 0, random v", (rv(), 0)),
          ("v = vd = 0", (0, 0))]
    for _ in range(nr):
        c = rv()
        L.append(("vd = v", (c, c)))
    T = targets(q, F.dom.N)
    W = [F.dom.wire(t) for t in _core(T, 12 if REDUCED else 24)]
    L += [("Montgomery extremes in v", (w, 1)) for w in W] + [("Montgomery extremes in vd", (1, w)) for w in W]
    L += [("Montgomery extremes in v and vd", (a, b)) for a in W[:8] for b in W[:8]]
    L += [("random", (rv(), rv())) for _ in range(nr)]
    for x in _golden_outputs(F)[:2 if REDUCED else None]:
        L += [("pairing output", (x[0], 1)), ("pairing output over random vd", (x[0], rv()))]
    return L


@pytest.mark.parametrize("name", SETS)
def test_final_stage_on_chosen_inputs(name):
    F = fam(name)
    rnd = random.Random("final-" + name)
    labelled = _classes_e(F, rnd) if F.kind == "e" else _classes_k2(F, rnd)
    # the classes the documented values rest on are exact in Python too, not just matched
    for lab, x in labelled:
        if lab.startswith("subfield") or lab.startswith("r-th power") or lab.startswith("v = 1") or lab == "vd = v":
            if F.kind == "e":
                assert pow(x[0] * pow(x[1], F.q - 2, F.q) % F.q, F.exp, F.q) == 1, lab
            else:
                assert F.pow(x, F.exp) == (1, 0), lab
        if lab.startswith("order-r part"):
            assert F.want(x) != (1, 0), lab
        if lab.startswith("r-th root"):                 # q = h r^2 + 1: r divides (q - 1)/r
            assert F.want(x) == (1,), lab
    if F.kind == "a":
        # the ladder's P = trace of f^(q - 1) = 2 Re(f^(q-1)) on the torus elements that reach it
        traces = set()
        for lab, x in labelled:
            if lab.startswith("order") and x[0] * x[1] % F.q:
                y = F.mul(F.pow(x, F.q), F.pow(x, F.q * F.q - 2))        # f^q / f
                traces.add(2 * y[0] % F.q)
        assert {F.q - 1, 0, 1} <= traces, sorted(t if t < 3 else t - F.q for t in traces)
    # wire coordinates in [q, 2^(8 wb)): every fifth item again with q added to each coordinate where that fits
    top = 1 << (8 * F.wb)
    nc = [("non-canonical " + lab, tuple(c + F.q if c + F.q < top else c for c in x)) for lab, x in labelled[::5]]
    nc = [(lab, x) for lab, x in nc if any(c >= F.q for c in x)]
    assert len(nc) >= 4, name
    _check(F, labelled + nc)


@pytest.mark.parametrize("name", [s for s in SETS if s.startswith("e")])
def test_type_e_without_denominators(name):
    """b = NULL: every denominator is 1, so the output is v^((q - 1)/r), the same bytes as with b all ones"""
    F = fam(name)
    rnd = random.Random("nob-" + name)
    q = F.q
    vs = [0, 1, q - 1] + [F.dom.wire(t) for t in targets(q, F.dom.N)[:8]] + [rnd.randrange(q) for _ in range(6)]
    vs += [pow(rnd.randrange(1, q), (q - 1) // m, q) for m in (2, 4) if F.exp % m == 0]
    got = F.pr.tower_op(3, F.enc(vs), None, len(vs))
    assert got == F.pr.tower_op(3, F.enc(vs), F.enc([1] * len(vs)), len(vs)), name
    bad = [hex(v) for i, v in enumerate(vs) if int.from_bytes(got[i * F.wb:(i + 1) * F.wb], "big") != F.want((v, 1))[0]]
    assert not bad, "%s: b = NULL, %d of %d wrong, first v: %s" % (name, len(bad), len(vs), bad[:3])


@pytest.mark.parametrize("name", [s for s in SETS if s in ("a", "a1", "a1_small")])
def test_python_power_matches_the_oracle_tateexp(name):
    """the exponent used here against the oracle's own final exponentiation, on random elements"""
    F = fam(name)
    orc = O.pairing_from_param(F.text)
    rnd = random.Random("oracle-" + name)
    for _ in range(3):
        x = F.rand2(rnd)
        assert F.pow(x, F.exp) == tuple(orc.tateexp(x)), name


def _chain_batch(F, T):
    """n a little over 3T (not a multiple of T) with shortcut elements at the heads and tails of chains, at
    both ends of the last chain that reaches the fourth row, and along one whole chain; the rest tiles a
    pool of POOL distinct elements"""
    assert T % POOL != 0
    n = 3 * T + T // 3 + 1
    rnd = random.Random("chains-" + F.name)
    q = F.q
    if F.kind == "e":
        pool = [(rnd.randrange(1, q), rnd.randrange(1, q)) for _ in range(POOL - 4)]
        pool += [(1, 1), (q - 1, 1), (0, 1), (0, rnd.randrange(1, q))]          # v = 0 (-> 0) inside chains
        short = [(rnd.randrange(1, q), 0), (0, 0), (1, 0)]
    else:
        pool = [F.rand2(rnd) for _ in range(POOL - 3)]
        pool += [(1, 1), (q - 1, 1), _exact_order(F, 3 if F.kind == "a" else _small_orders(F)[-1], rnd)]
        short = [(rnd.randrange(1, q), 0), (0, rnd.randrange(1, q)), (0, 0), (1, 0)]
    assert all(x[0] * x[1] % q if F.kind != "e" else x[1] for x in pool)   # no shortcut inside the pool
    items = [pool[i % POOL] for i in range(n)]
    K = -(-n // T)
    last = n - (K - 1) * T - 1                      # the last chain with K elements
    pos = set(range(0, T, 97)) | {0, T - 1}                                # heads
    pos |= {(K - 1) * T + t if (K - 1) * T + t < n else (K - 2) * T + t for t in range(5, T, 89)}   # tails
    pos |= {last, (K - 1) * T + last, last + 1, (K - 2) * T + last + 1}    # both ends of the last long and first short chain
    whole = 7 if 7 != last else 8
    pos |= {j * T + whole for j in range(K) if j * T + whole < n}
    pos |= {T + 3, T + 4, 2 * T + 3}                                       # consecutive in one chain and across chains
    for t, p in enumerate(sorted(pos)):
        items[p] = short[t % len(short)]
    return n, items, pool, short, pos, whole


@pytest.mark.parametrize("name", [s for s in SETS if not REDUCED or s in ("a", "a1_small", "e_s510")])
def test_batch_inversion_chains(name):
    F = fam(name)
    T = _sms() * chains_per_sm(F.kind)
    n, items, pool, short, pos, whole = _chain_batch(F, T)
    assert n % T and n > 3 * T and whole not in (0, T - 1)
    want_pool = [F.want(x) for x in pool]
    want_short = [F.want(x) for x in short]
    assert all(w == ((1,) if F.kind == "e" else (1, 0)) for w in want_short)
    got = F.run(items)
    sidx = {x: k for k, x in enumerate(short)}
    bad = []
    for i, (x, g) in enumerate(zip(items, got)):
        w = want_short[sidx[x]] if i in pos else want_pool[i % POOL]
        if g != w:
            bad.append(i)
    desc = ["%d (chain %d, row %d, %s)" % (i, i % T, i // T, "shortcut" if i in pos else "pool") for i in bad[:8]]
    assert not bad, "%s: %d of %d wrong with T = %d chains; first: %s" % (name, len(bad), n, T, desc)

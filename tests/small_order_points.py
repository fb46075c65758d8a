"""Points on the curves of oracle/pbc_oracle.py that the pairing tests need and no fixture holds: random
points of E(K) with no cofactor multiplication (on a twist: almost surely outside G2), and the points
with y = 0, whose x is a root of x^3 + a x + b in K.  Field arithmetic is the oracle's (PrimeField,
QuadExt, PolyModExt); K has `size` elements.  No test functions (tests/golden/make_small_order_golden.py
and tests/test_gpu_small_order_pairings.py use them)."""
from oracle import pbc_oracle as O


def kpow(K, a, e):
    r = K.one
    for bit in bin(e)[2:]:
        r = K.sqr(r)
        if bit == "1":
            r = K.mul(r, a)
    return r


def rand_el(K, rnd):
    if isinstance(K, O.PrimeField):
        return rnd.randrange(K.p)
    if isinstance(K, O.QuadExt):
        return (rand_el(K.b, rnd), rand_el(K.b, rnd))
    return tuple(rand_el(K.b, rnd) for _ in range(K.n))


def sqrt_el(K, a, size, rnd):
    """Tonelli-Shanks in a field of `size` elements; None if a is not a square"""
    if K.eq(a, K.zero):
        return a
    if not K.eq(kpow(K, a, (size - 1) // 2), K.one):
        return None
    s, t = 0, size - 1
    while t % 2 == 0:
        t //= 2
        s += 1
    minus1 = K.neg(K.one)
    while True:
        z = rand_el(K, rnd)
        if K.eq(kpow(K, z, (size - 1) // 2), minus1):
            break
    c, x, b, m = kpow(K, z, t), kpow(K, a, (t + 1) // 2), kpow(K, a, t), s
    while not K.eq(b, K.one):
        i, b2 = 0, b
        while not K.eq(b2, K.one):
            b2 = K.sqr(b2)
            i += 1
        g = c
        for _ in range(m - i - 1):
            g = K.sqr(g)
        x, c = K.mul(x, g), K.sqr(g)
        b, m = K.mul(b, c), i
    return x


def random_point(E, size, rnd):
    """a uniformly drawn x with a point, and one of its two y; y = 0 excluded"""
    K = E.K
    while True:
        x = rand_el(K, rnd)
        rhs = K.add(K.mul(K.add(K.sqr(x), E.a), x), E.b)
        y = sqrt_el(K, rhs, size, rnd)
        if y is not None and not K.eq(y, K.zero):
            return (x, y)


# ---- roots of the cubic: polynomials over K as coefficient lists, lowest power first ------------------

def _trim(K, f):
    while f and K.eq(f[-1], K.zero):
        f = f[:-1]
    return f


def _pmod(K, f, g):
    f, inv = list(f), K.inv(g[-1])
    while len(f) >= len(g):
        c = K.mul(f[-1], inv)
        for i in range(len(g)):
            f[len(f) - len(g) + i] = K.sub(f[len(f) - len(g) + i], K.mul(c, g[i]))
        f = _trim(K, f[:-1])
    return _trim(K, f)


def _pmulmod(K, f, g, m):
    out = [K.zero] * max(1, len(f) + len(g) - 1)
    for i, a in enumerate(f):
        for j, b in enumerate(g):
            out[i + j] = K.add(out[i + j], K.mul(a, b))
    return _pmod(K, _trim(K, out), m)


def _ppowmod(K, f, e, m):
    r = [K.one]
    for bit in bin(e)[2:]:
        r = _pmulmod(K, r, r, m)
        if bit == "1":
            r = _pmulmod(K, r, f, m)
    return r


def _pgcd(K, f, g):
    f, g = _trim(K, f), _trim(K, g)
    while g:
        f, g = g, _pmod(K, f, g)
    return f


def _split_roots(K, f, size, rnd):
    """the roots in K of f, a product of distinct monic linear factors (Cantor-Zassenhaus)"""
    if len(f) <= 1:
        return []
    if len(f) == 2:
        return [K.neg(K.mul(f[0], K.inv(f[1])))]
    while True:
        h = _ppowmod(K, [rand_el(K, rnd), K.one], (size - 1) // 2, f)
        h = list(h) + [K.zero] * (1 - len(h)) if h else [K.zero]
        h[0] = K.sub(h[0], K.one)
        g = _pgcd(K, f, h)
        if 1 < len(g) < len(f):
            q, r = _pdiv(K, f, g)
            return _split_roots(K, g, size, rnd) + _split_roots(K, q, size, rnd)


def _pdiv(K, f, g):
    f, q, inv = list(f), [K.zero] * (len(f) - len(g) + 1), K.inv(g[-1])
    while len(f) >= len(g):
        c = K.mul(f[-1], inv)
        q[len(f) - len(g)] = c
        for i in range(len(g)):
            f[len(f) - len(g) + i] = K.sub(f[len(f) - len(g) + i], K.mul(c, g[i]))
        f = f[:-1]
    return q, _trim(K, f)


def two_torsion(E, size, rnd):
    """every point (t, 0) of E(K): t runs over the roots of x^3 + a x + b in K (gcd with x^size - x,
    then Cantor-Zassenhaus), sorted by their wire bytes"""
    K = E.K
    cubic = [E.b, E.a, K.zero, K.one]
    xq = _ppowmod(K, [K.zero, K.one], size, cubic)
    xq = list(xq) + [K.zero] * (2 - len(xq))
    xq[1] = K.sub(xq[1], K.one)
    lin = _pgcd(K, cubic, xq)
    lin = [K.mul(c, K.inv(lin[-1])) for c in lin]
    pts = [(t, K.zero) for t in _split_roots(K, lin, size, rnd)]
    assert all(E.is_valid(P) for P in pts)
    return sorted(pts, key=E.to_bytes)

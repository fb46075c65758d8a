"""Type E (k = 1) pairing restated in Python integers with the kernels' formulas (pbc_b200/csrc/
pairing_e.cuh): Jacobian V, Q + R Jacobian with homogenised lines, the sign branches and the
skipped verticals at x(P).  R is an argument: for P in G1 the value does not depend on it, so the
restatement must equal the compiled reference (tests/golden/e*.json) for any R outside E[r], and the
library's own R (pbc_b200_derived_constant "R") must give the library's bytes.  Test infrastructure."""


def parse_param(text):
    toks = [t for line in text.splitlines() for t in line.split("#")[0].split()]
    tab = dict(zip(toks[::2], toks[1::2]))
    out = {k: int(tab[k]) for k in ("q", "r", "h", "a", "b", "exp2", "exp1", "sign1", "sign0")}
    return out


class PairingE:
    def __init__(self, text, R):
        p = parse_param(text)
        self.q, self.r, self.a, self.b = p["q"], p["r"], p["a"] % p["q"], p["b"] % p["q"]
        self.exp1, self.exp2, self.sign1, self.sign0 = p["exp1"], p["exp2"], p["sign1"], p["sign0"]
        self.wb = (self.q.bit_length() + 7) // 8
        self.R = R
        assert self.on_curve(R)

    # ---- wire format ----
    def point(self, data):
        """(x, y) reduced mod q, or None when not on the curve (the reference's O)"""
        wb = self.wb
        x = int.from_bytes(data[:wb], "big") % self.q
        y = int.from_bytes(data[wb:2 * wb], "big") % self.q
        return (x, y) if self.on_curve((x, y)) else None

    def on_curve(self, P):
        x, y = P
        return (y * y - (x * x * x + self.a * x + self.b)) % self.q == 0

    def gt_bytes(self, v):
        return v.to_bytes(self.wb, "big")

    # ---- the pairing ----
    def miller(self, P, Q):
        """(v, vd) of the kernel, Q + R homogenised"""
        q, a = self.q, self.a
        Rx, Ry = self.R
        # Q + R, Jacobian (mixed addition)
        H = (Rx - Q[0]) % q
        rr = (Ry - Q[1]) % q
        H2 = H * H % q
        H3 = H2 * H % q
        U = Q[0] * H2 % q
        Xq = (rr * rr - H3 - 2 * U) % q
        Yq = (rr * (U - Xq) - Q[1] * H3) % q
        Zq2, Zq3, XZq = H2, H3, Xq * H % q

        def line_q(la, lb, lc):
            return (la * XZq + lb * Yq + lc * Zq3) % q

        def line_r(la, lb, lc):
            return (la * Rx + lb * Ry + lc) % q

        def vert_q(Z2, X):
            return (Xq * Z2 - X * Zq2) % q

        def vert_r(Z2, X):
            return (Rx * Z2 - X) % q

        X, Y, Z = P[0], P[1], 1
        v = vd = 1
        v1 = vd1 = None
        for i in range(self.exp2):
            if i == self.exp1:
                Z2 = Z * Z % q
                if self.sign1 < 0:
                    v1, vd1, S = vd * vert_r(Z2, X) % q, v * vert_q(Z2, X) % q, (X, -Y % q, Z)
                else:
                    v1, vd1, S = v, vd, (X, Y, Z)
            v, vd = v * v % q, vd * vd % q
            Z2 = Z * Z % q
            M = (3 * X * X + a * Z2 * Z2) % q
            Y2 = Y * Y % q
            lc = (X * M - 2 * Y2) % q
            la = -M * Z2 % q
            Zn = 2 * Y * Z % q
            lb = Zn * Z2 % q
            vd = vd * line_r(la, lb, lc) % q
            v = v * line_q(la, lb, lc) % q
            S4 = 4 * X * Y2 % q
            Xn = (M * M - 2 * S4) % q
            Y = (M * (S4 - Xn) - 8 * Y2 * Y2) % q
            X, Z = Xn, Zn
            Z2 = Z * Z % q
            vd = vd * vert_q(Z2, X) % q
            v = v * vert_r(Z2, X) % q
        v, vd = v * v1 % q, vd * vd1 % q
        X1, Y1, Z1 = S
        Zv2, Zv3 = Z * Z % q, Z * Z * Z % q
        Z12, Z13 = Z1 * Z1 % q, Z1 * Z1 * Z1 % q
        ca = (Y * Z13 - Y1 * Zv3) % q
        cb = (X1 * Zv2 - X * Z12) * Z1 * Z % q
        cc = (X * Y1 * Z - Y * X1 * Z1) % q
        vd = vd * line_r(ca, cb, cc) % q
        v = v * line_q(ca, cb, cc) % q
        if self.sign0 < 0:
            vd = vd * (Xq - P[0] * Zq2) % q
            v = v * (Rx - P[0]) % q
        return v, vd

    def pairing(self, Pb, Qb):
        P, Q = self.point(Pb), self.point(Qb)
        if P is None or Q is None:
            return self.gt_bytes(1)
        v, vd = self.miller(P, Q)
        if vd == 0:
            return self.gt_bytes(1)
        return self.gt_bytes(pow(v * pow(vd, -1, self.q) % self.q, (self.q - 1) // self.r, self.q))

    def pairing_batch(self, P, Q, n):
        L = 2 * self.wb
        return b"".join(self.pairing(P[i * L:(i + 1) * L], Q[i * L:(i + 1) * L]) for i in range(n))


def any_r(text, start=1):
    """some point outside E[r] (the restatement's own R, not the library's): y^2 = x^3 + a x + b at the
    first x >= start with a square right-hand side and r (x, y) != O"""
    p = parse_param(text)
    q, a, b, r = p["q"], p["a"] % p["q"], p["b"] % p["q"], p["r"]
    x = start
    while True:
        t = (x * x * x + a * x + b) % q
        if t and pow(t, (q - 1) // 2, q) == 1:
            y = sqrt_mod(t, q)
            if not is_inf(mul(r, (x, y), a, q)):
                return (x, y)
        x += 1


def sqrt_mod(t, q):
    s, Q = 0, q - 1
    while Q % 2 == 0:
        Q //= 2
        s += 1
    z = 2
    while pow(z, (q - 1) // 2, q) != q - 1:
        z += 1
    m, c, x, b = s, pow(z, Q, q), pow(t, (Q + 1) // 2, q), pow(t, Q, q)
    while b != 1:
        i, b2 = 0, b
        while b2 != 1:
            b2 = b2 * b2 % q
            i += 1
        g = pow(c, 1 << (m - i - 1), q)
        x, c = x * g % q, g * g % q
        b, m = b * c % q, i
    return x


def is_inf(P):
    return P is None


def add(P, Q, a, q):
    if P is None:
        return Q
    if Q is None:
        return P
    if P[0] == Q[0]:
        if (P[1] + Q[1]) % q == 0:
            return None
        lam = (3 * P[0] * P[0] + a) * pow(2 * P[1], -1, q) % q
    else:
        lam = (Q[1] - P[1]) * pow(Q[0] - P[0], -1, q) % q
    x = (lam * lam - P[0] - Q[0]) % q
    return (x, (lam * (P[0] - x) - P[1]) % q)


def mul(k, P, a, q):
    acc = None
    for bit in bin(k)[2:]:
        acc = add(acc, acc, a, q)
        if bit == "1":
            acc = add(acc, P, a, q)
    return acc

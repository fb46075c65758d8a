"""ref.py -- ctypes binding of oracle/_ref/libpbcref.so (the compiled, unmodified reference).

TEST INFRASTRUCTURE ONLY: checker and CPU baseline.  Built by `make -C oracle`.
"""
from __future__ import annotations
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "_ref", "libpbcref.so")
BENCH_PATH = os.path.join(_HERE, "_ref", "benchmark")


def available() -> bool:
    if not os.path.exists(LIB_PATH):
        return False
    try:
        _lib()
        return True
    except OSError:
        return False


_cached = None


def _lib():
    global _cached
    if _cached is None:
        L = C.CDLL(LIB_PATH)
        L.pbcref_open.restype = C.c_void_p
        L.pbcref_open.argtypes = [C.c_char_p, C.c_size_t]
        L.pbcref_close.argtypes = [C.c_void_p]
        L.pbcref_sizes.argtypes = [C.c_void_p, C.POINTER(C.c_int)]
        L.pbcref_seed.argtypes = [C.c_ulong]
        L.pbcref_random.argtypes = [C.c_void_p, C.c_int, C.c_char_p, C.c_size_t]
        L.pbcref_walk.argtypes = [C.c_void_p, C.c_int, C.c_char_p, C.c_size_t]
        for f in (L.pbcref_pairing, L.pbcref_pp_pairing):
            f.restype = C.c_double
            f.argtypes = [C.c_void_p, C.c_char_p, C.c_char_p, C.c_char_p, C.c_size_t]
        L.pbcref_prod_pairing.restype = C.c_double
        L.pbcref_prod_pairing.argtypes = [C.c_void_p, C.c_char_p, C.c_char_p, C.c_char_p,
                                          C.c_size_t, C.c_size_t]
        L.pbcref_pow_zn.argtypes = [C.c_void_p, C.c_int, C.c_char_p, C.c_char_p, C.c_char_p,
                                    C.c_size_t]
        L.pbcref_mul.argtypes = [C.c_void_p, C.c_int, C.c_char_p, C.c_char_p, C.c_char_p,
                                 C.c_size_t]
        L.pbcref_from_str.argtypes = [C.c_void_p, C.c_int, C.c_char_p, C.c_char_p]
        L.pbcref_compressed_len.argtypes = [C.c_void_p, C.c_int]
        L.pbcref_compress.argtypes = [C.c_void_p, C.c_int, C.c_char_p, C.c_char_p, C.c_size_t]
        L.pbcref_decompress.argtypes = [C.c_void_p, C.c_int, C.c_char_p, C.c_char_p, C.c_size_t]
        L.pbcref_from_hash.argtypes = [C.c_void_p, C.c_int, C.c_char_p, C.c_int, C.c_char_p, C.c_size_t]
        L.pbcref_is_identity.argtypes = [C.c_void_p, C.c_int, C.c_char_p]
        _cached = L
    return _cached


G1, G2, GT, ZR = 1, 2, 3, 0


class RefPairing:
    """One reference pairing_t (the library is not thread-safe: one per process)."""

    def __init__(self, param_text: str):
        self.L = _lib()
        b = param_text.encode()
        self.h = self.L.pbcref_open(b, len(b))
        if not self.h:
            raise ValueError("reference rejected the parameters")
        sz = (C.c_int * 4)()
        self.L.pbcref_sizes(self.h, sz)
        self.g1_len, self.g2_len, self.gt_len, self.zr_len = list(sz)
        self.last_seconds = 0.0

    def close(self):
        """pairing_clear; the handle is unusable afterwards"""
        if self.h:
            self.L.pbcref_close(self.h)
            self.h = None

    def _len(self, group):
        return {G1: self.g1_len, G2: self.g2_len, GT: self.gt_len, ZR: self.zr_len}[group]

    @staticmethod
    def seed(s: int):
        _lib().pbcref_seed(s)

    def random(self, group, n) -> bytes:
        buf = C.create_string_buffer(n * self._len(group))
        self.L.pbcref_random(self.h, group, buf, n)
        return buf.raw

    def walk(self, group, n) -> bytes:
        buf = C.create_string_buffer(n * self._len(group))
        self.L.pbcref_walk(self.h, group, buf, n)
        return buf.raw

    def pairing(self, P: bytes, Q: bytes, n: int) -> bytes:
        out = C.create_string_buffer(n * self.gt_len)
        self.last_seconds = self.L.pbcref_pairing(self.h, P, Q, out, n)
        return out.raw

    def pp_pairing(self, P: bytes, Q: bytes, n: int) -> bytes:
        out = C.create_string_buffer(n * self.gt_len)
        self.last_seconds = self.L.pbcref_pp_pairing(self.h, P, Q, out, n)
        return out.raw

    def prod_pairing(self, P: bytes, Q: bytes, k: int, n_out: int) -> bytes:
        out = C.create_string_buffer(n_out * self.gt_len)
        self.last_seconds = self.L.pbcref_prod_pairing(self.h, P, Q, out, k, n_out)
        return out.raw

    def pow_zn(self, group, x: bytes, k: bytes, n: int) -> bytes:
        out = C.create_string_buffer(n * self._len(group))
        self.L.pbcref_pow_zn(self.h, group, x, k, out, n)
        return out.raw

    def from_hash(self, group, data: bytes, length: int, n: int) -> bytes:
        out = C.create_string_buffer(n * self._len(group))
        self.L.pbcref_from_hash(self.h, group, data, length, out, n)
        return out.raw

    def compress(self, group, x: bytes, n: int) -> bytes:
        clen = self.L.pbcref_compressed_len(self.h, group)
        out = C.create_string_buffer(n * clen)
        self.L.pbcref_compress(self.h, group, x, out, n)
        return out.raw

    def decompress(self, group, x: bytes, n: int) -> bytes:
        out = C.create_string_buffer(n * self._len(group))
        self.L.pbcref_decompress(self.h, group, x, out, n)
        return out.raw

    def mul(self, group, a: bytes, b: bytes, n: int) -> bytes:
        out = C.create_string_buffer(n * self._len(group))
        self.L.pbcref_mul(self.h, group, a, b, out, n)
        return out.raw

    def from_str(self, group, s: str) -> bytes:
        out = C.create_string_buffer(self._len(group))
        self.L.pbcref_from_str(self.h, group, s.encode(), out)
        return out.raw

    def is_identity(self, group, x: bytes) -> bool:
        return bool(self.L.pbcref_is_identity(self.h, group, x))

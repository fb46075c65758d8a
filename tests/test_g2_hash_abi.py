"""CPU-side checks of the G2 hashing and compressed-point entry points: the symbols are exported, the
compressed length is the x width plus one, and every argument error (null pointers, hash length outside
1..2^20, type e) is reported with its own message before any CUDA call, so it
reads the same with or without a GPU; n = 0 returns 0 and touches nothing."""
import ctypes as C
import os

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SYMBOLS = ("pbc_b200_g2_from_hash", "pbc_b200_g2_from_hash_device", "pbc_b200_pairing_length_in_bytes_compressed_G2",
           "pbc_b200_g2_from_bytes_compressed")


@pytest.fixture(scope="module")
def built():
    import __graft_entry__ as ge
    ge.build()
    from pbc_b200 import pairing
    return pairing


def _handle(built, name):
    from pbc_b200.params import PARAMS
    return built.Pairing(PARAMS[name])


def test_symbols_are_exported(built):
    lib = C.CDLL(os.path.join(ROOT, "pbc_b200", "libpbc_b200.so"))
    for n in SYMBOLS:
        assert hasattr(lib, n), n


@pytest.mark.parametrize("name,clen", [("a", 65), ("a1", 131), ("f", 41), ("d159", 61), ("g149", 96)])
def test_compressed_length(built, name, clen):
    from pbc_b200._lib import lib
    p = _handle(built, name)
    assert lib.pbc_b200_pairing_length_in_bytes_compressed_G2(p.handle) == clen == p.g2_len // 2 + 1
    if name in ("a", "a1"):
        assert lib.pbc_b200_pairing_length_in_bytes_compressed_G1(p.handle) == clen


def _no_cuda(built, fn, match):
    from pbc_b200._lib import lib, last_error
    before = lib.pbc_b200_kernel_launches()
    assert fn() != 0
    msg = last_error()
    assert match in msg and "CUDA" not in msg, msg
    assert lib.pbc_b200_kernel_launches() == before


@pytest.mark.parametrize("name", ("a", "f", "d159", "g149", "e"))
def test_argument_errors_come_before_any_cuda_call(built, name):
    from pbc_b200._lib import lib
    p = _handle(built, name)
    h, buf = p.handle, C.create_string_buffer(4096)
    if name == "e":
        with pytest.raises(built.PairingError, match="not available for type e"):
            p.g2_compress(bytes(p.g2_len), 1)
        _no_cuda(built, lambda: lib.pbc_b200_g2_from_hash(h, buf, buf, 32, 1), "type e")
        _no_cuda(built, lambda: lib.pbc_b200_g2_from_hash_device(h, buf, buf, 32, 1, None), "type e")
        _no_cuda(built, lambda: lib.pbc_b200_g2_from_bytes_compressed(h, buf, buf, 1), "type e")
        return
    _no_cuda(built, lambda: lib.pbc_b200_g2_from_hash(h, None, buf, 32, 1), "null argument")
    _no_cuda(built, lambda: lib.pbc_b200_g2_from_hash(h, buf, None, 32, 1), "null argument")
    _no_cuda(built, lambda: lib.pbc_b200_g2_from_hash(None, buf, buf, 32, 1), "null argument")
    _no_cuda(built, lambda: lib.pbc_b200_g2_from_hash(h, buf, buf, 0, 1), "1..2^20")
    _no_cuda(built, lambda: lib.pbc_b200_g2_from_hash(h, buf, buf, (1 << 20) + 1, 1), "1..2^20")
    _no_cuda(built, lambda: lib.pbc_b200_g2_from_hash_device(h, buf, buf, 0, 1, None), "1..2^20")
    _no_cuda(built, lambda: lib.pbc_b200_g2_from_bytes_compressed(h, None, buf, 1), "null argument")
    _no_cuda(built, lambda: lib.pbc_b200_g2_from_bytes_compressed(h, buf, None, 1), "null argument")
    # n = 0: nothing to do, success without a device
    assert lib.pbc_b200_g2_from_hash(h, None, None, 32, 0) == 0
    assert lib.pbc_b200_g2_from_bytes_compressed(h, None, None, 0) == 0


def test_python_wrappers_check_lengths(built):
    p = _handle(built, "f")
    with pytest.raises(ValueError):
        p.g2_from_hash(b"abc", 2, 2)
    with pytest.raises(ValueError):
        p.g2_decompress(b"\0" * 40, 1)
    # compression is host-only: x || (1 if the first non-zero coordinate of y is odd)
    x, y0, y1 = bytes(40), (2).to_bytes(20, "big"), (3).to_bytes(20, "big")
    assert p.g2_compress(x + y0 + y1, 1) == x + b"\0"
    assert p.g2_compress(x + bytes(20) + y1, 1) == x + b"\1"
    assert p.g2_compress(x + bytes(40), 1) == x + b"\0"

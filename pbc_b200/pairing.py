"""Host-side mirror of the reference pairing interface, batched.

Names follow the reference (include/pbc_pairing.h): a `Pairing` is a pairing_t initialised from
parameter text (pairing_init_set_str); `apply` is element_pairing over a batch;
`prod_apply` is element_prod_pairing (k pairs per output), `prod_apply_v` the same with a pair count
per output (ragged batches); `pp_apply` is pairing_pp_init + pairing_pp_apply.
Elements travel as reference wire-format bytes (element_to_bytes / element_from_bytes).
All arithmetic happens in libpbc_b200.so on the GPU; this file only marshals buffers.
"""
from __future__ import annotations
import ctypes as C

from ._lib import lib, last_error


class PairingError(RuntimeError):
    pass


def _addr(buf):
    """address of a host buffer: int, bytes, ctypes buffer, numpy array or torch tensor"""
    if buf is None:
        return None
    if isinstance(buf, int):
        return buf
    if hasattr(buf, "data_ptr"):          # torch tensor
        return buf.data_ptr()
    if hasattr(buf, "ctypes"):            # numpy array
        return buf.ctypes.data
    if isinstance(buf, bytes):
        return C.cast(C.c_char_p(buf), C.c_void_p).value
    if isinstance(buf, bytearray):
        return C.addressof((C.c_char * len(buf)).from_buffer(buf))
    return C.addressof(buf)


class Pairing:
    def __init__(self, param_text):
        """pairing_init_set_str (ecc/pairing.c:100-102); raises where the reference returns 1."""
        self._h = C.c_void_p()
        b = param_text.encode() if isinstance(param_text, str) else bytes(param_text)
        if lib.pbc_b200_pairing_init_set_buf(C.byref(self._h), b, len(b)):
            self._h = C.c_void_p()
            raise PairingError(last_error())
        self.g1_len = lib.pbc_b200_pairing_length_in_bytes_G1(self._h)
        self.g2_len = lib.pbc_b200_pairing_length_in_bytes_G2(self._h)
        self.gt_len = lib.pbc_b200_pairing_length_in_bytes_GT(self._h)
        t = chr(lib.pbc_b200_pairing_type(self._h))
        self.type = "a1" if t == "1" else t
        self.zr_len = lib.pbc_b200_pairing_length_in_bytes_Zr(self._h)

    def clear(self):
        """pairing_clear"""
        if getattr(self, "_h", None):
            lib.pbc_b200_pairing_clear(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.clear()
        except Exception:
            pass

    @property
    def handle(self):
        return self._h

    def set_devices(self, count: int):
        if lib.pbc_b200_set_devices(self._h, count):
            raise PairingError(last_error())

    # -- element_pairing over a batch -------------------------------------------------------
    def apply(self, in1: bytes, in2: bytes, n=None) -> bytes:
        if n is None:
            n = len(in1) // self.g1_len
        if len(in1) < n * self.g1_len or len(in2) < n * self.g2_len:
            raise ValueError("input buffers shorter than n elements")
        out = C.create_string_buffer(max(1, n * self.gt_len))
        if lib.pbc_b200_pairings_apply(self._h, C.addressof(out), _addr(in1), _addr(in2), n):
            raise PairingError(last_error())
        return out.raw[:n * self.gt_len]

    def apply_into(self, out, in1, in2, n: int):
        """Host buffers given by address-bearing objects (pinned torch tensors, numpy arrays)."""
        if lib.pbc_b200_pairings_apply(self._h, _addr(out), _addr(in1), _addr(in2), n):
            raise PairingError(last_error())

    def apply_device(self, d_out: int, d_in1: int, d_in2: int, n: int, stream: int = 0):
        """Device pointers (e.g. torch.Tensor.data_ptr()), asynchronous on `stream`."""
        if lib.pbc_b200_pairings_apply_device(self._h, d_out, d_in1, d_in2, n, stream):
            raise PairingError(last_error())

    # -- element_prod_pairing -----------------------------------------------------------------
    @staticmethod
    def _need(buf, nbytes, what):
        """length check for bytes-like host buffers (addresses and tensors are the caller's business)"""
        if isinstance(buf, (bytes, bytearray, memoryview)) and len(buf) < nbytes:
            raise ValueError("%s: buffer of %d bytes, %d needed" % (what, len(buf), nbytes))

    def prod_apply(self, in1: bytes, in2: bytes, k: int, n_out=None) -> bytes:
        if k < 1:
            raise ValueError("prod_apply: k must be positive")
        if n_out is None:
            n_out = len(in1) // (self.g1_len * k)
        self._need(in1, n_out * k * self.g1_len, "prod_apply in1")
        self._need(in2, n_out * k * self.g2_len, "prod_apply in2")
        out = C.create_string_buffer(max(1, n_out * self.gt_len))
        if lib.pbc_b200_prod_pairings_apply(self._h, C.addressof(out), _addr(in1), _addr(in2), k, n_out):
            raise PairingError(last_error())
        return out.raw[:n_out * self.gt_len]

    def prod_apply_into(self, out, in1, in2, k: int, n_out: int):
        if lib.pbc_b200_prod_pairings_apply(self._h, _addr(out), _addr(in1), _addr(in2), k, n_out):
            raise PairingError(last_error())

    def prod_apply_device(self, d_out, d_in1, d_in2, k, n_out, stream=0):
        if lib.pbc_b200_prod_pairings_apply_device(self._h, d_out, d_in1, d_in2, k, n_out, stream):
            raise PairingError(last_error())

    # -- element_prod_pairing with a pair count per output ---------------------------------------
    @staticmethod
    def _offsets(offsets):
        """offsets (any integer sequence or numpy array, n_out + 1 entries) as a C size_t array; the
        library checks that they start at 0 and increase"""
        vals = offsets.tolist() if hasattr(offsets, "tolist") else list(offsets)
        if not vals:
            raise ValueError("offsets: n_out + 1 entries needed")
        if any(isinstance(v, bool) or not isinstance(v, int) or v < 0 for v in vals):
            raise ValueError("offsets: non-negative integers needed")
        return (C.c_size_t * len(vals))(*vals), len(vals) - 1

    def prod_apply_v(self, in1: bytes, in2: bytes, offsets) -> bytes:
        """out[i] = prod of e(in1[j], in2[j]) over offsets[i] <= j < offsets[i+1]"""
        offs, n_out = self._offsets(offsets)
        m = offs[n_out]
        self._need(in1, m * self.g1_len, "prod_apply_v in1")
        self._need(in2, m * self.g2_len, "prod_apply_v in2")
        out = C.create_string_buffer(max(1, n_out * self.gt_len))
        if lib.pbc_b200_prod_pairings_apply_v(self._h, C.addressof(out), _addr(in1), _addr(in2), C.addressof(offs), n_out):
            raise PairingError(last_error())
        return out.raw[:n_out * self.gt_len]

    def prod_apply_v_into(self, out, in1, in2, offsets):
        offs, n_out = self._offsets(offsets)
        m = offs[n_out]
        self._need(out, n_out * self.gt_len, "prod_apply_v out")
        self._need(in1, m * self.g1_len, "prod_apply_v in1")
        self._need(in2, m * self.g2_len, "prod_apply_v in2")
        if lib.pbc_b200_prod_pairings_apply_v(self._h, _addr(out), _addr(in1), _addr(in2), C.addressof(offs), n_out):
            raise PairingError(last_error())

    def prod_apply_v_device(self, d_out, d_in1, d_in2, offsets, stream=0):
        """device pointers, offsets on the host; asynchronous on `stream`"""
        offs, n_out = self._offsets(offsets)
        if lib.pbc_b200_prod_pairings_apply_v_device(self._h, d_out, d_in1, d_in2, C.addressof(offs), n_out, stream):
            raise PairingError(last_error())

    # -- pairing_pp_init / pairing_pp_apply -------------------------------------------------------
    def pp_apply(self, in1: bytes, in2: bytes, n=None) -> bytes:
        if n is None:
            n = len(in2) // self.g2_len
        self._need(in1, self.g1_len, "pp_apply in1")
        self._need(in2, n * self.g2_len, "pp_apply in2")
        out = C.create_string_buffer(max(1, n * self.gt_len))
        if lib.pbc_b200_pp_pairings_apply(self._h, C.addressof(out), _addr(in1), _addr(in2), n):
            raise PairingError(last_error())
        return out.raw[:n * self.gt_len]

    def pp_apply_into(self, out, in1, in2, n: int):
        if lib.pbc_b200_pp_pairings_apply(self._h, _addr(out), _addr(in1), _addr(in2), n):
            raise PairingError(last_error())

    def pp_apply_device(self, d_out, d_in1, d_in2, n, stream=0):
        if lib.pbc_b200_pp_pairings_apply_device(self._h, d_out, d_in1, d_in2, n, stream):
            raise PairingError(last_error())

    def pp_init(self, in1: bytes) -> "PairingPP":
        """pairing_pp_init: preprocess one first argument; the table stays on the GPU until clear()"""
        self._need(in1, self.g1_len, "pp_init in1")
        return PairingPP(self, in1)

    # -- element_pow_zn on G1 / GT (include/pbc_field.h:262-275) ------------------------------------
    def g1_pow_zn(self, points: bytes, scalars: bytes, n=None) -> bytes:
        if n is None:
            n = len(points) // self.g1_len
        self._need(points, n * self.g1_len, "g1_pow_zn points")
        self._need(scalars, n * self.zr_len, "g1_pow_zn scalars")
        out = C.create_string_buffer(max(1, n * self.g1_len))
        if lib.pbc_b200_g1_pow_zn(self._h, C.addressof(out), _addr(points), _addr(scalars), n):
            raise PairingError(last_error())
        return out.raw[:n * self.g1_len]

    def g1_from_hash(self, data: bytes, length: int, n=None) -> bytes:
        """element_from_hash on G1 for n hashes of `length` bytes each, back to back"""
        if n is None:
            n = len(data) // length
        self._need(data, n * length, "g1_from_hash data")
        out = C.create_string_buffer(max(1, n * self.g1_len))
        if lib.pbc_b200_g1_from_hash(self._h, C.addressof(out), _addr(data), length, n):
            raise PairingError(last_error())
        return out.raw[:n * self.g1_len]

    def g1_from_hash_device(self, d_out, d_data, length, n, stream=0):
        if lib.pbc_b200_g1_from_hash_device(self._h, d_out, d_data, length, n, stream):
            raise PairingError(last_error())

    def g1_compress(self, points: bytes, n=None) -> bytes:
        """element_to_bytes_compressed (ecc/curve.c:762-775): x || (1 if y is odd else 0); host only"""
        L = self.g1_len
        if n is None:
            n = len(points) // L
        return b"".join(points[i * L:i * L + L // 2] + bytes([points[(i + 1) * L - 1] & 1]) for i in range(n))

    def g1_decompress(self, data: bytes, n=None) -> bytes:
        """element_from_bytes_compressed on the GPU"""
        clen = self.g1_len // 2 + 1
        if n is None:
            n = len(data) // clen
        self._need(data, n * clen, "g1_decompress data")
        out = C.create_string_buffer(max(1, n * self.g1_len))
        if lib.pbc_b200_g1_from_bytes_compressed(self._h, C.addressof(out), _addr(data), n):
            raise PairingError(last_error())
        return out.raw[:n * self.g1_len]

    def g2_from_hash(self, data: bytes, length: int, n=None) -> bytes:
        """element_from_hash on G2 for n hashes of `length` bytes each, back to back (types f, d, g: the
        twist point the reference finds, no cofactor; types a, a1: as g1_from_hash)"""
        if n is None:
            n = len(data) // length
        self._need(data, n * length, "g2_from_hash data")
        out = C.create_string_buffer(max(1, n * self.g2_len))
        if lib.pbc_b200_g2_from_hash(self._h, C.addressof(out), _addr(data), length, n):
            raise PairingError(last_error())
        return out.raw[:n * self.g2_len]

    def g2_from_hash_device(self, d_out, d_data, length, n, stream=0):
        if lib.pbc_b200_g2_from_hash_device(self._h, d_out, d_data, length, n, stream):
            raise PairingError(last_error())

    @staticmethod
    def _sign(coords, wb):
        """element_sign of a wire-format field element: the parity of its first non-zero coordinate
        (fp_sgn_odd, fq_sign, polymod_sgn), 1 odd, -1 even, 0 for zero"""
        for i in range(0, len(coords), wb):
            v = int.from_bytes(coords[i:i + wb], "big")
            if v:
                return 1 if v & 1 else -1
        return 0

    def g2_compress(self, points: bytes, n=None) -> bytes:
        """element_to_bytes_compressed on G2 (ecc/curve.c:762-775): x || (1 if sign(y) > 0 else 0), with
        the sign of the twist's field (the first non-zero coordinate of y decides); host only"""
        if self.type in ("a", "a1"):
            return self.g1_compress(points, n)
        if self.type not in ("f", "d", "g"):
            raise PairingError("element_to_bytes_compressed: not available for type %s" % self.type)
        L = self.g2_len
        if n is None:
            n = len(points) // L
        wb = {"f": L // 4, "d": L // 6, "g": L // 10}[self.type]
        return b"".join(points[i * L:i * L + L // 2] +
                        bytes([1 if self._sign(points[i * L + L // 2:(i + 1) * L], wb) > 0 else 0]) for i in range(n))

    def g2_decompress(self, data: bytes, n=None) -> bytes:
        """element_from_bytes_compressed on G2, on the GPU"""
        clen = lib.pbc_b200_pairing_length_in_bytes_compressed_G2(self._h)
        if n is None:
            n = len(data) // clen
        self._need(data, n * clen, "g2_decompress data")
        out = C.create_string_buffer(max(1, n * self.g2_len))
        if lib.pbc_b200_g2_from_bytes_compressed(self._h, C.addressof(out), _addr(data), n):
            raise PairingError(last_error())
        return out.raw[:n * self.g2_len]

    def g2_pow_zn(self, points: bytes, scalars: bytes, n=None) -> bytes:
        if n is None:
            n = len(points) // self.g2_len
        self._need(points, n * self.g2_len, "g2_pow_zn points")
        self._need(scalars, n * self.zr_len, "g2_pow_zn scalars")
        out = C.create_string_buffer(max(1, n * self.g2_len))
        if lib.pbc_b200_g2_pow_zn(self._h, C.addressof(out), _addr(points), _addr(scalars), n):
            raise PairingError(last_error())
        return out.raw[:n * self.g2_len]

    def gt_pow_zn(self, elems: bytes, scalars: bytes, n=None) -> bytes:
        if n is None:
            n = len(elems) // self.gt_len
        self._need(elems, n * self.gt_len, "gt_pow_zn elems")
        self._need(scalars, n * self.zr_len, "gt_pow_zn scalars")
        out = C.create_string_buffer(max(1, n * self.gt_len))
        if lib.pbc_b200_gt_pow_zn(self._h, C.addressof(out), _addr(elems), _addr(scalars), n):
            raise PairingError(last_error())
        return out.raw[:n * self.gt_len]

    # -- element_mul / element_cmp on GT, is_almost_coddh (include/pbc_pairing.h:240-243) -------------
    def gt_mul(self, a: bytes, b: bytes, n=None) -> bytes:
        if n is None:
            n = len(a) // self.gt_len
        self._need(a, n * self.gt_len, "gt_mul a")
        self._need(b, n * self.gt_len, "gt_mul b")
        out = C.create_string_buffer(max(1, n * self.gt_len))
        if lib.pbc_b200_gt_mul(self._h, C.addressof(out), _addr(a), _addr(b), n):
            raise PairingError(last_error())
        return out.raw[:n * self.gt_len]

    def gt_cmp(self, a: bytes, b: bytes, n=None) -> bytes:
        """one byte per element: 0 if equal (element_cmp returns 0), 1 otherwise"""
        if n is None:
            n = len(a) // self.gt_len
        self._need(a, n * self.gt_len, "gt_cmp a")
        self._need(b, n * self.gt_len, "gt_cmp b")
        out = C.create_string_buffer(max(1, n))
        if lib.pbc_b200_gt_cmp(self._h, C.addressof(out), _addr(a), _addr(b), n):
            raise PairingError(last_error())
        return out.raw[:n]

    def is_almost_coddh(self, a: bytes, b: bytes, c: bytes, d: bytes, n=None) -> bytes:
        """one byte per tuple: 1 if e(a, d) = e(b, c)^(+-1)"""
        if n is None:
            n = len(a) // self.g1_len
        self._need(a, n * self.g1_len, "is_almost_coddh a")
        self._need(b, n * self.g1_len, "is_almost_coddh b")
        self._need(c, n * self.g2_len, "is_almost_coddh c")
        self._need(d, n * self.g2_len, "is_almost_coddh d")
        out = C.create_string_buffer(max(1, n))
        if lib.pbc_b200_is_almost_coddh(self._h, C.addressof(out), _addr(a), _addr(b), _addr(c), _addr(d), n):
            raise PairingError(last_error())
        return out.raw[:n]

    def g1_pow_zn_device(self, d_out, d_in, d_k, n, stream=0):
        if lib.pbc_b200_g1_pow_zn_device(self._h, d_out, d_in, d_k, n, stream):
            raise PairingError(last_error())

    def g2_pow_zn_device(self, d_out, d_in, d_k, n, stream=0):
        if lib.pbc_b200_g2_pow_zn_device(self._h, d_out, d_in, d_k, n, stream):
            raise PairingError(last_error())

    def gt_pow_zn_device(self, d_out, d_in, d_k, n, stream=0):
        if lib.pbc_b200_gt_pow_zn_device(self._h, d_out, d_in, d_k, n, stream):
            raise PairingError(last_error())

    # -- test / bench hooks -----------------------------------------------------------------------
    def fp_op(self, op: int, a: bytes, b, n: int, widths=(1, 1, 1)) -> bytes:
        """widths: coordinates per item in a, b and the result (type a ops 8-14 take several, see
        pbc_b200_fp_op); the library knows them per op, they size and check the buffers here"""
        wb = self.g1_len // 2          # bytes per F_q coordinate
        self._need(a, n * wb * widths[0], "fp_op a")
        if b is not None:
            self._need(b, n * wb * widths[1], "fp_op b")
        out = C.create_string_buffer(max(1, n * wb * widths[2]))
        if lib.pbc_b200_fp_op(self._h, op, C.addressof(out), _addr(a), _addr(b), n):
            raise PairingError(last_error())
        return out.raw[:n * wb * widths[2]]

    def tower_op(self, op: int, a: bytes, b, n: int) -> bytes:
        """pbc_b200_tower_op: n GT wire elements in a (and b), n out.  Types f, d, g: the extension-tower
        ops 0-6.  Types a, a1, e: op 3 only, the final stage the pairings run (batch inversion, then the
        final exponentiation) on Miller values given in GT wire format -- a, a1: f = a[i], f0 f1 = 0 gives
        1; e: numerator a[i] over denominator b[i] (1 where b is None), vd = 0 gives 1, v = 0 gives 0."""
        out = C.create_string_buffer(n * self.gt_len)
        if lib.pbc_b200_tower_op(self._h, op, C.addressof(out), _addr(a), _addr(b), n):
            raise PairingError(last_error())
        return out.raw

    def derived_constant(self, name: str, width: int):
        """canonical residues of a constant derived at init time, as a list of ints (tests)"""
        buf = C.create_string_buffer(16 * width)
        got = lib.pbc_b200_derived_constant(self._h, name.encode(), C.addressof(buf), width, len(buf))
        if got < 0:
            raise PairingError(last_error())
        return [int.from_bytes(buf.raw[i:i + width], "big") for i in range(0, got, width)]

    def derived_constant_n(self, name: str, width: int, count: int):
        """the same for constants with up to `count` entries"""
        buf = C.create_string_buffer(count * width)
        got = lib.pbc_b200_derived_constant(self._h, name.encode(), C.addressof(buf), width, len(buf))
        if got < 0:
            raise PairingError(last_error())
        return [int.from_bytes(buf.raw[i:i + width], "big") for i in range(0, got, width)]

    def set_stage_profiling(self, on: bool):
        if lib.pbc_b200_set_stage_profiling(self._h, 1 if on else 0):
            raise PairingError(last_error())

    def stage_times(self):
        """ms of (main kernel, batch inversion, final exponentiation) of the last apply_device"""
        ms = (C.c_float * 3)()
        if lib.pbc_b200_stage_times(self._h, ms):
            raise PairingError(last_error())
        return list(ms)

    def bench_fpmul(self, mode: int, blocks: int, iters: int, reps: int) -> float:
        ms = lib.pbc_b200_bench_fpmul(self._h, mode, blocks, iters, reps)
        if ms < 0:
            raise PairingError(last_error())
        return ms

    def bench_fpmul_smem(self, smem_bytes: int, iters: int, reps: int) -> tuple[float, int]:
        """(ms, blocks per SM): the slot multiplier at the occupancy of smem_bytes per block, one full wave"""
        bps = C.c_int(0)
        ms = lib.pbc_b200_bench_fpmul_smem(self._h, smem_bytes, iters, reps, C.byref(bps))
        if ms < 0:
            raise PairingError(last_error())
        return ms, bps.value


class PairingPP:
    """pairing_pp_t (include/pbc_pairing.h:54-89): init once, apply many times, clear"""

    def __init__(self, pairing: Pairing, in1: bytes):
        self.pairing = pairing
        self._h = C.c_void_p()
        if lib.pbc_b200_pp_init(pairing.handle, C.byref(self._h), _addr(in1)):
            self._h = C.c_void_p()
            raise PairingError(last_error())

    def apply(self, in2: bytes, n=None) -> bytes:
        pr = self.pairing
        if n is None:
            n = len(in2) // pr.g2_len
        pr._need(in2, n * pr.g2_len, "pp apply in2")
        out = C.create_string_buffer(max(1, n * pr.gt_len))
        if lib.pbc_b200_pp_apply(self._h, C.addressof(out), _addr(in2), n):
            raise PairingError(last_error())
        return out.raw[:n * pr.gt_len]

    def apply_into(self, out, in2, n: int):
        if lib.pbc_b200_pp_apply(self._h, _addr(out), _addr(in2), n):
            raise PairingError(last_error())

    def apply_device(self, d_out, d_in2, n, stream=0):
        if lib.pbc_b200_pp_apply_device(self._h, d_out, d_in2, n, stream):
            raise PairingError(last_error())

    def clear(self):
        if getattr(self, "_h", None):
            lib.pbc_b200_pp_clear(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.clear()
        except Exception:
            pass


def pairing_init_set_str(param_text) -> Pairing:
    return Pairing(param_text)


def kernel_launches() -> int:
    return int(lib.pbc_b200_kernel_launches())


def bench_imad(blocks: int, threads: int, iters: int, reps: int) -> float:
    ms = lib.pbc_b200_bench_imad(blocks, threads, iters, reps)
    if ms < 0:
        raise PairingError(last_error())
    return ms

"""ctypes binding of libpbc_b200.so (the C ABI declared in include/pbc_b200.h).

There is deliberately no fallback: if the CUDA library has not been built (python
__graft_entry__.py) importing this module raises.
"""
from __future__ import annotations
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
# PBC_B200_LIB selects another build of the SAME library: A/B kernel variants on the GPU, and
# the test suite's CPU simulator of it (tests/host/, never shipped or installed).  Nothing in the
# product sets it; a simulator is refused unless the caller says it is a test (below).
LIB_PATH = os.environ.get("PBC_B200_LIB") or os.path.join(_HERE, "libpbc_b200.so")

if not os.path.exists(LIB_PATH):
    raise ImportError(
        "pbc_b200: %s is missing -- build it with `python __graft_entry__.py` (nvcc, sm_90a). "
        "There is no CPU fallback." % LIB_PATH)

lib = C.CDLL(LIB_PATH)
IS_SIMULATOR = hasattr(lib, "pbc_b200_sim_live_threads")
if IS_SIMULATOR and not os.environ.get("PBC_B200_LIB"):
    raise ImportError("pbc_b200: %s is the test suite's CPU simulator, not the CUDA library" % LIB_PATH)

_P = C.c_void_p
lib.pbc_b200_pairing_init_set_buf.argtypes = [C.POINTER(_P), C.c_char_p, C.c_size_t]
lib.pbc_b200_pairing_init_set_str.argtypes = [C.POINTER(_P), C.c_char_p]
lib.pbc_b200_pairing_clear.argtypes = [_P]
lib.pbc_b200_pairing_clear.restype = None
for _n in ("G1", "G2", "GT"):
    getattr(lib, "pbc_b200_pairing_length_in_bytes_" + _n).argtypes = [_P]
lib.pbc_b200_pairing_type.argtypes = [_P]
lib.pbc_b200_pairings_apply.argtypes = [_P, _P, _P, _P, C.c_size_t]
lib.pbc_b200_pairings_apply_device.argtypes = [_P, _P, _P, _P, C.c_size_t, _P]
lib.pbc_b200_prod_pairings_apply.argtypes = [_P, _P, _P, _P, C.c_size_t, C.c_size_t]
lib.pbc_b200_prod_pairings_apply_device.argtypes = [_P, _P, _P, _P, C.c_size_t, C.c_size_t, _P]
lib.pbc_b200_prod_pairings_apply_v.argtypes = [_P, _P, _P, _P, _P, C.c_size_t]
lib.pbc_b200_prod_pairings_apply_v_device.argtypes = [_P, _P, _P, _P, _P, C.c_size_t, _P]
lib.pbc_b200_pp_pairings_apply.argtypes = [_P, _P, _P, _P, C.c_size_t]
lib.pbc_b200_pp_pairings_apply_device.argtypes = [_P, _P, _P, _P, C.c_size_t, _P]
lib.pbc_b200_pp_init.argtypes = [_P, C.POINTER(_P), _P]
lib.pbc_b200_pp_apply.argtypes = [_P, _P, _P, C.c_size_t]
lib.pbc_b200_pp_apply_device.argtypes = [_P, _P, _P, C.c_size_t, _P]
lib.pbc_b200_pp_clear.argtypes = [_P]
lib.pbc_b200_pp_clear.restype = None
lib.pbc_b200_pairing_length_in_bytes_Zr.argtypes = [_P]
for _n in ("g1_pow_zn", "g2_pow_zn", "gt_pow_zn"):
    getattr(lib, "pbc_b200_" + _n).argtypes = [_P, _P, _P, _P, C.c_size_t]
    getattr(lib, "pbc_b200_" + _n + "_device").argtypes = [_P, _P, _P, _P, C.c_size_t, _P]
lib.pbc_b200_gt_mul.argtypes = [_P, _P, _P, _P, C.c_size_t]
lib.pbc_b200_gt_cmp.argtypes = [_P, _P, _P, _P, C.c_size_t]
lib.pbc_b200_is_almost_coddh.argtypes = [_P, _P, _P, _P, _P, _P, C.c_size_t]
lib.pbc_b200_g1_from_hash.argtypes = [_P, _P, _P, C.c_size_t, C.c_size_t]
lib.pbc_b200_g1_from_hash_device.argtypes = [_P, _P, _P, C.c_size_t, C.c_size_t, _P]
lib.pbc_b200_pairing_length_in_bytes_compressed_G1.argtypes = [_P]
lib.pbc_b200_g1_from_bytes_compressed.argtypes = [_P, _P, _P, C.c_size_t]
lib.pbc_b200_g2_from_hash.argtypes = [_P, _P, _P, C.c_size_t, C.c_size_t]
lib.pbc_b200_g2_from_hash_device.argtypes = [_P, _P, _P, C.c_size_t, C.c_size_t, _P]
lib.pbc_b200_pairing_length_in_bytes_compressed_G2.argtypes = [_P]
lib.pbc_b200_g2_from_bytes_compressed.argtypes = [_P, _P, _P, C.c_size_t]
lib.pbc_b200_set_devices.argtypes = [_P, C.c_int]
lib.pbc_b200_host_alloc.argtypes = [C.c_size_t]
lib.pbc_b200_host_alloc.restype = _P
lib.pbc_b200_host_free.argtypes = [_P]
lib.pbc_b200_host_free.restype = None
lib.pbc_b200_kernel_launches.restype = C.c_uint64
lib.pbc_b200_last_error.restype = C.c_char_p
lib.pbc_b200_bench_fpmul.argtypes = [_P, C.c_int, C.c_int, C.c_int, C.c_int]
lib.pbc_b200_bench_fpmul.restype = C.c_double
lib.pbc_b200_bench_fpmul_smem.argtypes = [_P, C.c_int, C.c_int, C.c_int, C.POINTER(C.c_int)]
lib.pbc_b200_bench_fpmul_smem.restype = C.c_double
lib.pbc_b200_bench_imad.argtypes = [C.c_int, C.c_int, C.c_int, C.c_int]
lib.pbc_b200_bench_imad.restype = C.c_double
lib.pbc_b200_set_stage_profiling.argtypes = [_P, C.c_int]
lib.pbc_b200_stage_times.argtypes = [_P, C.POINTER(C.c_float)]
lib.pbc_b200_derived_constant.argtypes = [_P, C.c_char_p, _P, C.c_size_t, C.c_size_t]
lib.pbc_b200_tower_op.argtypes = [_P, C.c_int, _P, _P, _P, C.c_size_t]
lib.pbc_b200_fp_op.argtypes = [_P, C.c_int, _P, _P, _P, C.c_size_t]


def last_error() -> str:
    return (lib.pbc_b200_last_error() or b"").decode()

"""Generate tests/golden/e.json, e_s510.json and e_s513.json for type E (k = 1) from the compiled,
unmodified reference (oracle/_ref), seeded.

Run next to the reference sources:  make -C oracle && python tests/golden/make_e_golden.py
  e       param/e.param (1020-bit q, sign1 = +1, sign0 = +1)
  e_s510  pbc_param_init_e_gen(160, 512) after srand(1): 510-bit q, sign1 = +1, sign0 = -1
  e_s513  the sixth set of the same sequence (srand(2) .. srand(6) before the 2nd .. 6th call, one
          pbc seed 1 for all six): 513-bit q (65-byte coordinates), sign1 = -1, sign0 = -1
Each fixture carries the sections of the d_wide_*.json files except hash and compressed (type E has
neither on the GPU) and embeds its parameter text.  All byte strings are the reference wire format
(element_to_bytes), hex-encoded.
"""
import ctypes as C
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle import ref as R  # noqa: E402

SEED = 20261016
PARAM_DIR = os.environ.get("PBC_PARAM_DIR", "/root/reference/param")
N_SINGLE = 12
PROD = (4, 3)   # (k, n_out)


def chunks(b, n):
    return [b[i:i + n].hex() for i in range(0, len(b), n)]


# struct pbc_param_interface_s / struct pbc_param_s of the reference's public header include/pbc_param.h:
# pbc_param_out_str and pbc_param_clear are static inline there, so they are restated on these two structs
_OUT_STR = C.CFUNCTYPE(None, C.c_void_p, C.c_void_p)
_CLEAR = C.CFUNCTYPE(None, C.c_void_p)


class _ParamInterface(C.Structure):
    _fields_ = [("clear", _CLEAR), ("init_pairing", C.c_void_p), ("out_str", _OUT_STR)]


class _Param(C.Structure):
    _fields_ = [("api", C.POINTER(_ParamInterface)), ("data", C.c_void_p)]


def generated_params(count):
    """The texts pbc_param_init_e_gen(160, 512) writes after srand(1), .., srand(count), in one
    sequence after pbc seed 1."""
    L = R._lib()
    libc = C.CDLL("libc.so.6")
    libc.fopen.restype = C.c_void_p
    libc.fopen.argtypes = [C.c_char_p, C.c_char_p]
    libc.fclose.argtypes = [C.c_void_p]
    L.pbc_param_init_e_gen.argtypes = [C.POINTER(_Param), C.c_int, C.c_int]
    L.pbcref_seed(1)
    texts = []
    for srand_seed in range(1, count + 1):
        libc.srand(srand_seed)
        par = _Param()
        L.pbc_param_init_e_gen(C.byref(par), 160, 512)
        path = os.path.join(os.environ.get("TMPDIR", "/tmp"), "e_gen_%d_%d.param" % (os.getpid(), srand_seed))
        f = libc.fopen(path.encode(), b"w")
        par.api.contents.out_str(f, par.data)               # pbc_param_out_str
        libc.fclose(f)
        par.api.contents.clear(par.data)                     # pbc_param_clear
        with open(path) as fh:
            texts.append(fh.read())
        os.unlink(path)
    return texts


def fixture(name, text, source):
    rp = R.RefPairing(text)
    R.RefPairing.seed(SEED)
    n = N_SINGLE
    P = rp.random(R.G1, n)
    Q = rp.random(R.G2, n)
    E = rp.pairing(P, Q, n)
    k, n_out = PROD
    PP = rp.random(R.G1, k * n_out)
    QQ = rp.random(R.G2, k * n_out)
    EP = rp.prod_pairing(PP, QQ, k, n_out)
    EPP = rp.pp_pairing(P[:rp.g1_len], Q, 4)
    a = rp.random(R.ZR, 4)
    Pa = rp.pow_zn(R.G1, P[:4 * rp.g1_len], a, 4)
    Ea = rp.pairing(Pa, Q[:4 * rp.g2_len], 4)
    Qa = rp.pow_zn(R.G2, Q[:4 * rp.g2_len], a, 4)
    Eaa = rp.pairing(Pa, Qa, 4)
    Ga = rp.pow_zn(R.GT, E[:4 * rp.gt_len], a, 4)
    Gm = rp.mul(R.GT, E[:4 * rp.gt_len], E[4 * rp.gt_len:8 * rp.gt_len], 4)
    badP = bytes([P[0] ^ 1]) + P[1:rp.g1_len]
    badQ = Q[:rp.g2_len - 1] + bytes([Q[rp.g2_len - 1] ^ 1])
    e_badP = rp.pairing(badP, Q[:rp.g2_len], 1)
    e_badQ = rp.pairing(P[:rp.g1_len], badQ, 1)
    assert rp.is_identity(R.GT, e_badP) and rp.is_identity(R.GT, e_badQ)
    return {
        "source": "oracle/_ref/libpbcref.so (unmodified reference), pbc_random_set_deterministic(%d)" % SEED,
        "param": name,
        "param_source": source,
        "param_text": text,
        "lengths": {"g1": rp.g1_len, "g2": rp.g2_len, "gt": rp.gt_len, "zr": rp.zr_len},
        "pairing": {"P": chunks(P, rp.g1_len), "Q": chunks(Q, rp.g2_len), "e": chunks(E, rp.gt_len)},
        "prod": {"k": k, "P": chunks(PP, rp.g1_len), "Q": chunks(QQ, rp.g2_len), "e": chunks(EP, rp.gt_len)},
        "pp": {"P": P[:rp.g1_len].hex(), "e": chunks(EPP, rp.gt_len)},
        "pow": {"a": chunks(a, rp.zr_len), "Pa": chunks(Pa, rp.g1_len), "e_Pa_Q": chunks(Ea, rp.gt_len),
                "Qa": chunks(Qa, rp.g2_len), "e_Pa_Qa": chunks(Eaa, rp.gt_len), "ea": chunks(Ga, rp.gt_len)},
        "gt_mul": {"e0_e4": chunks(Gm, rp.gt_len)},
        "offcurve": {"badP": badP.hex(), "badQ": badQ.hex(), "identity": e_badP.hex()},
    }


def main():
    gen = generated_params(6)
    sets = {
        "e": (open(os.path.join(PARAM_DIR, "e.param")).read(), "param/e.param"),
        "e_s510": (gen[0], "pbc_param_init_e_gen(160, 512), 1st of a sequence after srand(1..6), pbc seed 1"),
        "e_s513": (gen[5], "pbc_param_init_e_gen(160, 512), 6th of a sequence after srand(1..6), pbc seed 1"),
    }
    for name, (text, source) in sets.items():
        doc = fixture(name, text, source)
        with open(os.path.join(ROOT, "tests", "golden", name + ".json"), "w") as f:
            json.dump(doc, f, indent=0)
        print(name, "ok", doc["lengths"])


if __name__ == "__main__":
    main()

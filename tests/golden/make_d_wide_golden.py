"""Generate tests/golden/d_wide_<name>.json for the type D (MNT, k = 6) parameter sets with 160- to
255-bit q, from the compiled, unmodified reference (oracle/_ref), seeded.

Run next to the reference sources:  make -C oracle && python tests/golden/make_d_wide_golden.py
Each fixture carries the same sections as d159.json and embeds the parameter text it was drawn with
(data: the tests pass it to the library; pbc_b200/params.py does not list these sets).
All byte strings are the reference wire format (element_to_bytes), hex-encoded.
"""
import json
import os
import random
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle import ref as R  # noqa: E402

SEED = 20261016
PARAM_DIR = os.environ.get("PBC_PARAM_DIR", "/root/reference/param")
SETS = {"d175": "d277699-175-167.param", "d190": "d278027-190-181.param", "d196": "d105171-196-185.param",
        "d201": "d201.param", "d224": "d224.param"}
N_SINGLE = 12
PROD = (4, 3)   # (k, n_out)


def chunks(b, n):
    return [b[i:i + n].hex() for i in range(0, len(b), n)]


def main():
    only = sys.argv[1:]
    for name, fname in SETS.items():
        if only and name not in only:
            continue
        text = open(os.path.join(PARAM_DIR, fname)).read()
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
        Ga = rp.pow_zn(R.GT, E[:4 * rp.gt_len], a, 4)           # e(P, Q)^a in GT
        Gm = rp.mul(R.GT, E[:4 * rp.gt_len], E[4 * rp.gt_len:8 * rp.gt_len], 4)
        badP = bytes([P[0] ^ 1]) + P[1:rp.g1_len]
        badQ = Q[:rp.g2_len - 1] + bytes([Q[rp.g2_len - 1] ^ 1])
        e_badP = rp.pairing(badP, Q[:rp.g2_len], 1)
        e_badQ = rp.pairing(P[:rp.g1_len], badQ, 1)
        assert rp.is_identity(R.GT, e_badP) and rp.is_identity(R.GT, e_badQ)
        doc = {
            "source": "oracle/_ref/libpbcref.so (unmodified reference), pbc_random_set_deterministic(%d)" % SEED,
            "param": name,
            "param_file": fname,
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
        rnd = random.Random(SEED)
        doc["hash"] = {}
        for ln in (20, 32, 70, 3):
            data = [bytes(rnd.randrange(256) for _ in range(ln)) for _ in range(6)]
            H = rp.from_hash(R.G1, b"".join(data), ln, len(data))
            doc["hash"][str(ln)] = {"data": [d.hex() for d in data], "G1": chunks(H, rp.g1_len)}
        nc = 8
        comp = rp.compress(R.G1, P[:nc * rp.g1_len], nc)
        clen = len(comp) // nc
        flipped = b"".join(comp[i * clen:(i + 1) * clen - 1] + bytes([comp[(i + 1) * clen - 1] ^ 1])
                           for i in range(nc))
        doc["compressed"] = {"len": clen, "G1": chunks(comp, clen),
                             "G1_flipped_sign": chunks(rp.decompress(R.G1, flipped, nc), rp.g1_len)}
        with open(os.path.join(ROOT, "tests", "golden", "d_wide_%s.json" % name), "w") as f:
            json.dump(doc, f, indent=0)
        print(name, "ok")


if __name__ == "__main__":
    main()

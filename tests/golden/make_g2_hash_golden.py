"""Generate tests/golden/g2_hash.json: element_from_hash and compressed points on G2 from the compiled,
unmodified reference (oracle/_ref), seeded, for a, f, d159, g149 and the five type D sets with 160- to
255-bit q.

Run next to the reference sources:  make -C oracle && python tests/golden/make_g2_hash_golden.py
Per set: hashes of lengths 1, 2, 3, wb - 1, wb, wb + 1, 2 wb, 2 wb + 1 and 70 (wb = bytes of q), random G2
points with their compressed form and the same with the sign byte flipped, and for the twists the points
with y = 0 (x a root of x^3 + a'x + b', found by tests/small_order_points.py; the reference decompresses
them).  All byte strings are the reference wire format, hex-encoded.
"""
import json
import os
import random
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle import ref as R  # noqa: E402
from oracle import pbc_oracle as O  # noqa: E402
from tests import live_reference as L  # noqa: E402
from tests import small_order_points as S  # noqa: E402

SEED = 20261018
SETS = ("a", "f", "d159", "g149") + L.WIDE_D
EXT_DEGREE = {"f": 2, "d": 3, "g": 5}
PER_LENGTH = 3
N_POINTS = 6


def chunks(b, n):
    return [b[i:i + n].hex() for i in range(0, len(b), n)]


def main():
    doc = {"source": "oracle/_ref/libpbcref.so (unmodified reference), pbc_random_set_deterministic(%d)" % SEED,
           "sets": {}}
    for name in SETS:
        info = L.SetInfo(name)
        rp = R.RefPairing(info.text)
        R.RefPairing.seed(SEED)
        rnd = random.Random("%s/%d" % (name, SEED))
        wb = info.count
        ent = {"compressed_len": rp.g2_len // 2 + 1, "hash": {}}
        for length in sorted({1, 2, 3, wb - 1, wb, wb + 1, 2 * wb, 2 * wb + 1, 70}):
            data = bytes(rnd.getrandbits(8) for _ in range(PER_LENGTH * length))
            ent["hash"][str(length)] = {"data": chunks(data, length),
                                        "G2": chunks(rp.from_hash(R.G2, data, length, PER_LENGTH), rp.g2_len)}
        pts = rp.random(R.G2, N_POINTS)
        comp = rp.compress(R.G2, pts, N_POINTS)
        clen = len(comp) // N_POINTS
        flipped = b"".join(comp[i:i + clen - 1] + bytes([1 - comp[i + clen - 1]]) for i in range(0, len(comp), clen))
        ent["compressed"] = {"points": chunks(pts, rp.g2_len), "G2": chunks(comp, clen),
                             "G2_flipped_sign": chunks(flipped, clen),
                             "points_flipped": chunks(rp.decompress(R.G2, flipped, N_POINTS), rp.g2_len)}
        if info.type in EXT_DEGREE:
            orc = O.pairing_from_param(info.text)
            K = orc.Et.K
            ent["y_zero"] = []
            for T in S.two_torsion(orc.Et, info.q ** EXT_DEGREE[info.type], rnd):
                c = K.to_bytes(T[0]) + b"\1"
                got = rp.decompress(R.G2, c, 1)
                assert got == orc.Et.to_bytes(T), name
                ent["y_zero"].append({"compressed": c.hex(), "point": got.hex()})
        doc["sets"][name] = ent
        rp.close()
        print(name, "ok", file=sys.stderr)
    with open(os.path.join(ROOT, "tests", "golden", "g2_hash.json"), "w") as f:
        json.dump(doc, f, indent=1)
        f.write("\n")


if __name__ == "__main__":
    main()

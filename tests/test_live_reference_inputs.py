"""The generators of tests/live_reference.py make what they claim (Python integers and the oracle), and
tests/test_gpu_live_reference.py runs at reduced sizes on the CPU simulator of the library
(tests/host/make_host_sim.py, make_host_sim_d_wide.py for the eight-limb type D sets)."""
import os
import random
import shutil
import subprocess
import sys

import pytest

from tests import live_reference as L
from tests.type_e_model import mul

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HOST = os.path.join(ROOT, "tests", "host")


def _ref_or_skip(name, seed=5):
    if not os.path.exists(L.REF_LIB):
        pytest.skip(L.ref_missing_message())
    return L.open_ref(name, seed)


@pytest.mark.parametrize("name", L.SETS)
def test_off_subgroup_points_are_on_the_curve_and_outside_g1(name):
    info = L.SetInfo(name)
    with _ref_or_skip(name) as ref:
        pts = L.off_subgroup_points(info, ref, random.Random(name), 3)
    if info.cofactor == 1:
        assert pts == []            # E(F_q) = G1: there is nothing outside it
        return
    assert len(pts) == 3
    for p in pts:
        x, y = info.coords(p)
        assert x < info.q and 0 < y < info.q and (y * y - info.rhs(x)) % info.q == 0
        assert mul(info.r, (x, y), info.a, info.q) is not None, (name, "r P = O")


@pytest.mark.parametrize("name", L.SETS)
def test_gt_field_elements_lie_outside_gt_and_non_canonical_ones_fit(name):
    info = L.SetInfo(name)
    with _ref_or_skip(name) as ref:
        gt_len = ref.gt_len
    k = gt_len // info.wb
    els = L.gt_field_elements(info, random.Random(name), k, 6)
    assert all(len(e) == gt_len for e in els)
    assert els[6] == bytes(gt_len) and info.coords(els[7]) == [1] + [0] * (k - 1)
    for e in els[8:]:
        cs = info.coords(e)
        assert any(c >= info.q for c in cs)
        assert all(c < 1 << (8 * info.wb) and (c < info.q or c % info.q != 0) for c in cs)
    if k == 1:                      # GT in F_q^* (type e): x^r != 1 for a random x
        for e in els[:6]:
            assert pow(info.coords(e)[0], info.r, info.q) != 1


@pytest.mark.parametrize("name", L.SETS)
def test_gt_field_elements_lie_outside_gt_by_the_reference(name):
    """x^r != 1 in the reference's own GT field, every set: x * x^(r-1) is not the identity"""
    from oracle.ref import GT
    info = L.SetInfo(name)
    with _ref_or_skip(name) as ref:
        k = ref.gt_len // info.wb
        els = L.gt_field_elements(info, random.Random(name), k, 6)[:6]
        rm1 = L.scalar_bytes(info, [info.r - 1] * len(els))
        x = b"".join(els)
        xr = ref.mul(GT, x, ref.pow_zn(GT, x, rm1, len(els)), len(els))
        one = info.from_coords([1] + [0] * (k - 1))
        assert all(e != one for e in L.split(xr, ref.gt_len)), name


def test_gt_field_elements_outside_gt_in_the_extension_fields():
    """x^r != 1 in F_q^2 (types a, a1: i^2 = -1) for the random elements"""
    for name in ("a", "a1"):
        info = L.SetInfo(name)
        q = info.q
        for e in L.gt_field_elements(info, random.Random(name), 2, 6)[:6]:
            a0, a1 = info.coords(e)

            def m(u, v):
                return ((u[0] * v[0] - u[1] * v[1]) % q, (u[0] * v[1] + u[1] * v[0]) % q)
            acc, b, k = (1, 0), (a0, a1), info.r
            while k:
                if k & 1:
                    acc = m(acc, b)
                b, k = m(b, b), k >> 1
            assert acc != (1, 0)


@pytest.mark.parametrize("name", L.SETS)
def test_non_canonical_encodings_fit_and_are_never_zero(name):
    info = L.SetInfo(name)
    with _ref_or_skip(name) as ref:
        P, Q = L.random_pairs(ref, 8)
        g1, g2 = ref.g1_len, ref.g2_len
    made = 0
    for e in L.split(P, g1) + L.split(Q, g2):
        v = L.non_canonical(info, e)
        if v is None:
            continue
        made += 1
        for a, b in zip(info.coords(e), info.coords(v)):
            assert b < 1 << (8 * info.wb) and b % info.q == a % info.q
            assert b == a or (b == a + info.q and a != 0)
    assert made > 0, name


@pytest.mark.parametrize("name", L.SETS)
def test_scalars_lie_where_claimed(name):
    info = L.SetInfo(name)
    ks = L.scalars(info, random.Random(name), 40)
    top = (1 << (8 * info.zlen)) - 1
    assert all(0 <= k <= top for k in ks)
    assert max(ks[:40]) > info.r              # random ones reach above r
    r1, r0, r2, big, ones, zero = ks[40:]
    assert (r1, r0, r2, ones, zero) == (info.r - 1, info.r, info.r + 1, top, 0)
    assert big % info.r == 0 and big <= top < big + info.r
    assert len(L.scalar_bytes(info, ks)) == info.zlen * len(ks)


def _mpz_from_hash_spelled_out(q, data):
    """pbc_mpz_from_hash, arith/field.c:643-668, as a byte loop"""
    count = (q.bit_length() + 7) // 8
    buf = bytearray()
    counter = 0
    while len(buf) < count:
        for b in data:
            if len(buf) == count:
                break
            buf.append(b)
        if len(buf) == count:
            break
        buf.append(counter)
        counter += 1
    z, j = int.from_bytes(buf, "big"), 0
    while z > q:
        z, j = z >> 1, j + 1
    return z, j


@pytest.mark.parametrize("name", L.SETS)
def test_hash_data_makes_the_intended_values_and_halvings(name):
    info = L.SetInfo(name)
    rnd = random.Random(name)
    lengths = L.hash_data_by_length(info, rnd, 2)
    assert sorted(lengths) == list(range(1, 2 * info.count + 3))
    for length, data in lengths.items():
        assert len(data) == 2 * length
        for i in range(2):
            d = data[i * length:(i + 1) * length]
            assert L.mpz_from_hash(info.q, d) == _mpz_from_hash_spelled_out(info.q, d)
    got = {lab: L.mpz_from_hash(info.q, d) for lab, d in L.hash_data_by_value(info, rnd)}
    assert len(got) == 6
    top = (1 << (8 * info.count)) - 1
    want = {"0": 0, "1": 1, "q-1": info.q - 1, "q": info.q, "q+1": (info.q + 1) >> 1}
    for lab, v in want.items():
        assert got[lab][0] == v, (lab, got[lab])
    assert got["ones"][1] == L.max_halvings(info)
    assert L.max_halvings(info) in (8 * info.count - info.q.bit_length(), 8 * info.count - info.q.bit_length() + 1)
    seen = set()
    for j, d in L.hash_data_by_halvings(info, rnd):
        z, h = _mpz_from_hash_spelled_out(info.q, d)
        assert h == j and z <= info.q
        seen.add(j)
    assert seen == set(range(L.max_halvings(info) + 1))


@pytest.mark.parametrize("name", [s for s in L.SETS if s != "e"])
def test_decompression_inputs(name):
    info = L.SetInfo(name)
    items = L.decompression_inputs(info, random.Random(name), 8)
    labels = {lab for lab, _ in items}
    assert {"random", "x+q", "sign2", "sign255"} <= labels, labels
    for lab, d in items:
        assert len(d) == info.wb + 1
        x = int.from_bytes(d[:info.wb], "big")
        assert info.legendre(info.rhs(x)) == 1            # a point with y != 0 exists
        if lab == "x+q":
            assert info.q <= x < 1 << (8 * info.wb) and x % info.q != 0
        else:
            assert x < info.q
        if lab.startswith("sign"):
            assert d[-1] == int(lab[4:])
        else:
            assert d[-1] in (0, 1)


# ---- the GPU file at reduced sizes on the CPU simulator -------------------------------------------

def _sim(tmp, script):
    if not shutil.which("g++"):
        pytest.skip("no g++")
    cpp, so = str(tmp / "host_sim.cpp"), str(tmp / "libpbc_b200_sim.so")
    subprocess.check_call([sys.executable, os.path.join(HOST, script), cpp])
    subprocess.check_call(["g++", "-O1", "-std=c++17", "-shared", "-fPIC", "-Wno-unknown-pragmas", "-pthread",
                           "-o", so, cpp])
    return so


def _run_gpu_file(so, selection, min_passed, name="test_gpu_live_reference.py"):
    if not os.path.exists(L.REF_LIB):
        pytest.skip(L.ref_missing_message())
    env = dict(os.environ)
    env["PBC_B200_LIB"] = so
    env["PBC_LIVE_REFERENCE_REDUCED"] = "1"
    env["PYTHONPATH"] = ROOT + os.pathsep + env.get("PYTHONPATH", "")
    # the _device forms take torch.cuda tensors: without a CUDA device the reduced run leaves them out
    cmd = [sys.executable, "-m", "pytest", "-q", "-m", "gpu", "-p", "no:cacheprovider"]
    cmd += ["-k", selection, os.path.join(ROOT, "tests", name)]
    try:
        import xdist  # noqa: F401
        cmd += ["-n", str(max(1, min(8, len(os.sched_getaffinity(0)))))]
    except Exception:
        pass
    out = subprocess.run(cmd, env=env, capture_output=True, text=True, timeout=3000, cwd=ROOT)
    assert out.returncode == 0, out.stdout[-4000:]
    tail = out.stdout.strip().splitlines()[-1]
    assert int(tail.split(" passed")[0].split()[-1]) >= min_passed, tail


def test_live_reference_file_on_the_simulator(tmp_path):
    so = _sim(tmp_path, "make_host_sim.py")
    sel = " or ".join("%s_set" % s for s in ("a", "a1", "e", "f", "d159", "g149"))
    sel += " or sharing or zero_gt or (outside_g1 and (d159 or a1))"
    _run_gpu_file(so, sel, 50)


def test_live_reference_file_on_the_eight_limb_simulator(tmp_path):
    so = _sim(tmp_path, "make_host_sim_d_wide.py")
    sel = " or ".join("%s_set" % s for s in L.WIDE_D)
    sel += " or (outside_g1 and (%s))" % " or ".join(s for s in L.WIDE_D if s != "d224")
    _run_gpu_file(so, sel, 40)


def test_small_order_pairings_file_on_the_simulator(tmp_path):
    so = _sim(tmp_path, "make_host_sim.py")
    sel = " or ".join("%s_set" % s for s in ("a", "d159", "g149", "f")) + " or sharing"
    _run_gpu_file(so, sel, 18, "test_gpu_small_order_pairings.py")


def test_small_order_pairings_file_on_the_eight_limb_simulator(tmp_path):
    so = _sim(tmp_path, "make_host_sim_d_wide.py")
    _run_gpu_file(so, "d190_set or d201_set", 8, "test_gpu_small_order_pairings.py")

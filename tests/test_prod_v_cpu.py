"""Products with a pair count per output (pbc_b200_prod_pairings_apply_v) without a GPU:
  - the GPU tests of tests/test_gpu_prod_v.py, unchanged and at reduced size (PBC_PROD_V_REDUCED=1), on
    the CPU simulator of the library (tests/host/make_host_sim.py) for a, a1, e, f, d159 and g149, and on
    the simulator with the eight-limb type D instance (make_host_sim_d_wide.py) for d201;
  - the argument checks of the built library, which fail before any CUDA call;
  - the multi-device split of pbc_b200.sharding.shard_bounds_v;
  - the SASS of the new type A kernel: no local memory, as tests/test_sass_local_memory.py pins for
    the other type A kernels."""
import ctypes as C
import os
import random
import re
import shutil
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HOST = os.path.join(ROOT, "tests", "host")
LIB = os.path.join(ROOT, "pbc_b200", "libpbc_b200.so")


def _sim(tmp, script):
    if not shutil.which("g++"):
        pytest.skip("no g++")
    cpp, so = str(tmp / "host_sim.cpp"), str(tmp / "libpbc_b200_sim.so")
    subprocess.check_call([sys.executable, os.path.join(HOST, script), cpp])
    subprocess.check_call(["g++", "-O1", "-std=c++17", "-shared", "-fPIC", "-Wno-unknown-pragmas", "-pthread",
                           "-o", so, cpp])
    return so


def _run_gpu_file(so, names):
    """the tests of tests/test_gpu_prod_v.py for the sets `names`, by node id; returns the number passed"""
    env = dict(os.environ)
    env["PBC_B200_LIB"] = so
    env["PBC_PROD_V_REDUCED"] = "1"
    env["PYTHONPATH"] = ROOT + os.pathsep + env.get("PYTHONPATH", "")
    f = os.path.join("tests", "test_gpu_prod_v.py")
    ids = ["%s::test_random_lengths_with_special_inputs_against_the_reference[%s_set]" % (f, n) for n in names]
    for t in ("test_lengths_around_every_pass_boundary_in_one_call", "test_bad_input_turns_only_its_own_product_into_one",
              "test_many_random_lengths_equal_grouped_uniform_calls"):
        ids += ["%s::%s[%s]" % (f, t, n) for n in names]
    ids += ["%s::test_one_long_product_of_cancelling_pairs[%s]" % (f, n) for n in names if n in ("a", "f", "d159", "g149")]
    cmd = [sys.executable, "-m", "pytest", "-q", "-m", "gpu", "-p", "no:cacheprovider"] + ids
    try:
        import xdist  # noqa: F401
        cmd += ["-n", str(max(1, min(8, len(os.sched_getaffinity(0)))))]
    except Exception:
        pass
    out = subprocess.run(cmd, env=env, capture_output=True, text=True, timeout=3000, cwd=ROOT)
    tail = out.stdout.strip().splitlines()[-1] if out.stdout.strip() else out.stderr[-500:]
    assert out.returncode == 0, out.stdout[-3000:]
    passed = int(tail.split(" passed")[0].split()[-1])
    assert passed == len(ids), tail


def _ref_built():
    if not os.path.exists(os.path.join(ROOT, "oracle", "_ref", "libpbcref.so")):
        pytest.skip("oracle/_ref not built")


def test_gpu_file_on_the_simulator(tmp_path):
    _ref_built()
    _run_gpu_file(_sim(tmp_path, "make_host_sim.py"), ("a", "a1", "e", "f", "d159", "g149"))


def test_gpu_file_on_the_eight_limb_simulator(tmp_path):
    _ref_built()
    _run_gpu_file(_sim(tmp_path, "make_host_sim_d_wide.py"), ("d201",))


# ---- argument checks of the built library ---------------------------------------------------------

@pytest.fixture(scope="module")
def lib():
    if not os.path.exists(LIB):
        pytest.skip("library not built")
    if ROOT not in sys.path:
        sys.path.insert(0, ROOT)
    from pbc_b200.pairing import Pairing
    from pbc_b200.params import PARAMS
    from pbc_b200 import _lib
    return _lib, Pairing(PARAMS["f"])


def _call(lib, pr, offs, n_out, device=False):
    L, _ = lib
    arr = None if offs is None else (C.c_size_t * len(offs))(*offs)
    buf = C.create_string_buffer(64)
    if device:
        rc = L.lib.pbc_b200_prod_pairings_apply_v_device(pr.handle, buf, buf, buf, arr, n_out, None)
    else:
        rc = L.lib.pbc_b200_prod_pairings_apply_v(pr.handle, buf, buf, buf, arr, n_out)
    return rc, L.last_error()


@pytest.mark.parametrize("device", (False, True))
def test_offsets_are_checked_before_any_device_call(lib, device):
    _, pr = lib
    assert _call(lib, pr, None, 0, device)[0] == 0                        # n_out = 0: nothing to do
    rc, msg = _call(lib, pr, None, 2, device)
    assert rc and "NULL" in msg
    rc, msg = _call(lib, pr, [1, 2, 3], 2, device)
    assert rc and "offsets[0]" in msg
    rc, msg = _call(lib, pr, [0, 2, 2, 5], 3, device)
    assert rc and "offsets[2]" in msg
    rc, msg = _call(lib, pr, [0, 3, 1], 2, device)
    assert rc and "offsets[2]" in msg
    big = (1 << 64) - 1
    rc, msg = _call(lib, pr, [0, big // 8], 1, device)
    assert rc and "overflow" in msg


def test_python_offsets_are_checked(lib):
    from pbc_b200.pairing import PairingError
    _, pr = lib
    for bad in ([], [0, -1], [0, 1.5]):
        with pytest.raises(ValueError):
            pr.prod_apply_v(b"", b"", bad)
    with pytest.raises(ValueError):
        pr.prod_apply_v(b"\0" * pr.g1_len, b"\0" * pr.g2_len, [0, 2])     # two pairs, one given
    with pytest.raises(PairingError):
        pr.prod_apply_v(b"\0" * pr.g1_len, b"\0" * pr.g2_len, [0, 1, 1])
    assert pr.prod_apply_v(b"", b"", [0]) == b""


# ---- sharding ------------------------------------------------------------------------------------

@pytest.mark.parametrize("world", (1, 2, 3, 8))
def test_shard_bounds_v_cover_and_balance(world):
    if ROOT not in sys.path:
        sys.path.insert(0, ROOT)
    from pbc_b200.sharding import shard_bounds_v, shard_inputs_v
    rnd = random.Random(world)
    for _ in range(40):
        lens = [rnd.choice((1, 2, 16, 17, 300, 5000)) for _ in range(rnd.randint(1, 30))]
        off = [0]
        for n in lens:
            off.append(off[-1] + n)
        b = shard_bounds_v(off, world)
        assert len(b) == world and b[0][0] == 0 and b[-1][1] == len(lens)
        assert all(b[g][1] == b[g + 1][0] and b[g][0] <= b[g][1] for g in range(world - 1))
        total, longest = off[-1], max(lens)
        for lo, hi in b:
            assert abs((off[hi] - off[lo]) - total / world) <= longest, (lens, world, b)
        in1, in2 = bytes(range(256)) * 80, bytes(range(256)) * 160
        r = rnd.randrange(world)
        a1, a2, o = shard_inputs_v(in1[:3 * total], in2[:6 * total], off, 3, 6, r, world)
        lo, hi = b[r]
        assert o[0] == 0 and len(o) == hi - lo + 1 and o[-1] == off[hi] - off[lo]
        assert a1 == in1[3 * off[lo]:3 * off[hi]] and a2 == in2[6 * off[lo]:6 * off[hi]]


# ---- compiler output -----------------------------------------------------------------------------

def test_type_a_segmented_product_uses_no_local_memory():
    exe = shutil.which("cuobjdump") or os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "cuobjdump")
    if not os.path.exists(exe):
        pytest.skip("no cuobjdump")
    if not os.path.exists(LIB):
        pytest.skip("library not built")
    sass = subprocess.run([exe, "-sass", LIB], capture_output=True, text=True, check=True).stdout
    fn, count = None, {}
    for line in sass.splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            # k_prod_v<ProdVF2<Ops<16, true, 128>, 16>, 128>
            fn = m.group(1) if m.group(1).startswith("_ZN7pbcb2008k_prod_vINS_7ProdVF2INS_3OpsILi16ELb1E") else None
            if fn:
                count[fn] = 0
        elif fn and re.search(r"\b(LDL|STL)(\.\S+)?\s", line):
            count[fn] += 1
    assert count, "the type A segmented-product kernel is missing from the SASS"
    assert not any(count.values()), count

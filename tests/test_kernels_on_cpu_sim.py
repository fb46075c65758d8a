"""The product library -- engine.cu's host code and every kernel it launches -- compiled for the CPU
and run against the reference fixtures and the GPU parity tests themselves.

tests/host/make_host_sim.py turns engine.cu plus its headers into one C++ file: inline PTX goes
through tests/host/ptx_emul.hpp, kernel launches and the CUDA runtime through tests/host/cuda_sim.hpp
(device memory = host memory, one simulated thread at a time).  The result exports the same C ABI, so
PBC_B200_LIB=<simulator> lets pbc_b200.pairing and the `-m gpu` tests run unchanged -- the small
cases, here, without a GPU.  This pins the kernels' logic (formulas, indexing, wire conversion,
workspace layout, host-side constants); clocks, occupancy and the real PTX->SASS path are what the
GPU runs add.  TEST INFRASTRUCTURE: nothing in the product links or loads the simulator."""
import json
import os
import shutil
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HOST = os.path.join(ROOT, "tests", "host")


def _build(tmp, *defs):
    cpp, so = str(tmp / "host_sim.cpp"), str(tmp / "libpbc_b200_sim.so")
    subprocess.check_call([sys.executable, os.path.join(HOST, "make_host_sim.py"), cpp] + list(defs))
    subprocess.check_call(["g++", "-O1", "-std=c++17", "-shared", "-fPIC", "-Wno-unknown-pragmas", "-pthread",
                           "-o", so, cpp])
    return so


def _env(so):
    env = dict(os.environ)
    env["PBC_B200_LIB"] = so
    env["PYTHONPATH"] = ROOT + os.pathsep + env.get("PYTHONPATH", "")
    return env


@pytest.fixture(scope="module")
def sim(tmp_path_factory):
    if not shutil.which("g++"):
        pytest.skip("no g++")
    return _build(tmp_path_factory.mktemp("sim"))


def _battery(so, *args):
    out = subprocess.run([sys.executable, os.path.join(HOST, "sim_driver.py")] + list(args), env=_env(so),
                         capture_output=True, text=True, timeout=1800)
    assert out.returncode == 0, out.stderr[-2000:]
    return json.loads(out.stdout.strip().splitlines()[-1])


def test_every_entry_point_reproduces_the_reference_fixtures(sim):
    res = _battery(sim)
    assert len(res) >= 38 and all(res.values()), {k: v for k, v in res.items() if not v}


def test_gpu_parity_tests_pass_on_the_simulator(sim):
    """the `-m gpu` tests, unchanged, with the simulator in place of libpbc_b200.so; left out: the
    cases sized for a GPU (2^14 .. 2^18 outputs), the device-pointer entry points (they take
    torch.cuda tensors), the C programs of the shim (they link the real library) and the wide type D
    cases (tests/test_d_wide_cpu.py runs them on the eight-limb simulator)"""
    files = [os.path.join(ROOT, "tests", f) for f in ("test_gpu_towers.py", "test_gpu_type_a.py", "test_gpu_type_a1.py",
                                                       "test_gpu_type_fd.py", "test_gpu_edge_cases.py", "test_gpu_group_ops.py",
                                                       "test_gpu_zz_a1_group_ops.py", "test_gpu_small_order_powers.py",
                                                       "test_gpu_montgomery_extremes.py")]
    cmd = [sys.executable, "-m", "pytest", "-q", "-m", "gpu", "-p", "no:cacheprovider",
           "-k", "not large_batch and not device_pointer and not tiles and not across_blocks and not d_wide"] + files
    try:
        import xdist  # noqa: F401
        cmd += ["-n", str(max(1, min(8, len(os.sched_getaffinity(0)))))]
    except Exception:
        pass
    out = subprocess.run(cmd, env=_env(sim), capture_output=True, text=True, timeout=3000, cwd=ROOT)
    tail = out.stdout.strip().splitlines()[-1] if out.stdout.strip() else out.stderr[-500:]
    assert out.returncode == 0, out.stdout[-3000:]
    passed = int(tail.split(" passed")[0].split()[-1])
    assert passed >= 310, tail


def test_multiplier_work_counted_by_the_simulator_matches_bench(sim):
    """bench.py's roofline numerator (32x32 products the Miller kernel executes per pairing) against
    the count the PTX interpreter takes while running that kernel"""
    code = """
import ctypes, json, sys
sys.argv = ["bench.py"]
import bench
from pbc_b200 import _lib
from pbc_b200.pairing import Pairing
from pbc_b200.params import PARAMS
lib = _lib.lib
lib.pbc_b200_sim_products.restype = ctypes.c_ulonglong
out = {}
for wl in ("a", "a1", "f", "d", "g"):
    w = bench.WORKLOADS[wl]
    g = json.load(open("tests/golden/%s.json" % w["param"]))["pairing"]
    pr = Pairing(PARAMS[w["param"]])
    P, Q = bytes.fromhex(g["P"][0]), bytes.fromhex(g["Q"][0])
    pr.set_stage_profiling(False)
    pr.apply(P, Q, 1)                      # warm: constants resident
    c0 = lib.pbc_b200_sim_products()
    pr.apply(P, Q, 1)
    out[wl] = [lib.pbc_b200_sim_products() - c0, w["exec_unit_ops_main"] or w["exec_unit_ops_all"], bool(w["exec_unit_ops_main"])]
# products of 4 pairings with two pairs per thread sharing one Miller accumulator (bench.py's prod16 figure)
g = json.load(open("tests/golden/a.json"))["prod"]
pr = Pairing(PARAMS["a"] + chr(10) + "b200_prod_share 2" + chr(10))
P, Q = b"".join(bytes.fromhex(x) for x in g["P"][:4]), b"".join(bytes.fromhex(x) for x in g["Q"][:4])
pr.prod_apply(P, Q, 4, 1)
c0 = lib.pbc_b200_sim_products()
pr.prod_apply(P, Q, 4, 1)
out["prod_share2"] = [lib.pbc_b200_sim_products() - c0, int(4 * ((159 * 10 + 23.5) * 528 + (159 * 6 + 7) * 408)), True]
print(json.dumps(out))
"""
    out = subprocess.run([sys.executable, "-c", code], env=_env(sim), capture_output=True, text=True, timeout=900, cwd=ROOT)
    assert out.returncode == 0, out.stderr[-2000:]
    res = json.loads(out.stdout.strip().splitlines()[-1])
    for wl, (counted, claimed, miller_only) in res.items():
        if miller_only:
            # counted = the whole call (Miller loop + batch inversion of one element + final
            # exponentiation); the Miller kernel bench.py names is the bulk of it, never more
            assert claimed < counted < 1.6 * claimed, (wl, counted, claimed)
        else:
            assert counted == claimed, (wl, counted, claimed)     # types f, d, g: the whole sequence


@pytest.mark.parametrize("name", ["a", "g149", "a1_small"])
def test_pbc_api_through_the_shim_on_the_simulator(sim, tmp_path, name):
    """oracle/_ref/shim/shim_test (element_pairing, element_prod_pairing, pairing_pp_*, the batch entry
    points and element_pow_zn_batch through the reference's own pbc.h, compared inside the program
    with a pairing_t that keeps the reference's CPU vtable), the simulator standing in for
    libpbc_b200.so.  Type A1 goes through the shim here as well."""
    exe = os.path.join(ROOT, "oracle", "_ref", "shim", "shim_test")
    if not os.path.exists(exe):
        pytest.skip("oracle/_ref/shim/shim_test not built (needs the reference headers: make -C oracle shim)")
    if name == "a1_small":
        with open(os.path.join(ROOT, "tests", "golden", "a1_small.json")) as f:
            text = json.load(f)["param_text"]
    else:
        sys.path.insert(0, ROOT)
        from pbc_b200.params import PARAMS
        text = PARAMS[name]
    (tmp_path / "p.param").write_text(text)
    libdir = tmp_path / "lib"
    libdir.mkdir()
    shutil.copy(sim, str(libdir / "libpbc_b200.so"))         # RUNPATH of the program yields to LD_LIBRARY_PATH
    env = dict(os.environ)
    env["LD_LIBRARY_PATH"] = str(libdir) + os.pathsep + env.get("LD_LIBRARY_PATH", "")
    r = subprocess.run([exe, str(tmp_path / "p.param"), "24"], env=env, capture_output=True, text=True, timeout=1800)
    assert r.returncode == 0 and "shim_test: OK" in r.stdout, r.stdout[-1500:] + r.stderr[-500:]


def test_plain_c_caller_of_the_c_abi_on_the_simulator(sim, tmp_path):
    """examples/batch_pairing_demo.c (includes only include/pbc_b200.h; pinned staging buffers through
    pbc_b200_host_alloc) with the simulator standing in for libpbc_b200.so"""
    exe = os.path.join(ROOT, "examples", "_build", "batch_pairing_demo")
    if not os.path.exists(exe):
        pytest.skip("examples/_build/batch_pairing_demo not built (make -C examples)")
    sys.path.insert(0, ROOT)
    from pbc_b200.params import PARAMS
    with open(os.path.join(ROOT, "tests", "golden", "d159.json")) as f:
        g = json.load(f)["pairing"]
    (tmp_path / "p.param").write_text(PARAMS["d159"])
    (tmp_path / "P.bin").write_bytes(b"".join(bytes.fromhex(x) for x in g["P"]))
    (tmp_path / "Q.bin").write_bytes(b"".join(bytes.fromhex(x) for x in g["Q"]))
    libdir = tmp_path / "lib"
    libdir.mkdir()
    shutil.copy(sim, str(libdir / "libpbc_b200.so"))
    env = dict(os.environ)
    env["LD_LIBRARY_PATH"] = str(libdir) + os.pathsep + env.get("LD_LIBRARY_PATH", "")
    r = subprocess.run([exe, str(tmp_path / "p.param"), str(tmp_path / "P.bin"), str(tmp_path / "Q.bin"),
                        str(tmp_path / "E.bin")], env=env, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr
    assert (tmp_path / "E.bin").read_bytes() == b"".join(bytes.fromhex(x) for x in g["e"])


def test_single_process_fan_out_over_two_simulated_devices(sim):
    """pbc_b200_set_devices (SURVEY 8e, the one-process front end): one host thread and two streams
    per device, contiguous output slices written at their offset of the caller's buffer.  The
    simulator reports two devices (PBC_SIM_DEVICES=2): same bytes as one device, twice the launches."""
    code = """
import json
from pbc_b200.pairing import Pairing, kernel_launches
from pbc_b200.params import PARAMS
cat = lambda xs: b"".join(bytes.fromhex(x) for x in xs)
out = {}
for name in ("a", "f", "d159"):
    g = json.load(open("tests/golden/%s.json" % name))
    n = len(g["pairing"]["e"])
    P, Q, E = cat(g["pairing"]["P"]), cat(g["pairing"]["Q"]), cat(g["pairing"]["e"])
    pr = Pairing(PARAMS[name])
    l0 = kernel_launches(); one = pr.apply(P, Q, n); l1 = kernel_launches()
    pr.set_devices(2)
    two = pr.apply(P, Q, n); l2 = kernel_launches()
    odd = pr.apply(P, Q, n - 1)                       # uneven slices
    k, no = g["prod"]["k"], len(g["prod"]["e"])
    prod = pr.prod_apply(cat(g["prod"]["P"]), cat(g["prod"]["Q"]), k, no)
    out[name] = [one == E, two == E, odd == E[:len(odd)], prod == cat(g["prod"]["e"]), l2 - l1 == 2 * (l1 - l0)]
print(json.dumps(out))
"""
    env = _env(sim)
    env["PBC_SIM_DEVICES"] = "2"
    out = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, timeout=900, cwd=ROOT)
    assert out.returncode == 0, out.stderr[-2000:]
    res = json.loads(out.stdout.strip().splitlines()[-1])
    assert all(all(v) for v in res.values()), res

"""The reference's own C API (pbc.h) through the shim on type E (param/e.param and the 513-bit set
e_s513): the shim's vtable check (shim/shim_test.c, which compares against a second pairing_t of the
reference whose R is drawn at random) and the reference's unmodified benchmark/benchmark.c."""
import json
import os
import subprocess

import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BUILD = os.path.join(ROOT, "oracle", "_ref", "shim")


def _need(name):
    path = os.path.join(BUILD, name)
    assert os.path.exists(path), "oracle/_ref/shim/%s is missing: run `python __graft_entry__.py` where the reference sources are" % name
    return path


def _param(name):
    with open(os.path.join(ROOT, "tests", "golden", name + ".json")) as f:
        return json.load(f)["param_text"]


@pytest.mark.parametrize("name", ["e", "e_s513"])
def test_pbc_api_on_gpu_matches_reference_vtable(tmp_path, name):
    exe = _need("shim_test")
    pf = tmp_path / (name + ".param")
    pf.write_text(_param(name))
    r = subprocess.run([exe, str(pf), "200"], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "shim_test: OK" in r.stdout


@pytest.mark.parametrize("name", ["e", "e_s513"])
def test_reference_benchmark_program_runs_on_gpu(name):
    exe = _need("benchmark_b200")
    r = subprocess.run([exe], input=_param(name), capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr
    assert "BUG" not in r.stdout and "average pairing time" in r.stdout
    t = {}
    for line in r.stdout.splitlines():
        if line.startswith("average pairing time (preprocessed) ="):
            t["pp"] = float(line.split("=")[1])
        elif line.startswith("average pairing time ="):
            t["plain"] = float(line.split("=")[1])
    assert t["pp"] < t["plain"], t

"""The slot programs the Type A1 kernels run (pbc_b200/csrc/a_steps.cuh) instantiated on the CPU
with a big-integer policy class (tests/host/a_steps_host.cpp) and pinned to fixtures the compiled
reference produced: the formulas are checked here, the limb arithmetic and the plumbing on the GPU."""
import json
import os
import shutil
import subprocess

import pytest

from oracle import pbc_oracle as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def harness(tmp_path_factory):
    if not shutil.which("g++"):
        pytest.skip("no g++")
    exe = str(tmp_path_factory.mktemp("host") / "a_steps_host")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-o", exe,
                           os.path.join(ROOT, "tests", "host", "a_steps_host.cpp")])
    return exe


def _run(exe, mode, pr, pairs):
    lines = ["%d %d %d %d" % (pr.q, pr.r, pr.l, len(pairs))]
    for P, Q in pairs:
        lines.append("%d %d %d %d" % (P[0], P[1], Q[0], Q[1]))
    out = subprocess.run([exe] + mode, input="\n".join(lines) + "\n", capture_output=True, text=True,
                         timeout=600, check=True)
    res = []
    for line in out.stdout.strip().split("\n"):
        re_, im = (int(t, 16) for t in line.split())
        res.append(pr.GT.to_bytes((re_, im)).hex())
    return res


@pytest.mark.parametrize("mode", [["pp"], ["5t"], ["5t-naf"]])
def test_a1_slot_programs_reproduce_reference_pairings(harness, mode):
    with open(os.path.join(ROOT, "tests", "golden", "a1_small.json")) as f:
        g = json.load(f)
    pr = O.pairing_from_param(g["param_text"])
    pairs = [(pr.G1.from_bytes(bytes.fromhex(P)), pr.G2.from_bytes(bytes.fromhex(Q)))
             for P, Q in zip(g["pairing"]["P"], g["pairing"]["Q"])]
    assert _run(harness, mode, pr, pairs) == g["pairing"]["e"]

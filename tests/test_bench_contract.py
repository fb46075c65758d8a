"""bench.py's CPU-only legs: the reference arm (`--impl reference`) prints the contract's JSON line;
the synthetic inputs are points of the right subgroup.  The GPU arm is exercised on the H100."""
import json
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _ref_available():
    from oracle import ref
    return ref.available()


@pytest.mark.parametrize("workload", ["a", "a1"])
def test_reference_arm_prints_the_contract_line(workload):
    if not _ref_available():
        pytest.skip("oracle/_ref not built")
    out = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference", "--workload", workload,
                          "--steps", "1", "--warmup", "1", "--ref-seconds", "0.5"],
                         capture_output=True, text=True, timeout=600, check=True)
    lines = [l for l in out.stdout.splitlines() if l.startswith("{")]
    assert len(lines) == 1, out.stdout
    d = json.loads(lines[0])
    assert d["impl"] == "reference" and d["metric"] == "pairings/sec" and d["higher_is_better"] is True
    assert d["value"] > 0 and d["n_gpus"] == 1 and d["steps"] == 1 and d["gpu_launches"] == 0
    cb = d["cpu_baseline"]
    assert cb["kind"] == "reference" and cb["cores"] >= 1 and cb["value"] == d["value"]
    assert 0 < cb["effective_cores"] <= cb["cores"] * 1.05
    assert d["e2e"] == {"value": d["value"], "unit": d["unit"], "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}


def test_synthetic_a1_inputs_lie_in_the_order_n_subgroup():
    sys.path.insert(0, ROOT)
    import bench
    from oracle import pbc_oracle as O
    from pbc_b200.params import PARAMS
    w = bench.WORKLOADS["a1"]
    P, Q = bench.make_inputs(w, 3)
    pr = O.pairing_from_param(PARAMS["a1"])
    for buf in (P, Q):
        for i in range(3):
            pt = pr.G1.from_bytes(bytes(buf[i * 260:(i + 1) * 260]))
            assert pt is not None and pr.E.is_valid(pt) and pr.E.mul(pr.r, pt) is None
    assert w["exec_unit_ops_main"] == 56225715      # signed-digit scan of n (k_a1_miller, since round 2)


def test_parity_sample_is_seeded_distinct_and_reaches_the_last_chunk():
    """the index sample bench.py checks against oracle/_ref on every rank: distinct, reproducible,
    different per rank, and always containing the tail of the batch"""
    sys.path.insert(0, ROOT)
    import bench
    a = bench.sample_indices(1 << 20, 20000, 7)
    b = bench.sample_indices(1 << 20, 20000, 7)
    c = bench.sample_indices(1 << 20, 20000, 8)
    assert (a == b).all() and not (a == c).all()
    assert len(set(a.tolist())) == 20000 and a[-1] == (1 << 20) - 1 and a[-256] == (1 << 20) - 256
    assert (a[:-256] < (1 << 20) - 256).all() and a[0] >= 0
    # spread over every 2^18-output pipeline chunk of the host path
    assert all(((a >> 18) == ch).sum() > 1000 for ch in range(4))
    assert list(bench.sample_indices(5, 100, 1)) == [0, 1, 2, 3, 4]


def test_shard_sizes_follow_the_scaling_mode():
    sys.path.insert(0, ROOT)
    import bench
    W = bench.WORKLOADS
    assert bench.shard_size(W["a"], 8, "weak") == 1 << 20 and bench.shard_size(W["a"], 8, "strong") == 1 << 17
    assert bench.shard_size(W["prod16"], 8, "weak") == 1 << 13 and bench.shard_size(W["d"], 2, "weak") == 1 << 18


def test_dump_outputs_write_a_fixed_seeded_sample_per_config(tmp_path):
    """--dump-outputs: DIR/<config>.npy, float32, the rows dump_rows picks (every row of a small batch, a fixed
    seeded sample of DUMP_ROWS of a large one), and at most 64 MB over every workload bench.py knows"""
    sys.path.insert(0, ROOT)
    import numpy as np
    import bench
    assert (bench.dump_rows(100) == np.arange(100)).all()
    r = bench.dump_rows(1 << 20)
    assert len(r) == bench.DUMP_ROWS == len(set(r.tolist())) and (np.diff(r) > 0).all() and r[-1] < 1 << 20
    assert (r == bench.dump_rows(1 << 20)).all()
    assert bench.DUMP_ROWS * 4 * sum(bench.WIRE[w["param"]][2] for w in bench.WORKLOADS.values()) <= 64 << 20
    n, gt = 3 * bench.DUMP_ROWS, 120
    out = np.random.default_rng(1).integers(0, 256, size=n * gt, dtype=np.uint8)
    path = bench.write_dump(str(tmp_path), "d", out, n, gt)
    assert path == str(tmp_path / "d.npy")
    got = np.load(path)
    assert got.dtype == np.float32 and got.shape == (bench.DUMP_ROWS, gt)
    assert (got == out.reshape(n, gt)[bench.dump_rows(n)]).all()


def test_every_config_times_the_steps_asked_for():
    sys.path.insert(0, ROOT)
    import bench
    a = bench.parse_args(["--steps", "7"])
    assert bench.timed_steps(a, True) == 7 and bench.timed_steps(a, False) == 7
    b = bench.parse_args(["--steps", "7", "--extra-steps", "2", "--dump-outputs", "x"])
    assert bench.timed_steps(b, True) == 7 and bench.timed_steps(b, False) == 2 and b.dump_outputs == "x"

#!/usr/bin/env python
"""bench_e.py -- type E (param/e.param, k = 1, 1020-bit q) pairings/s on one GPU.

  python tools/bench_e.py [--n 262144] [--steps 5] [--warmup 2] [--ref-sample 16] [--sets e,e_s510,e_s513]

For every set: pairings/s with inputs resident in device memory (CUDA events around
pbc_b200_pairings_apply_device, median of --steps), end to end through the host-buffer call (median of
--steps after one warm-up call), the three
stage times (Miller loop, batch inversion, final exponentiation), the rate of a pairing_pp_t handle
(one fixed P, resident inputs), parity of a seeded sample of the outputs against oracle/_ref (the
compiled reference), and the reference's own rate on all host cores (one process per core,
--ref-sample pairings each).  Inputs are the fixture points repeated.  The card's name and power
limit are read in the same run.  One JSON line per set, then a summary.
"""
from __future__ import annotations
import argparse
import json
import multiprocessing as mp
import os
import random
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.dont_write_bytecode = True


def _card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except Exception as e:  # noqa: BLE001
        return "unknown (%s)" % e


def _ref_worker(args):
    text, P, Q, n = args
    from oracle import ref as R
    rp = R.RefPairing(text)
    t0 = time.perf_counter()
    rp.pairing(P, Q, n)
    return n, time.perf_counter() - t0


def _timed(fn, warmup, steps, stream):
    import torch
    times = []
    for it in range(warmup + steps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        fn()
        e1.record(stream)
        torch.cuda.synchronize()
        if it >= warmup:
            times.append(e0.elapsed_time(e1) / 1e3)
    return times


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=1 << 18)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--ref-sample", type=int, default=16)
    ap.add_argument("--sets", default="e")
    a = ap.parse_args()
    import torch
    from pbc_b200.pairing import Pairing
    from oracle import ref as R
    card = _card()
    results = []
    for name in a.sets.split(","):
        g = json.load(open(os.path.join(ROOT, "tests", "golden", name + ".json")))
        pr = Pairing(g["param_text"])
        P = [bytes.fromhex(x) for x in g["pairing"]["P"]]
        Q = [bytes.fromhex(x) for x in g["pairing"]["Q"]]
        n = a.n
        idx = [i % len(P) for i in range(n)]
        hP = b"".join(P[i] for i in idx)
        hQ = b"".join(Q[i] for i in idx)
        dP = torch.frombuffer(bytearray(hP), dtype=torch.uint8).cuda()
        dQ = torch.frombuffer(bytearray(hQ), dtype=torch.uint8).cuda()
        out = torch.empty(n * pr.gt_len, dtype=torch.uint8, device="cuda")
        st = torch.cuda.current_stream()
        pr.set_stage_profiling(True)
        stages = []

        def run():
            pr.apply_device(out.data_ptr(), dP.data_ptr(), dQ.data_ptr(), n, st.cuda_stream)

        times = []
        for it in range(a.warmup + a.steps):
            t = _timed(run, 0, 1, st)[0]
            if it >= a.warmup:
                times.append(t)
                stages.append(pr.stage_times())
        res = statistics.median(times)
        got = out.cpu().numpy().tobytes()
        # end to end through the host-buffer call: one warm-up call (staging buffers are allocated on first
        # use), then the median of --steps timed calls
        got_e2e = pr.apply(hP, hQ, n)
        e2e_times = []
        for _ in range(a.steps):
            t0 = time.perf_counter()
            pr.apply(hP, hQ, n)
            e2e_times.append(time.perf_counter() - t0)
        e2e = statistics.median(e2e_times)
        # pairing_pp_t handle: one fixed P against the resident Q
        h = pr.pp_init(P[0])
        pp_out = torch.empty(n * pr.gt_len, dtype=torch.uint8, device="cuda")
        pp_times = _timed(lambda: h.apply_device(pp_out.data_ptr(), dQ.data_ptr(), n, st.cuda_stream),
                          a.warmup, a.steps, st)
        pp_got = pp_out.cpu().numpy().tobytes()
        h.clear()
        rnd = random.Random(20261016)
        sample = sorted(rnd.sample(range(n), 16))
        parity = None
        if R.available():
            rp = R.RefPairing(g["param_text"])
            L = pr.gt_len
            ref = rp.pairing(b"".join(P[idx[i]] for i in sample), b"".join(Q[idx[i]] for i in sample), len(sample))
            ref_pp = rp.pairing(P[0] * len(sample), b"".join(Q[idx[i]] for i in sample), len(sample))
            parity = all(got[i * L:(i + 1) * L] == ref[j * L:(j + 1) * L] == got_e2e[i * L:(i + 1) * L]
                         and pp_got[i * L:(i + 1) * L] == ref_pp[j * L:(j + 1) * L]
                         for j, i in enumerate(sample))
        ref_rate = None
        if R.available() and a.ref_sample > 0:
            cores = len(os.sched_getaffinity(0))
            m = a.ref_sample
            job = (g["param_text"], b"".join(P[idx[i]] for i in range(m)), b"".join(Q[idx[i]] for i in range(m)), m)
            t0 = time.perf_counter()
            with mp.get_context("spawn").Pool(cores) as pool:
                done = pool.map(_ref_worker, [job] * cores)
            wall = time.perf_counter() - t0
            ref_rate = {"pairings_per_s": sum(d[0] for d in done) / max(d[1] for d in done), "cores": cores,
                        "wall_s_with_startup": wall}
        from tests.type_e_model import parse_param
        r = {"set": name, "q_bits": parse_param(g["param_text"])["q"].bit_length(), "n": n,
             "resident_pairings_per_s": n / res, "e2e_pairings_per_s": n / e2e,
             "stage_ms_median": [statistics.median(s[k] for s in stages) for k in range(3)],
             "resident_ms_all": [t * 1e3 for t in times], "e2e_ms_all": [t * 1e3 for t in e2e_times],
             "pp_handle_pairings_per_s": n / statistics.median(pp_times),
             "parity_vs_reference": parity, "reference_all_cores": ref_rate, "card": card}
        if ref_rate:
            r["resident_over_reference_all_cores"] = r["resident_pairings_per_s"] / ref_rate["pairings_per_s"]
        print(json.dumps(r), flush=True)
        results.append(r)
        pr.clear()
    print(json.dumps({"card": card, "summary": {r["set"]: round(r["resident_pairings_per_s"]) for r in results}}))


if __name__ == "__main__":
    main()

#!/usr/bin/env python
"""bench_prod_v.py -- products of pairings with a pair count per output (prod_apply_v_device) on one GPU.

  python tools/bench_prod_v.py [--steps 5] [--warmup 2] [--types a,f,d159] [--outputs 65536] [--long 262144]

Inputs are resident in device memory; every time is CUDA events around the calls, the median of --steps
after --warmup untimed runs.  Per type:
  1. equal lengths 16 at --outputs outputs: the ragged call against prod_apply_device(k = 16);
  2. lengths drawn uniformly from 1..31 at --outputs outputs: one ragged call against grouping by length
     (one uniform call per length on inputs already grouped, plus the scatter of the outputs back to
     order, on the device);
  3. one product of --long pairs against --long single pairings (apply_device), and against
     prod_apply_device(k = 2^16, n_out = 1), the uniform product's one-thread reduction.
Every configuration checks that the ragged outputs are byte-equal to the uniform or grouped ones (3: to
prod_apply_device(k = --long, n_out = 1), untimed).  Pairs are the fixture pairs of tests/golden repeated
at a stride of 29.  The card's name and power limit are read in the same run.  One JSON line per type.
"""
from __future__ import annotations
import argparse
import json
import os
import random
import statistics
import subprocess
import sys

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
            times.append(e0.elapsed_time(e1))
    return statistics.median(times)          # ms


def _offsets(lengths):
    off = [0]
    for n in lengths:
        off.append(off[-1] + n)
    return off


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--types", default="a,f,d159")
    ap.add_argument("--outputs", type=int, default=1 << 16)
    ap.add_argument("--long", type=int, default=1 << 18)
    a = ap.parse_args()
    import numpy as np
    import torch
    from pbc_b200.pairing import Pairing
    from pbc_b200.params import PARAMS
    import ctypes as C
    from pbc_b200._lib import lib
    card = _card()
    st = torch.cuda.current_stream()
    s = st.cuda_stream
    for name in a.types.split(","):
        g = json.load(open(os.path.join(ROOT, "tests", "golden", name + ".json")))
        pr = Pairing(PARAMS[name])
        gt = pr.gt_len
        Ps = [bytes.fromhex(x) for x in g["pairing"]["P"]]
        Qs = [bytes.fromhex(x) for x in g["pairing"]["Q"]]

        def pairs(m):
            P = b"".join(Ps[(29 * j) % len(Ps)] for j in range(m))
            Q = b"".join(Qs[(29 * j + j // len(Qs)) % len(Qs)] for j in range(m))
            return (torch.frombuffer(bytearray(P), dtype=torch.uint8).cuda(),
                    torch.frombuffer(bytearray(Q), dtype=torch.uint8).cuda())

        def ragged(o, p, q, off):
            """the C entry point on an offsets array converted once (no per-call Python conversion)"""
            arr = (C.c_size_t * len(off))(*[int(x) for x in off])
            return lambda: lib.pbc_b200_prod_pairings_apply_v_device(pr.handle, o.data_ptr(), p.data_ptr(), q.data_ptr(),
                                                                     arr, len(off) - 1, s)

        def out(n):
            return torch.zeros(n * gt, dtype=torch.uint8, device="cuda")

        res = {"type": name, "card": card}
        n = a.outputs
        # 1. equal lengths 16
        dP, dQ = pairs(16 * n)
        ov, ou = out(n), out(n)
        off = _offsets([16] * n)
        t_v = _timed(ragged(ov, dP, dQ, off), a.warmup, a.steps, st)
        t_u = _timed(lambda: pr.prod_apply_device(ou.data_ptr(), dP.data_ptr(), dQ.data_ptr(), 16, n, s), a.warmup, a.steps, st)
        res["equal16"] = {"outputs": n, "ragged_ms": t_v, "uniform_k16_ms": t_u, "ragged_outputs_per_s": n / t_v * 1e3,
                          "uniform_outputs_per_s": n / t_u * 1e3, "ragged_over_uniform_time": t_v / t_u,
                          "equal": bool(torch.equal(ov, ou))}
        del dP, dQ
        # 2. lengths uniform in 1..31: one ragged call against one uniform call per length
        rnd = random.Random(20261018)
        lengths = [rnd.randint(1, 31) for _ in range(n)]
        off = np.array(_offsets(lengths), dtype=np.uint64)
        dP, dQ = pairs(int(off[-1]))
        g1, g2 = pr.g1_len, pr.g2_len
        order = sorted(range(n), key=lambda i: lengths[i])                # outputs grouped by length
        src = np.concatenate([np.arange(off[i], off[i + 1]) for i in order]).astype(np.int64)
        gP = dP.view(-1, g1)[torch.from_numpy(src).cuda()].reshape(-1)   # inputs already grouped: not timed
        gQ = dQ.view(-1, g2)[torch.from_numpy(src).cuda()].reshape(-1)
        groups, o = [], 0
        for k in sorted(set(lengths)):
            cnt = lengths.count(k)
            groups.append((k, cnt, o))
            o += cnt
        perm = torch.tensor(order, dtype=torch.int64, device="cuda")
        ov, og, ogs = out(n), out(n), out(n)
        pos = {}
        acc = 0
        for k, cnt, first in groups:
            pos[k] = acc
            acc += k * cnt

        def grouped():
            for k, cnt, first in groups:
                pr.prod_apply_device(og.data_ptr() + first * gt, gP.data_ptr() + pos[k] * g1,
                                     gQ.data_ptr() + pos[k] * g2, k, cnt, s)
            ogs.view(n, gt)[perm] = og.view(n, gt)                        # scatter back to order

        t_v = _timed(ragged(ov, dP, dQ, off), a.warmup, a.steps, st)
        t_g = _timed(grouped, a.warmup, a.steps, st)
        res["mixed_1_31"] = {"outputs": n, "pairs": int(off[-1]), "ragged_ms": t_v, "grouped_ms": t_g,
                             "calls_grouped": len(groups), "ragged_over_grouped_time": t_v / t_g,
                             "equal": bool(torch.equal(ov, ogs))}
        del dP, dQ, gP, gQ
        # 3. one long product
        m = a.long
        dP, dQ = pairs(m)
        ov, ou = out(1), out(1)
        os_ = torch.zeros(m * gt, dtype=torch.uint8, device="cuda")
        t_v = _timed(ragged(ov, dP, dQ, [0, m]), a.warmup, a.steps, st)
        t_s = _timed(lambda: pr.apply_device(os_.data_ptr(), dP.data_ptr(), dQ.data_ptr(), m, s), a.warmup, a.steps, st)
        k16 = min(m, 1 << 16)
        t_u = _timed(lambda: pr.prod_apply_device(ou.data_ptr(), dP.data_ptr(), dQ.data_ptr(), k16, 1, s), 1, max(1, a.steps // 2), st)
        pr.prod_apply_device(ou.data_ptr(), dP.data_ptr(), dQ.data_ptr(), m, 1, s)
        torch.cuda.synchronize()
        res["one_long"] = {"pairs": m, "ragged_ms": t_v, "singles_ms": t_s, "uniform_k65536_ms": t_u,
                           "ragged_over_singles_time": t_v / t_s, "equal": bool(torch.equal(ov, ou))}
        del dP, dQ, os_
        print(json.dumps(res), flush=True)
        pr.clear()


if __name__ == "__main__":
    main()

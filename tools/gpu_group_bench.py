"""Throughput of the batched group operations (element_pow_zn on G1 and GT, element_from_hash on G1 and G2,
decompression on G2) next to the compiled reference on the host cores.  One JSON line per (type, operation)."""
import json, os, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import multiprocessing as mp
import random


def _cpu(args):
    name, which, elems, ks, n = args
    from oracle import ref as R
    from pbc_b200.params import PARAMS
    rp = R.RefPairing(PARAMS[name])
    t0 = time.perf_counter()
    out = rp.pow_zn(R.G1 if which == "g1" else R.GT, elems, ks, n)
    return out, time.perf_counter() - t0


def main():
    import bench
    from pbc_b200.params import PARAMS
    n = int(sys.argv[1]) if len(sys.argv) > 1 else 1 << 18
    cores = bench.host_cores()
    jobs = []
    for wn in ("a", "f", "d"):
        w = bench.WORKLOADS[wn]
        P, Q = bench.make_inputs(w, n)
        rnd = random.Random(5)
        ks = b"".join(rnd.getrandbits(157).to_bytes(20, "big") for _ in range(4096)) * (n // 4096)
        jobs.append((wn, w, P.tobytes(), Q.tobytes(), ks))
    # CPU legs first (fork before CUDA): bounded samples
    cpu = {}
    pool = mp.get_context("fork").Pool(cores)
    for wn, w, P, Q, ks in jobs:
        g1 = bench.WIRE[w["param"]][0]
        m = cores * 8
        per = m // cores
        args = [(w["param"], "g1", P[c * per * g1:(c + 1) * per * g1], ks[c * per * 20:(c + 1) * per * 20], per) for c in range(cores)]
        t0 = time.perf_counter(); res = pool.map(_cpu, args); wall = time.perf_counter() - t0
        cpu[(wn, "g1")] = (m / wall, b"".join(r[0] for r in res), m)
    pool.close(); pool.join()
    import torch
    from pbc_b200.pairing import Pairing
    for wn, w, P, Q, ks in jobs:
        pr = Pairing(PARAMS[w["param"]])
        dP = torch.frombuffer(bytearray(P), dtype=torch.uint8).cuda()
        dQ = torch.frombuffer(bytearray(Q), dtype=torch.uint8).cuda()
        dK = torch.frombuffer(bytearray(ks), dtype=torch.uint8).cuda()
        dE = torch.empty(n * pr.gt_len, dtype=torch.uint8, device="cuda")
        dO1 = torch.empty(n * pr.g1_len, dtype=torch.uint8, device="cuda")
        dO2 = torch.empty(n * pr.gt_len, dtype=torch.uint8, device="cuda")
        st = torch.cuda.current_stream()
        pr.apply_device(dE.data_ptr(), dP.data_ptr(), dQ.data_ptr(), n, st.cuda_stream)
        for which, fn, out in (("g1", pr.g1_pow_zn_device, dO1), ("gt", pr.gt_pow_zn_device, dO2)):
            src = dP if which == "g1" else dE
            for _ in range(2):
                fn(out.data_ptr(), src.data_ptr(), dK.data_ptr(), n, st.cuda_stream)
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(st)
            for _ in range(3):
                fn(out.data_ptr(), src.data_ptr(), dK.data_ptr(), n, st.cuda_stream)
            e1.record(st)
            torch.cuda.synchronize()
            ms = e0.elapsed_time(e1) / 3
            line = {"type": wn, "op": "element_pow_zn " + which.upper(), "n": n, "ms": ms, "per_s": n / ms * 1e3}
            if (wn, which) in cpu:
                rate, ref_out, m = cpu[(wn, which)]
                line["cpu_reference_per_s"] = rate
                line["cpu_cores"] = cores
                line["parity_vs_reference"] = bytes(out[:m * pr.g1_len].cpu().numpy().tobytes()) == ref_out
            print(json.dumps(line))
        # element_from_hash on G1: n SHA-256-sized inputs
        import numpy as np
        dH = torch.from_numpy(np.random.default_rng(7).integers(0, 256, n * 32, dtype=np.uint8)).cuda()
        for _ in range(2):
            pr.g1_from_hash_device(dO1.data_ptr(), dH.data_ptr(), 32, n, st.cuda_stream)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(st)
        for _ in range(3):
            pr.g1_from_hash_device(dO1.data_ptr(), dH.data_ptr(), 32, n, st.cuda_stream)
        e1.record(st)
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / 3
        print(json.dumps({"type": wn, "op": "element_from_hash G1 (32-byte inputs)", "n": n, "ms": ms, "per_s": n / ms * 1e3}))

    g2_lines(n, cores)


def _cpu_g2(args):
    """one worker's share of a G2 leg on the reference: (outputs, seconds of the reference work alone --
    after the imports, the pairing init and one warm-up item)"""
    name, op, data, n = args
    from oracle import ref as R
    from pbc_b200.params import PARAMS
    rp = R.RefPairing(PARAMS[name])
    run = (lambda d, k: rp.from_hash(R.G2, d, 32, k)) if op == "hash" else (lambda d, k: rp.decompress(R.G2, d, k))
    run(data[:len(data) // n], 1)
    t0 = time.perf_counter()
    out = run(data, n)
    return out, time.perf_counter() - t0


# reference items per host core in the G2 legs: about a second of work each (one core does roughly 40 000
# type f, 90 d159 and 15 g149 hashes per second)
G2_CPU_PER_CORE = {"f": 8192, "d159": 96, "g149": 24}


def _cpu_leg(pool, name, op, data, item, cores):
    """run cores x G2_CPU_PER_CORE[name] items of `data` (item bytes each) on the reference, one share per
    worker; returns (outputs, items/s over the cores = items / the slowest worker's work time, items/s of
    one core = items / the summed work times)"""
    per = G2_CPU_PER_CORE[name]
    res = pool.map(_cpu_g2, [(name, op, data[c * per * item:(c + 1) * per * item], per) for c in range(cores)])
    m = per * cores
    return b"".join(r[0] for r in res), m / max(r[1] for r in res), m / sum(r[1] for r in res)


def _time(fn, st):
    import torch
    for _ in range(2):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(st)
    for _ in range(3):
        fn()
    e1.record(st)
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / 3


def g2_lines(n, cores):
    """element_from_hash on G2 (32-byte inputs) and G2 decompression (of those hashes, compressed on the
    host) for f, d159 and g149; the reference runs a sample of G2_CPU_PER_CORE items per host core (worker
    processes spawned fresh: this process has a CUDA context by now), timed on its work alone, and the
    GPU's bytes for the same items are compared with its output"""
    import numpy as np
    import torch
    from pbc_b200.pairing import Pairing
    from pbc_b200.params import PARAMS
    st = torch.cuda.current_stream()
    pool = mp.get_context("spawn").Pool(cores)
    for name in ("f", "d159", "g149"):
        pr = Pairing(PARAMS[name])
        H = np.random.default_rng(11).integers(0, 256, n * 32, dtype=np.uint8)
        dH = torch.from_numpy(H).cuda()
        dO = torch.empty(n * pr.g2_len, dtype=torch.uint8, device="cuda")
        ms = _time(lambda: pr.g2_from_hash_device(dO.data_ptr(), dH.data_ptr(), 32, n, st.cuda_stream), st)
        pts = bytes(dO.cpu().numpy().tobytes())
        m = G2_CPU_PER_CORE[name] * cores
        ref_out, rate, rate1 = _cpu_leg(pool, name, "hash", H.tobytes(), 32, cores)
        print(json.dumps({"type": name, "op": "element_from_hash G2 (32-byte inputs)", "n": n, "ms": ms,
                          "per_s": n / ms * 1e3, "cpu_reference_per_s": rate, "cpu_reference_per_core_per_s": rate1,
                          "cpu_cores": cores, "cpu_sample": m, "parity_vs_reference": ref_out == pts[:m * pr.g2_len]}))
        comp = pr.g2_compress(pts, n)
        clen = len(comp) // n
        # host buffers: the compressed items are clen (odd) bytes apart
        pr.g2_decompress(comp[:clen * 1024], 1024)
        t0 = time.perf_counter()
        back = pr.g2_decompress(comp, n)
        ms = (time.perf_counter() - t0) * 1e3
        ref_out, rate, rate1 = _cpu_leg(pool, name, "dec", comp, clen, cores)
        print(json.dumps({"type": name, "op": "element_from_bytes_compressed G2 (host buffers, copies included)",
                          "n": n, "ms": ms, "per_s": n / ms * 1e3, "cpu_reference_per_s": rate,
                          "cpu_reference_per_core_per_s": rate1, "cpu_cores": cores, "cpu_sample": m,
                          "roundtrip": back == pts, "parity_vs_reference": ref_out == back[:m * pr.g2_len]}))
    pool.close()
    pool.join()


if __name__ == "__main__":
    main()

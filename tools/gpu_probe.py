"""First-light GPU probe: integer-pipe peak, F_p multiplier throughput vs occupancy, Type A
pairing throughput (device-resident).  Prints one JSON object per line."""
import json, os, subprocess, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from pbc_b200.pairing import Pairing, bench_imad, kernel_launches
from pbc_b200.params import PARAMS

def main():
    pr = Pairing(PARAMS["a"])
    sm = torch.cuda.get_device_properties(0).multi_processor_count
    smi = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    print(json.dumps({"gpu": torch.cuda.get_device_name(0), "sms": sm, "power_limit_and_max_sm_clock": smi}))
    for blocks_per_sm, threads in ((4, 256), (8, 256)):
        iters = 4000
        ms = bench_imad(sm * blocks_per_sm, threads, iters, 3)
        n = sm * blocks_per_sm * threads * 32 * iters
        print(json.dumps({"probe": "imad_wide_peak", "blocks_per_sm": blocks_per_sm, "threads": threads,
                          "ms": ms, "imad_per_s": n / (ms * 1e-3)}))
    # units = multiplier products (IMAD.WIDE.U32) one call executes: 528 per multiplication, 408 per squaring,
    # 2 x 256 + 272 = 784 for the lazy two-product routine (two products, one reduction)
    modes = {0: ("regs_operand_scan_mul", 528), 2: ("regs_product_scan_mul", 528), 3: ("regs_sqr", 408),
             1: ("slots_mul", 528), 6: ("slots_sqr", 408), 7: ("slots_lazy_two_products", 784)}
    for mode, (label, units) in modes.items():
        for bps in (1, 2, 3, 4, 6, 8):
            iters = 2000
            ms = pr.bench_fpmul(mode, sm * bps, iters, 3)
            ops = sm * bps * 128 * iters
            print(json.dumps({"probe": "fpmul512", "mode": label, "blocks_per_sm": bps, "warps_per_sm": bps * 4,
                              "ms": ms, "ns_per_op_per_sm": ms * 1e6 * sm / ops, "ops_per_s": ops / (ms * 1e-3),
                              "units_per_op": units, "units_per_s": units * ops / (ms * 1e-3)}))
    g = json.load(open(os.path.join(os.path.dirname(__file__), "..", "tests", "golden", "a.json")))["pairing"]
    P = b"".join(bytes.fromhex(x) for x in g["P"]); Q = b"".join(bytes.fromhex(x) for x in g["Q"])
    m = len(g["e"])
    for n in (sm * 256, sm * 256 * 4, 1 << 18):
        reps = n // m + 1
        dP = torch.frombuffer(bytearray((P * reps)[:n * 128]), dtype=torch.uint8).cuda()
        dQ = torch.frombuffer(bytearray((Q * reps)[:n * 128]), dtype=torch.uint8).cuda()
        out = torch.empty(n * 128, dtype=torch.uint8, device="cuda")
        st = torch.cuda.current_stream()
        pr.apply_device(out.data_ptr(), dP.data_ptr(), dQ.data_ptr(), n, st.cuda_stream)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(st)
        pr.apply_device(out.data_ptr(), dP.data_ptr(), dQ.data_ptr(), n, st.cuda_stream)
        e1.record(st)
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1)
        print(json.dumps({"probe": "pairing_a_device", "n": n, "ms": ms, "pairings_per_s": n / (ms * 1e-3)}))
    print(json.dumps({"launches": kernel_launches()}))

if __name__ == "__main__":
    main()

"""Slot-machine multiplier throughput against resident blocks per SM.

k_fpmul_slots (the 512-bit multiplier the type A kernels call, through shared-memory slots) launched
with its dynamic shared memory padded to the footprint of a pairing kernel: 72 KB is the nine-slot
Miller kernel, 56 KB the footprint of a seven-slot one (four blocks per SM), 32 KB and 16 KB leave
registers as the limit.  The blocks per
SM of each size come from the device (cudaOccupancyMaxActiveBlocksPerMultiprocessor).  Prints one JSON
object per line; the first names the GPU and its power limit."""
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402
from pbc_b200.pairing import Pairing  # noqa: E402
from pbc_b200.params import PARAMS  # noqa: E402


def gpu_info():
    q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm",
                        "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    return {"gpu": torch.cuda.get_device_name(0), "nvidia_smi": q,
            "sms": torch.cuda.get_device_properties(0).multi_processor_count}


def main():
    print(json.dumps(gpu_info()), flush=True)
    pr = Pairing(PARAMS["a"])
    iters, reps = 2000, 3
    pr.bench_fpmul_smem(0, iters, 1)             # module load and clocks up
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    for kb in (72, 56, 32, 16):
        for rep in range(2):
            ms, bps = pr.bench_fpmul_smem(kb * 1024, iters, reps)
            muls = bps * sms * 128 * iters
            print(json.dumps({"probe": "fpmul_slots_smem", "smem_kb": kb, "blocks_per_sm": bps,
                              "warps_per_sm": 4 * bps, "rep": rep, "ms": ms,
                              "mulmod_per_s": muls / (ms * 1e-3), "imad_equiv_per_s": 528 * muls / (ms * 1e-3)}),
                  flush=True)
    pr.clear()


if __name__ == "__main__":
    main()

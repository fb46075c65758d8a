"""The CPU simulator of the product library WITH its eight-limb type D instance: make_host_sim.py's file
for engine.cu (made with PBC_HOST_SIM_D_WIDE, so engine.cu leaves the instance's launchers to it), then
pbc_b200/csrc/engine_d_wide.cu -- a second translation unit with its own macros (eight limbs, namespace
pbcb200_dw) -- preprocessed on its own the same way and appended.  TEST INFRASTRUCTURE: lets
tests/test_d_wide_cpu.py run the wide type D kernels without a GPU.

usage: python make_host_sim_d_wide.py <out.cpp> [-DNAME=VALUE ...]"""
import os
import re
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from make_host_sim import rewrite_launches  # noqa: E402
from make_host_fp import translate  # noqa: E402

# the prelude make_host_sim.py puts in front of engine.cu
PRELUDE = ("#define __device__\n#define __forceinline__ inline\n#define __noinline__ __attribute__((noinline))\n"
           "#define __constant__\n#define __host__\n#define __global__\n#define __launch_bounds__(...)\n"
           "#define PBC_HOST_SIM 1\n")


def main():
    dst, defs = sys.argv[1], sys.argv[2:]
    subprocess.check_call([sys.executable, os.path.join(HERE, "make_host_sim.py"), dst, "-DPBC_HOST_SIM_D_WIDE=1"] + defs)
    # make_host_sim.py left the adapted copies of pbc_b200/csrc (system includes hidden, inline PTX marked,
    # shared memory made host memory) in _sim_src next to dst; the system headers the wide unit needs are
    # a subset of engine.cu's, already included at the top of dst.  engine_d_wide.h is skipped: the part
    # made from engine.cu declares that interface.
    work = os.path.join(os.path.dirname(os.path.abspath(dst)), "_sim_src")
    pre = subprocess.run(["g++", "-E", "-P", "-x", "c++", "-std=c++17", "-I", work, "-DPBC_ENGINE_D_WIDE_H"] + defs + ["-"],
                         input=PRELUDE + open(os.path.join(work, "engine_d_wide.cu")).read(),
                         capture_output=True, text=True, check=True, cwd=work).stdout
    body = rewrite_launches(translate(pre))
    body = re.sub(r"(\bbool live = idx < n\w*;)", r"\1 if (!live) return;", body)
    assert "<<<" not in body and "__PTX__" not in body
    with open(dst, "a") as f:
        f.write("\n// ---- engine_d_wide.cu (appended by tests/host/make_host_sim_d_wide.py) ----\n")
        f.write(body)


if __name__ == "__main__":
    main()

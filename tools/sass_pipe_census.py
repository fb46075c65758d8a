"""Static instruction census of the built library's kernels, by issue pipe, from `cuobjdump -sass`.

    python tools/sass_pipe_census.py [--lib pbc_b200/libpbc_b200.so] [--filter k_a_] [--json]
    python tools/sass_pipe_census.py --compare OTHER.so        # kernels whose SASS differs between two builds

Per kernel (out-of-line device functions are part of the kernel that calls them): IMAD.WIDE*, the other
instructions of the multiplier pipe (IMAD, IMAD.X, IMAD.MOV, IMAD.HI, IMAD.SHL, IMAD.IADD), IADD3*, shared-memory
and local-memory loads / stores, barriers, and the total.  The counts are static: they say what ptxas made of a
routine (for instance how many additions and moves it placed on the multiplier pipe), not how often it runs.

The register-resident probes k_fpmul_chain<16, true, 0> (multiplication) and k_fpmul_chain<16, true, 2> (squaring)
hold one field operation in their timed loop, so loop_census() of them is the cost of one operation."""
from __future__ import annotations

import argparse
import hashlib
import json
import os
import re
import shutil
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEFAULT_LIB = os.path.join(ROOT, "pbc_b200", "libpbc_b200.so")
MUL_PROBE = "_ZN7pbcb20013k_fpmul_chainILi16ELb1ELi0EE"
SQR_PROBE = "_ZN7pbcb20013k_fpmul_chainILi16ELb1ELi2EE"
COLUMNS = ("imad_wide", "imad_other", "iadd3", "lds_sts", "ldl_stl", "bar", "total")


def cuobjdump():
    exe = shutil.which("cuobjdump")
    if not exe:
        exe = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "cuobjdump")
    return exe if os.path.exists(exe) else None


def kernels(lib):
    """{mangled name: [(address, opcode with modifiers, operand text), ...]}"""
    exe = cuobjdump()
    if not exe:
        raise RuntimeError("cuobjdump not found")
    sass = subprocess.run([exe, "-sass", lib], capture_output=True, text=True, check=True).stdout
    out, cur = {}, None
    for line in sass.splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            cur = out.setdefault(m.group(1), [])
            continue
        m = re.match(r"\s*/\*([0-9a-f]{4,})\*/\s+(?:@!?U?P\d+\s+)?([A-Z][A-Z0-9_.]*)\s*(.*?);", line)
        if m and cur is not None:
            cur.append((int(m.group(1), 16), m.group(2), m.group(3)))
    return out


def census(insns):
    c = dict.fromkeys(COLUMNS, 0)
    for _, op, _ in insns:
        base = op.split(".")[0]
        c["total"] += 1
        if op.startswith("IMAD.WIDE"):
            c["imad_wide"] += 1
        elif base == "IMAD":
            c["imad_other"] += 1
        elif base == "IADD3":
            c["iadd3"] += 1
        elif base in ("LDS", "STS"):
            c["lds_sts"] += 1
        elif base in ("LDL", "STL"):
            c["ldl_stl"] += 1
        elif base == "BAR":
            c["bar"] += 1
    c["mul_pipe"] = c["imad_wide"] + c["imad_other"]
    return c


def loop_census(insns):
    """census of the largest backward-branch loop of a kernel (the timed loop of a probe kernel)"""
    best = None
    for addr, op, args in insns:
        if op.split(".")[0] != "BRA":
            continue
        m = re.search(r"0x([0-9a-f]+)", args)
        if m and int(m.group(1), 16) < addr:
            lo = int(m.group(1), 16)
            if best is None or addr - lo > best[1] - best[0]:
                best = (lo, addr)
    if best is None:
        return None
    return census([i for i in insns if best[0] <= i[0] <= best[1]])


def digest(insns):
    return hashlib.sha256("\n".join("%x %s %s" % i for i in insns).encode()).hexdigest()


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--lib", default=os.environ.get("PBC_B200_LIB") or DEFAULT_LIB)
    ap.add_argument("--filter", default="", help="substring of the mangled kernel name")
    ap.add_argument("--compare", metavar="LIB", help="list the kernels whose SASS differs from this other build")
    ap.add_argument("--json", action="store_true")
    a = ap.parse_args()
    ks = kernels(a.lib)
    if a.compare:
        other = kernels(a.compare)
        same = sorted(k for k in ks if k in other and digest(ks[k]) == digest(other[k]))
        diff = sorted(k for k in ks if k in other and digest(ks[k]) != digest(other[k]))
        print("%d kernels identical, %d differ, %d only in %s, %d only in %s" % (
            len(same), len(diff), len(set(ks) - set(other)), a.lib, len(set(other) - set(ks)), a.compare))
        for k in diff:
            print("differs:", k)
        for k in sorted(set(ks) ^ set(other)):
            print("only in one:", k)
        return 0
    rows = {k: census(v) for k, v in sorted(ks.items()) if a.filter in k}
    for name, probe in (("one multiplication (loop of k_fpmul_chain<16,true,0>)", MUL_PROBE),
                        ("one squaring (loop of k_fpmul_chain<16,true,2>)", SQR_PROBE)):
        hit = [k for k in ks if k.startswith(probe)]
        if hit and loop_census(ks[hit[0]]):
            rows[name] = loop_census(ks[hit[0]])
    if a.json:
        print(json.dumps(rows, indent=1))
        return 0
    print("%10s %10s %8s %8s %8s %5s %8s  kernel" % COLUMNS)
    for k, c in rows.items():
        print("%10d %10d %8d %8d %8d %5d %8d  %s" % (tuple(c[x] for x in COLUMNS) + (k,)))
    return 0


if __name__ == "__main__":
    sys.exit(main())

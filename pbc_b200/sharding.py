"""One-process-per-GPU sharding of a batch (SURVEY 8e): contiguous slices of the OUTPUTS, no
collective on the data path, a host-side gather of the result bytes at the end.

The same split rule as the single-process multi-GPU fan-out inside libpbc_b200.so
(engine.cu run_host: per = ceil(n / world), slice g = [g*per, min(n, (g+1)*per))), so a batch
sharded across ranks with torch.distributed and a batch handed to one process with
pbc_b200_set_devices(world) land on the same devices.  A product of k pairings is never split:
slices are taken over outputs, inputs follow with stride k (element_prod_pairing semantics,
include/pbc_pairing.h:153-171).

Products with a pair count per output (prod_apply_v) are split by shard_bounds_v, the rule of
engine.cu run_host_v: slices of whole outputs balanced by pairs, rank g starting at the first output i
with offsets[i] * world >= g * offsets[-1]; shard_inputs_v cuts the inputs and rebases the offsets.
"""
from __future__ import annotations


def shard_bounds(n_out: int, world: int):
    """[(lo, hi)] per rank; empty slices (lo == hi) when there are more ranks than outputs."""
    if world <= 0:
        raise ValueError("world must be positive")
    per = (n_out + world - 1) // world if n_out else 0
    out = []
    for g in range(world):
        lo = min(n_out, g * per)
        out.append((lo, min(n_out, lo + per)))
    return out


def shard_inputs(in1: bytes, in2: bytes, n_out: int, k: int, len1: int, len2: int, rank: int, world: int):
    """this rank's slice of the inputs (k pairings per output) and its output count"""
    lo, hi = shard_bounds(n_out, world)[rank]
    return in1[lo * k * len1:hi * k * len1], in2[lo * k * len2:hi * k * len2], hi - lo


def shard_bounds_v(offsets, world: int):
    """[(lo, hi)] output slices per rank for a product batch with offsets (n_out + 1 entries): each
    slice holds whole outputs, and its pair count is within the longest output of total / world"""
    if world <= 0:
        raise ValueError("world must be positive")
    offs = [int(v) for v in (offsets.tolist() if hasattr(offsets, "tolist") else offsets)]
    n_out, total = len(offs) - 1, offs[-1]
    starts = []
    for g in range(world + 1):
        lo, hi = 0, n_out                  # first i with offs[i] * world >= g * total (offs increases)
        while lo < hi:
            mid = (lo + hi) // 2
            if offs[mid] * world >= g * total:
                hi = mid
            else:
                lo = mid + 1
        starts.append(lo)
    return [(starts[g], starts[g + 1]) for g in range(world)]


def shard_inputs_v(in1: bytes, in2: bytes, offsets, len1: int, len2: int, rank: int, world: int):
    """this rank's pairs and its offsets rebased to 0 (len(offsets) - 1 = its output count)"""
    offs = [int(v) for v in (offsets.tolist() if hasattr(offsets, "tolist") else offsets)]
    lo, hi = shard_bounds_v(offs, world)[rank]
    a, b = offs[lo], offs[hi]
    return in1[a * len1:b * len1], in2[a * len2:b * len2], [o - a for o in offs[lo:hi + 1]]


def gather_outputs(local: bytes, n_out: int, out_len: int, rank: int, world: int, group=None, dst: int = 0):
    """Host-side gather of the per-rank result bytes to `dst` (torch.distributed: gloo on CPU
    tensors, or any backend that supports gather_object's tensor path).  Returns the full
    n_out * out_len bytes on dst, None elsewhere."""
    import torch
    import torch.distributed as dist
    if world == 1:
        return local
    bounds = shard_bounds(n_out, world)
    per = max(hi - lo for lo, hi in bounds) * out_len
    buf = torch.zeros(max(per, 1), dtype=torch.uint8)
    if local:
        buf[:len(local)] = torch.frombuffer(bytearray(local), dtype=torch.uint8)
    if rank == dst:
        parts = [torch.zeros_like(buf) for _ in range(world)]
        dist.gather(buf, gather_list=parts, dst=dst, group=group)
        return b"".join(bytes(parts[g][:(hi - lo) * out_len].numpy().tobytes())
                        for g, (lo, hi) in enumerate(bounds))
    dist.gather(buf, dst=dst, group=group)
    return None


def sharded_apply(compute, in1: bytes, in2: bytes, n_out: int, k: int, len1: int, len2: int, out_len: int,
                  rank: int, world: int, group=None):
    """compute(in1_slice, in2_slice, n_local) -> bytes runs on this rank's slice (on its GPU);
    rank 0 receives the concatenation in output order."""
    a, b, m = shard_inputs(in1, in2, n_out, k, len1, len2, rank, world)
    local = compute(a, b, m) if m else b""
    return gather_outputs(local, n_out, out_len, rank, world, group)

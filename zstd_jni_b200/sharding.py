"""Multi-GPU host logic: how a batch of independent frames is split over ranks and how the per-rank
results are stitched back into one stream index (SURVEY.md section 8e).

Frames never depend on each other, so the compute needs no collective: every rank compresses /
decompresses its own contiguous range of chunks.  Two shapes are supported:

  * shards born on their rank (weak scaling, bench.py's main line): the only exchange is an all_gather of the
    per-frame sizes (8 bytes per frame) from which every rank derives the global offsets of the concatenated stream;
  * a batch resident on ONE rank (BASELINE.json configs[2], SURVEY.md section 8e items 1-3): `scatter_chunks`
    deals contiguous chunk ranges out over NVLink (grouped send/recv), every rank works on its range,
    `gather_sizes` + `global_offsets` are the size scan, and `gatherv_bytes` lands every rank's packed frames
    at its offset of the one contiguous stream on the root (variable-length gather) -- `gather_fixed` is the same
    for the fixed-size regenerated chunks of the decompression direction.

Works on any torch.distributed backend (NCCL between GPUs, gloo in the CPU tests).
"""
from __future__ import annotations

from typing import List, Tuple

import torch
import torch.distributed as dist


def shard_range(n_items: int, rank: int, world: int) -> Tuple[int, int]:
    """Contiguous, balanced split: the first (n % world) ranks get one extra item."""
    base, extra = divmod(n_items, world)
    start = rank * base + min(rank, extra)
    return start, start + base + (1 if rank < extra else 0)


def gather_sizes(local_sizes: torch.Tensor, n_items: int, group=None) -> torch.Tensor:
    """all_gather the per-frame sizes of every rank -> tensor of n_items sizes in global frame order."""
    world = dist.get_world_size(group) if dist.is_initialized() else 1
    if world == 1:
        return local_sizes.clone()
    counts = [shard_range(n_items, r, world) for r in range(world)]
    longest = max(e - s for s, e in counts)
    padded = torch.zeros(longest, dtype=local_sizes.dtype, device=local_sizes.device)
    padded[: local_sizes.numel()] = local_sizes
    bufs = [torch.zeros_like(padded) for _ in range(world)]
    dist.all_gather(bufs, padded, group=group)
    return torch.cat([bufs[r][: counts[r][1] - counts[r][0]] for r in range(world)])


def global_offsets(all_sizes: torch.Tensor) -> torch.Tensor:
    """Exclusive scan: offsets[i] = start of frame i in the concatenated stream; offsets[n] = total."""
    out = torch.zeros(all_sizes.numel() + 1, dtype=torch.int64, device=all_sizes.device)
    out[1:] = torch.cumsum(all_sizes.to(torch.int64), 0)
    return out


def rank_byte_range(offsets: torch.Tensor, n_items: int, rank: int, world: int) -> Tuple[int, int]:
    """Where rank's frames live in the concatenated stream (for gatherv-style placement)."""
    s, e = shard_range(n_items, rank, world)
    return int(offsets[s]), int(offsets[e])


# ------------------------------------------------------------------------------------------ data plane
def _p2p(ops):
    if ops:
        for w in dist.batch_isend_irecv(ops):
            w.wait()


def scatter_chunks(src_root, n_items: int, item_bytes: int, recv_buf: torch.Tensor, root: int = 0, group=None) -> Tuple[int, int]:
    """Deal items [shard_range(rank)] of the root's contiguous batch `src_root` (uint8, n_items * item_bytes; None elsewhere) into
    every rank's `recv_buf` (uint8, at least its shard's bytes).  One grouped send/recv (NCCL: a single fused launch over
    NVLink); the root keeps its own shard with a local copy.  Returns the rank's item range."""
    world = dist.get_world_size(group) if dist.is_initialized() else 1
    rank = dist.get_rank(group) if dist.is_initialized() else 0
    s, e = shard_range(n_items, rank, world)
    if world == 1:
        recv_buf[: (e - s) * item_bytes].copy_(src_root[s * item_bytes: e * item_bytes])
        return s, e
    ops = []
    if rank == root:
        for r in range(world):
            rs, re = shard_range(n_items, r, world)
            if r == root:
                recv_buf[: (re - rs) * item_bytes].copy_(src_root[rs * item_bytes: re * item_bytes])
            elif re > rs:
                ops.append(dist.P2POp(dist.isend, src_root[rs * item_bytes: re * item_bytes], r, group))
    elif e > s:
        ops.append(dist.P2POp(dist.irecv, recv_buf[: (e - s) * item_bytes], root, group))
    _p2p(ops)
    return s, e


def gatherv_bytes(local: torch.Tensor, rank_ranges: List[Tuple[int, int]], out_root, root: int = 0, group=None) -> None:
    """Variable-length gather: rank r's `local` bytes (uint8, rank_ranges[r][1] - rank_ranges[r][0] of them) land at
    out_root[rank_ranges[r][0] : rank_ranges[r][1]] on the root -- the contiguous stream, frames in global order."""
    world = dist.get_world_size(group) if dist.is_initialized() else 1
    rank = dist.get_rank(group) if dist.is_initialized() else 0
    lo, hi = rank_ranges[rank]
    if world == 1:
        out_root[lo:hi].copy_(local[: hi - lo])
        return
    ops = []
    if rank == root:
        out_root[lo:hi].copy_(local[: hi - lo])
        for r in range(world):
            rl, rh = rank_ranges[r]
            if r != root and rh > rl:
                ops.append(dist.P2POp(dist.irecv, out_root[rl:rh], r, group))
    elif hi > lo:
        ops.append(dist.P2POp(dist.isend, local[: hi - lo], root, group))
    _p2p(ops)


def rank_byte_ranges(offsets: torch.Tensor, n_items: int, world: int) -> List[Tuple[int, int]]:
    """Byte range of every rank's frames in the concatenated stream (from the global offsets)."""
    host = offsets.cpu()
    return [(int(host[s]), int(host[e])) for s, e in (shard_range(n_items, r, world) for r in range(world))]


def gather_fixed(local: torch.Tensor, n_items: int, item_bytes: int, out_root, root: int = 0, group=None) -> None:
    """Decompression direction: every rank's regenerated chunks (fixed size) back to the root, in global order."""
    world = dist.get_world_size(group) if dist.is_initialized() else 1
    ranges = [(s * item_bytes, e * item_bytes) for s, e in (shard_range(n_items, r, world) for r in range(world))]
    gatherv_bytes(local, ranges, out_root, root, group)


def bind_to_gpu_numa(device_index: int) -> str:
    """Pin the calling process to the CPUs of the NUMA node its GPU hangs off, so that page-locked buffers allocated afterwards
    (first touch) and the copy threads sit next to the GPU's PCIe root.  Best effort; returns what was done."""
    import os
    try:
        props = torch.cuda.get_device_properties(device_index)
        bdf = f"{props.pci_domain_id:04x}:{props.pci_bus_id:02x}:{props.pci_device_id:02x}.0"
        node = int(open(f"/sys/bus/pci/devices/{bdf}/numa_node").read().strip())
        if node < 0:
            return "numa_node unknown"
        cpus = set()
        for part in open(f"/sys/devices/system/node/node{node}/cpulist").read().strip().split(","):
            a, _, b = part.partition("-")
            cpus.update(range(int(a), int(b or a) + 1))
        cpus &= os.sched_getaffinity(0)
        if not cpus:
            return f"node {node}: no allowed cpu"
        os.sched_setaffinity(0, cpus)
        return f"node {node} ({len(cpus)} cpus)"
    except Exception as ex:      # noqa: BLE001 -- sysfs layout / permissions differ between hosts
        return f"not bound ({type(ex).__name__})"

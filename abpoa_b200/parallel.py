"""Multi-GPU: shard independent read groups over ranks (one process per GPU).

The path shards naturally (SURVEY 8e): groups share nothing, a single alignment never spans GPUs,
so there is NO collective on the data path.  torch.distributed (NCCL on GPUs, gloo on CPU for the
tests) is used only to scatter the encoded reads from rank 0 and to gather the per-group results.
"""
from __future__ import annotations

from typing import Callable, Sequence

import numpy as np


def shard_bounds(n_items: int, rank: int, world: int) -> tuple[int, int]:
    """Contiguous, balanced [lo, hi) of `n_items` for `rank` (sizes differ by at most one)."""
    base, extra = divmod(n_items, world)
    lo = rank * base + min(rank, extra)
    return lo, lo + base + (1 if rank < extra else 0)


def lpt_assignment(costs: Sequence[float], world: int) -> list[list[int]]:
    """Longest-processing-time-first assignment of groups to ranks for unequal groups
    (cost ~ sum of read_len^2); returns the group indices of every rank, each in input order."""
    load = [0.0] * world
    out: list[list[int]] = [[] for _ in range(world)]
    for g in sorted(range(len(costs)), key=lambda i: -costs[i]):
        r = min(range(world), key=lambda k: load[k])
        out[r].append(g)
        load[r] += costs[g]
    return [sorted(x) for x in out]


def group_cost(reads: Sequence[np.ndarray]) -> float:
    return float(sum(len(r) for r in reads)) * (max((len(r) for r in reads), default=0) + 1)


# ---- tensor payloads: everything that crosses ranks is a flat uint8 tensor (NCCL moves tensors, not pickles) ----
def pack_groups(groups) -> np.ndarray:
    """[n_groups i32][reads per group i32 x G][read length i32 x R][bases u8 ...] as one uint8 array."""
    n_reads = np.array([len(g) for g in groups], dtype=np.int32)
    lens = np.array([len(r) for g in groups for r in g], dtype=np.int32)
    bases = np.concatenate([np.ascontiguousarray(r, dtype=np.uint8) for g in groups for r in g]) if lens.size else np.zeros(0, np.uint8)
    head = np.array([len(groups)], dtype=np.int32)
    return np.concatenate([head.view(np.uint8), n_reads.view(np.uint8), lens.view(np.uint8), bases])


def unpack_groups(buf: np.ndarray):
    buf = np.ascontiguousarray(buf, dtype=np.uint8)
    g = int(buf[:4].view(np.int32)[0])
    n_reads = buf[4: 4 + 4 * g].view(np.int32)
    r = int(n_reads.sum())
    lens = buf[4 + 4 * g: 4 + 4 * g + 4 * r].view(np.int32)
    off = 4 + 4 * g + 4 * r
    groups, k = [], 0
    for n in n_reads:
        grp = []
        for _ in range(int(n)):
            grp.append(buf[off: off + int(lens[k])].copy())
            off += int(lens[k]); k += 1
        groups.append(grp)
    return groups


_DT = {0: np.uint8, 1: np.int32, 2: np.int64}
_DTC = {np.dtype(np.uint8): 0, np.dtype(np.int32): 1, np.dtype(np.int64): 2}


def pack_results(results) -> np.ndarray:
    """results: per group a list of numpy arrays (uint8 / int32 / int64).  [n_groups i32] then per group
    [n_arrays i32] and per array [dtype code i32][length i32][bytes, padded to 4]."""
    parts = [np.array([len(results)], dtype=np.int32).view(np.uint8)]
    for arrs in results:
        parts.append(np.array([len(arrs)], dtype=np.int32).view(np.uint8))
        for a in arrs:
            a = np.ascontiguousarray(a)
            if a.dtype not in _DTC:
                a = a.astype(np.int64)
            raw = a.view(np.uint8).reshape(-1)
            parts.append(np.array([_DTC[a.dtype], a.size], dtype=np.int32).view(np.uint8))
            parts.append(raw)
            if raw.size % 4:
                parts.append(np.zeros(4 - raw.size % 4, np.uint8))
    return np.concatenate(parts)


def unpack_results(buf: np.ndarray):
    buf = np.ascontiguousarray(buf, dtype=np.uint8)
    n = int(buf[:4].view(np.int32)[0]); off = 4
    out = []
    for _ in range(n):
        k = int(buf[off: off + 4].view(np.int32)[0]); off += 4
        arrs = []
        for _ in range(k):
            code, size = (int(x) for x in buf[off: off + 8].view(np.int32)); off += 8
            dt = np.dtype(_DT[code]); nb = size * dt.itemsize
            arrs.append(buf[off: off + nb].view(dt).copy()); off += (nb + 3) & ~3
        out.append(arrs)
    return out


def distributed_msa(groups, cfg, runner: Callable | None = None, balance: bool = True):
    """Run the MSA of every group on the ranks of the default process group.

    groups : list of read groups on rank 0 (ignored elsewhere).
    runner : callable(cfg, list_of_groups) -> per group a list of numpy arrays; defaults to the GPU batch engine
             on the rank's current CUDA device, returning [consensus..., coverage...] per group.
    Returns the per-group results in input order on rank 0, None on the other ranks.

    Communication = one scatter of the packed reads and one gather of the packed results, both as uint8 tensors
    (CUDA tensors over NCCL, CPU tensors over gloo); nothing is exchanged while the ranks compute.
    """
    import torch
    import torch.distributed as dist

    rank, world = dist.get_rank(), dist.get_world_size()
    dev = torch.device("cuda", torch.cuda.current_device()) if dist.get_backend() == "nccl" else torch.device("cpu")
    if runner is None:
        from .batch import BatchEngine

        def runner(c, gs):
            with BatchEngine() as eng:
                return [list(r.cons) + list(r.cov) for r in eng.run(c, gs)]

    # ---- scatter: rank 0 decides the assignment and ships every rank its groups ----
    sizes = torch.zeros(world, dtype=torch.int64, device=dev)
    payload, assign = None, None
    if rank == 0:
        n = len(groups)
        if balance:
            assign = lpt_assignment([group_cost(g) for g in groups], world)
        else:
            assign = [list(range(*shard_bounds(n, r, world))) for r in range(world)]
        payload = [pack_groups([groups[i] for i in idx]) for idx in assign]
        sizes = torch.tensor([p.size for p in payload], dtype=torch.int64, device=dev)
    dist.broadcast(sizes, src=0)
    cap = int(sizes.max().item())
    mine = torch.zeros(cap, dtype=torch.uint8, device=dev)
    if rank == 0:
        slist = []
        for p in payload:
            t = torch.zeros(cap, dtype=torch.uint8)
            t[: p.size] = torch.from_numpy(p)
            slist.append(t.to(dev))
        dist.scatter(mine, slist, src=0)
    else:
        dist.scatter(mine, None, src=0)
    my_groups = unpack_groups(mine[: int(sizes[rank].item())].cpu().numpy())

    # ---- compute: no communication ----
    results = runner(cfg, my_groups) if my_groups else []

    # ---- gather ----
    packed = pack_results(results)
    rsz = torch.tensor([packed.size], dtype=torch.int64, device=dev)
    all_sz = [torch.zeros(1, dtype=torch.int64, device=dev) for _ in range(world)]
    dist.all_gather(all_sz, rsz)
    rcap = max(int(t.item()) for t in all_sz)
    send = torch.zeros(rcap, dtype=torch.uint8)
    send[: packed.size] = torch.from_numpy(packed)
    send = send.to(dev)
    glist = [torch.zeros(rcap, dtype=torch.uint8, device=dev) for _ in range(world)] if rank == 0 else None
    dist.gather(send, glist, dst=0)
    if rank != 0:
        return None
    out = [None] * sum(len(i) for i in assign)
    for r in range(world):
        res = unpack_results(glist[r][: int(all_sz[r].item())].cpu().numpy())
        for g, x in zip(assign[r], res):
            out[g] = x
    return out

"""Multi-GPU fan-out of a keyed history: one process per GPU, shards (independent keys) partitioned
across ranks, ONE tiny collective to merge the verdicts.

This is the multi-GPU shape of `jepsen.independent/checker` (workloads/set_full.clj:155): linearizability is
local (Herlihy–Wing), so per-key verdicts compose with no cross-shard state; ranks never exchange
configurations.  The only exchange is `all_reduce(MAX)` over int32 verdict codes (true 0 < :unknown 1 <
false 2 == checker/merge-valid) and witness indices — bytes over NVLink/NVSwitch through NCCL
(`torch.distributed`, backend "nccl"; "gloo" for the CPU tests).
"""
from __future__ import annotations

from typing import Callable, Sequence

import numpy as np

from .history import FlatHistory


def shard_costs(h: FlatHistory) -> np.ndarray:
    """Cost proxy per shard for load balancing: events^2 (search work grows super-linearly)."""
    n = np.diff(h.shard_off).astype(np.float64)
    return n * n


def assign_shards(costs: Sequence[float], world_size: int) -> list[list[int]]:
    """Longest-processing-time-first partition of shards over ranks (deterministic)."""
    order = sorted(range(len(costs)), key=lambda s: (-float(costs[s]), s))
    load = [0.0] * world_size
    out: list[list[int]] = [[] for _ in range(world_size)]
    for s in order:
        r = min(range(world_size), key=lambda k: (load[k], k))
        out[r].append(s)
        load[r] += float(costs[s])
    for lst in out:
        lst.sort()
    return out


def check_sharded(h: FlatHistory, check_fn: Callable[[FlatHistory], Sequence[dict]], rank: int,
                  world_size: int, all_reduce_max: Callable[[np.ndarray], np.ndarray] | None = None) -> dict:
    """Run `check_fn` on this rank's shards and merge per-shard results over all ranks.

    check_fn(sub_history) -> one dict per shard with integer fields `valid` and (optionally)
    `witness_index`.  all_reduce_max(int32 array) -> element-wise MAX over ranks (identity when None).
    Returns {"valid": merged code, "shard_valid": int32[n_shards], "shard_witness": int32[n_shards],
             "mine": [...shards checked here...]}."""
    parts = assign_shards(shard_costs(h), world_size)
    mine = parts[rank]
    packed = np.full(2 * h.n_shards, -1, np.int32)  # [valid..., witness...], -1 = not mine
    if mine:
        sub = h.select_shards(mine)
        res = check_fn(sub)
        for s, r in zip(mine, res):
            packed[s] = int(r["valid"])
            packed[h.n_shards + s] = int(r.get("witness_index", -1))
    if all_reduce_max is not None:
        packed = all_reduce_max(packed)
    valid = packed[:h.n_shards].copy()
    valid[valid < 0] = 0  # shards nobody owned (only when n_shards == 0)
    return {"valid": int(valid.max()) if valid.size else 0, "shard_valid": valid,
            "shard_witness": packed[h.n_shards:].copy(), "mine": mine}


def torch_all_reduce_max(device=None):
    """all_reduce(MAX) through torch.distributed (NCCL on GPUs, gloo on CPU)."""
    import torch
    import torch.distributed as dist

    def fn(arr: np.ndarray) -> np.ndarray:
        t = torch.from_numpy(arr.copy())
        if device is not None:
            t = t.to(device)
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
        return t.cpu().numpy()

    return fn

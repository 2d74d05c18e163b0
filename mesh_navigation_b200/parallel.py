"""One-goal-per-GPU sharding of batched multi-goal potential fields (SURVEY.md 8e).

The path shards perfectly across queries (independent goals, the map is replicated read-only on
every GPU) and not at all inside one query, so the only collective is the final gather of the
potential arrays.  One process per GPU; `torch.distributed` (NCCL over NVLink/NVSwitch on the GPU
box, gloo in the CPU tests) is plumbing only -- there is no compute step that a collective follows
tile by tile, hence nothing to fuse.

goal k -> rank k mod N.  By default a rank computes all its goals in ONE batch call (the batch kernel wants as many
concurrent wavefronts as the GPU holds) followed by one all_gather_into_tensor straight into the final buffer: over
NVLink / NVSwitch the gather of 1024 x 1M-vertex fields (4 GB per rank) is a small fraction of the batch's compute, so
there is nothing worth overlapping.  `chunk > 0` keeps the chunked, overlapped variant (gather of chunk i
runs while chunk i+1 is computed) for maps / goal counts where the fields of a rank do not fit next to the gathered buffer.
"""
from __future__ import annotations

from typing import Callable, List, Sequence

import numpy as np


def shard_indices(n_goals: int, rank: int, world: int) -> np.ndarray:
    """indices of the goals owned by `rank` (goal k -> rank k mod world)"""
    return np.arange(rank, n_goals, world, dtype=np.int64)


def goals_per_rank(n_goals: int, world: int) -> List[int]:
    return [len(range(r, n_goals, world)) for r in range(world)]


def unshard_order(n_goals: int, world: int) -> np.ndarray:
    """row permutation that maps the rank-major gathered buffer back to goal order"""
    per = goals_per_rank(n_goals, world)
    pad = max(per)
    order = np.empty(n_goals, dtype=np.int64)
    for r in range(world):
        idx = shard_indices(n_goals, r, world)
        order[idx] = r * pad + np.arange(len(idx))
    return order


def sharded_potentials(compute_chunk: Callable[[np.ndarray, "object"], None], n_goals: int, V: int, *, rank: int,
                       world: int, device, chunk: int = 0, dist=None, torch=None, timings: dict = None):
    """Run `compute_chunk(goal_indices, out_tensor)` for this rank's goals and all-gather every rank's
    fields (every rank gets all of them, float32 on `device`).  Return value, indexable by goal either way:
      world == 1: the [n_goals, V] tensor itself;
      world  > 1: a zero-copy [pad, world, V] view of the rank-major gather buffer -- row (i, r) is the field of goal
                  i * world + r, rows of the ragged last shard are +inf.  `goal_order_rows(result, n_goals, V)` gives the
                  contiguous [n_goals, V] tensor when a consumer needs one (it copies).

    compute_chunk fills out_tensor[:len(goal_indices)] (float32, [chunk, V], on `device`) with the
    potential fields of the given global goal indices.  chunk = 0: all goals of the rank in one call.
    timings (optional dict): receives "gather_ms" (CUDA events around the collective; single-chunk mode on CUDA only).
    """
    if torch is None:
        import torch as _t
        torch = _t
    mine = shard_indices(n_goals, rank, world)
    pad = max(goals_per_rank(n_goals, world))
    if chunk <= 0:
        chunk = max(pad, 1)
    if world > 1 and chunk >= pad and hasattr(dist, "all_gather_into_tensor"):
        # one batch call, one collective, gathered in place: rank r's rows land at [r*pad, (r+1)*pad) of the final buffer
        gathered = torch.empty((world * pad, V), dtype=torch.float32, device=device)
        local = gathered[rank * pad:(rank + 1) * pad]
        if pad > len(mine):
            local[len(mine):].fill_(float("inf"))
        if len(mine):
            compute_chunk(mine, local[:len(mine)])
        cuda = getattr(device, "type", str(device)) == "cuda"
        if cuda and timings is not None:
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
        dist.all_gather_into_tensor(gathered, local.clone() if not cuda else local)   # (gloo: no in-place aliasing)
        if cuda and timings is not None:
            e1.record(); torch.cuda.synchronize(); timings["gather_ms"] = e0.elapsed_time(e1)
        return gathered.view(world, pad, V).transpose(0, 1)
    local = torch.empty((pad, V), dtype=torch.float32, device=device)
    if pad > len(mine):
        local[len(mine):].fill_(float("inf"))                 # padding rows of the ragged last shard
    if world == 1:
        for s in range(0, len(mine), chunk):
            idx = mine[s:s + chunk]
            compute_chunk(idx, local[s:s + len(idx)])
        return local[:n_goals]
    gathered = torch.empty((world * pad, V), dtype=torch.float32, device=device)
    views = [gathered[r * pad:(r + 1) * pad] for r in range(world)]
    pending = []
    # chunk boundaries are identical on every rank (pad is global) so the collectives line up
    for s in range(0, pad, chunk):
        e = min(pad, s + chunk)
        idx = mine[s:min(e, len(mine))]
        if len(idx):
            compute_chunk(idx, local[s:s + len(idx)])
        outs = [v[s:e] for v in views]
        pending.append(dist.all_gather(outs, local[s:e], async_op=True))   # overlaps with the next chunk
    for p in pending:
        p.wait()
    # rank-major buffer -> goal order without a copy: row (i, r) of the [pad, world, V] view is goal i*world + r
    return gathered.view(world, pad, V).transpose(0, 1)


def goal_order_rows(result, n_goals: int, V: int):
    """materialise the result of sharded_potentials as a contiguous [n_goals, V] tensor (tests / consumers)"""
    if result.dim() == 2:
        return result[:n_goals]
    return result.reshape(-1, V)[:n_goals]

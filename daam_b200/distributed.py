"""Multi-GPU: independent prompts shard across ranks, one optional collective returns the finished maps.

The reference has no distributed code (SURVEY.md section 5); every prompt's accumulators are independent, so the hot
path needs no exchange: rank r traces prompts ``r, r + world, ...`` on its own GPU (one process per GPU). The only
collective is :func:`gather_heat_maps` -- an ``all_gather`` of the final ``[77, xh, xw]`` fp32 maps (1.26 MB per prompt;
NCCL over NVLink on GPUs, gloo in the CPU tests).
"""
from __future__ import annotations

from typing import List, Optional, Sequence

import torch
import torch.distributed as dist

__all__ = ['shard_prompts', 'gather_heat_maps', 'pad_heat_map']

TOKENS = 77


def shard_prompts(prompts: Sequence[str], rank: int, world_size: int) -> List[int]:
    """Indices of the prompts rank ``rank`` owns (round-robin, so uneven counts differ by at most one)."""
    if not 0 <= rank < world_size:
        raise ValueError(f'rank {rank} outside world of {world_size}')
    return list(range(rank, len(prompts), world_size))


def pad_heat_map(maps: torch.Tensor, tokens: int = TOKENS) -> torch.Tensor:
    """``[n_rows, xh, xw]`` -> ``[tokens, xh, xw]`` zero-padded, so that maps of different prompts stack."""
    out = maps.new_zeros((tokens,) + tuple(maps.shape[1:]))
    out[:maps.shape[0]] = maps
    return out


def gather_heat_maps(local_maps: Sequence[torch.Tensor], n_total: int, x, group=None,
                     tokens: int = TOKENS, device=None) -> Optional[torch.Tensor]:
    """All-gathers per-prompt global heat maps. ``local_maps[j]`` belongs to prompt ``rank + j * world``; returns
    ``[n_total, tokens, xh, xw]`` (rows beyond a prompt's length are zero) on every rank. ``x``: the map side, or
    ``(xh, xw)`` for non-square images. Compact maps of a ``long_prompts`` trace with ``c``-chunk contexts have up to
    ``75 c + 2`` rows: pass ``tokens=75 * c + 2``.

    ``device``: where the exchange buffers live. Default: the device of ``local_maps``; a rank that owns no prompt
    (``n_total < world``, or an uneven shard) has no map to infer it from and then uses the current CUDA device under
    NCCL (every rank of a NCCL collective must pass CUDA tensors) and the CPU under gloo."""
    world = dist.get_world_size(group) if dist.is_initialized() else 1
    per_rank = (n_total + world - 1) // world
    if device is None:
        if local_maps:
            device = local_maps[0].device
        elif dist.is_initialized() and dist.get_backend(group) == 'nccl':
            device = torch.device('cuda', torch.cuda.current_device())
        else:
            device = torch.device('cpu')
    xh, xw = (int(x[0]), int(x[1])) if isinstance(x, (tuple, list)) else (int(x), int(x))
    mine = torch.zeros((per_rank, tokens, xh, xw), dtype=torch.float32, device=device)
    for j, m in enumerate(local_maps):
        mine[j] = pad_heat_map(m.float(), tokens)
    if world == 1:
        return mine[:n_total]
    gathered = torch.empty((world * per_rank, tokens, xh, xw), dtype=torch.float32, device=device)
    dist.all_gather_into_tensor(gathered, mine, group=group)      # rank-major concatenation along dim 0
    # row r * per_rank + j is prompt r + j * world
    gathered = gathered.view(world, per_rank, tokens, xh, xw)
    return gathered.permute(1, 0, 2, 3, 4).reshape(per_rank * world, tokens, xh, xw)[:n_total].contiguous()

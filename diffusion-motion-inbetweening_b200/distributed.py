"""Batch-sharded sampling across the GPUs of one node (SURVEY.md 8(e)).

Samples of a batch never interact (attention is within a sequence, LayerNorm per token, schedule per sample), so
rank r takes rows [r*B/G, (r+1)*B/G) of every per-sample input, runs the whole loop locally with no per-step
traffic, and ONE all-gather of the finished samples over NVLink (NCCL) assembles the batch.  The engine's noise
generator is keyed by the GLOBAL sample index (`sample_offset`), so results do not depend on G.
"""
from __future__ import annotations

from typing import Optional

import torch
import torch.distributed as dist


def _shard(v, lo, hi, B):
    if torch.is_tensor(v) and v.dim() > 0 and v.shape[0] == B:
        return v[lo:hi]
    if isinstance(v, (list, tuple)) and len(v) == B:
        return v[lo:hi]
    return v


def shard_model_kwargs(model_kwargs: dict, lo: int, hi: int, B: int) -> dict:
    out = {}
    for k, v in model_kwargs.items():
        out[k] = {kk: _shard(vv, lo, hi, B) for kk, vv in v.items()} if isinstance(v, dict) else _shard(v, lo, hi, B)
    return out


def sharded_sample(diffusion, model, shape, model_kwargs: Optional[dict] = None, sampler: str = "p_sample_loop",
                   noise: Optional[torch.Tensor] = None, group=None, gather: bool = True, **kwargs) -> torch.Tensor:
    """Run `diffusion.<sampler>` on this rank's slice of the batch and all-gather the results.

    shape is the GLOBAL (B, njoints, 1, nframes); B must divide by the world size.  Works with any backend
    (NCCL on GPUs; gloo is used by the CPU tests of the sharding logic with a stand-in sampler).
    """
    if getattr(diffusion, "window", None) is not None:
        raise NotImplementedError("sharded_sample does not shard overlapping windows (diffusion.window)")
    world = dist.get_world_size(group) if dist.is_initialized() else 1
    rank = dist.get_rank(group) if dist.is_initialized() else 0
    B = int(shape[0])
    if B % world != 0:
        raise ValueError(f"global batch {B} is not divisible by world size {world}")
    per = B // world
    lo, hi = rank * per, (rank + 1) * per
    local_kwargs = shard_model_kwargs(model_kwargs or {}, lo, hi, B)
    local_noise = None if noise is None else noise[lo:hi]
    prev_offset = getattr(diffusion, "sample_offset", 0)
    prev_tape = getattr(diffusion, "noise_tape", None)
    prev_rng = getattr(diffusion, "rng", "engine")
    prev_seed = getattr(diffusion, "engine_seed", None)
    diffusion.sample_offset = lo
    diffusion.rng = "engine"  # keyed by global sample index: the result does not depend on the number of ranks
    if prev_seed is None:
        # one Philox key for the whole job: rank 0 draws it from torch's global CPU generator (so `fixseed` still
        # decides it) and every rank uses that one; x_T and the per-step noise of global sample g are then functions
        # of (key, g) only
        key = torch.randint(0, 2 ** 62, (1,), dtype=torch.int64)
        if world > 1:
            dev = torch.device("cuda", torch.cuda.current_device()) if dist.get_backend(group) == "nccl" else torch.device("cpu")
            key = key.to(dev)
            dist.broadcast(key, src=dist.get_global_rank(group, 0) if group is not None else 0, group=group)
        diffusion.engine_seed = int(key.item())
    if prev_tape is not None:
        diffusion.noise_tape = prev_tape[:, lo:hi].contiguous()
    try:
        local = getattr(diffusion, sampler)(model, (per,) + tuple(shape[1:]), noise=local_noise, model_kwargs=local_kwargs,
                                           **kwargs)
    finally:
        diffusion.sample_offset = prev_offset
        diffusion.rng = prev_rng
        diffusion.engine_seed = prev_seed
        diffusion.noise_tape = prev_tape
    if world == 1 or not gather:
        return local
    out = torch.empty((B,) + tuple(local.shape[1:]), dtype=local.dtype, device=local.device)
    dist.all_gather_into_tensor(out, local.contiguous(), group=group)
    return out

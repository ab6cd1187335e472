"""The evaluation-loop caller of the sampling path (SURVEY.md 8(f)-3), re-organised for a multi-GPU box.

Reference: `CompMDMGeneratedDatasetCondMDI.__init__`
(data_loaders/humanml/motion_loaders/comp_v6_model_dataset_condmdi.py:99-383) walks the evaluation dataloader and, for
every batch i of 32 motions and every repetition t (1, or `mm_num_repeats` for the multimodality batches), calls

    fixseed(seed * 100_000 + i * 100 + t)                                                    (:293-294)
    sample = motion_diffusion.p_sample_loop(motion_model, (bs, njoints, nfeats, nframes), clip_denoised=False,
                                            model_kwargs=model_kwargs, skip_timesteps=0, init_image=None, progress=False,
                                            dump_steps=None, noise=None, const_noise=False)   (:343-356)

one call after the other on one GPU ("about 20 hours", README.md:238).  The calls are independent of each other (only
the post-processing and the metric bookkeeping consume them in order), so this module runs the SAME list of calls

  * sharded over the ranks of a torch.distributed job (job j -> rank j % world; no per-step traffic),
  * optionally MERGED: consecutive jobs that differ only in their per-sample inputs are concatenated into one engine
    batch (the engine is fastest at 64 motions per GPU; the evaluation's batches are 32), and
  * returns every job's sample, in job order, on every rank (one gather of finished samples).

Noise: `rng="torch"` reproduces the reference call by call (fixseed per job, torch's generator stream; jobs are then
never merged); `rng="engine"` keys every motion's noise by (seed, global motion index), so the result depends on
neither the merge width nor the number of ranks.

The metric code around the call (kps error, skating ratio, abs<->rel conversion, the T2M evaluators) stays the
reference's: INTEGRATION.md shows the replacement of the double loop at :190-356 by `EvalJob` construction + one call.
"""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import Callable, Dict, List, Optional, Sequence

import torch
import torch.distributed as dist


@dataclass
class EvalJob:
    """One sampler call of the reference's evaluation loop."""
    batch_index: int                       # i: index of the dataloader batch
    repeat: int                            # t: repetition (0 unless the batch is a multimodality batch)
    shape: Sequence[int]                   # (bs, njoints, nfeats, nframes)
    model_kwargs: dict                     # {'y': {...}, optionally 'obs_x0' / 'obs_mask'} exactly as the reference builds it
    seed_number: Optional[int] = None      # the reference's seed * 100_000 + i * 100 + t   (:293)
    extra: dict = field(default_factory=dict)


def eval_seed_number(seed: int, batch_index: int, repeat: int) -> int:
    """comp_v6_model_dataset_condmdi.py:293."""
    return seed * 100_000 + batch_index * 100 + repeat


def build_jobs(batches, seed: int, mm_idxs: Sequence[int] = (), mm_num_repeats: int = 1) -> List[EvalJob]:
    """The reference's double loop (:190, :291) as a flat job list.  `batches` yields (shape, model_kwargs) per
    dataloader batch, already carrying the conditioning the reference adds before the call (:209-287)."""
    jobs = []
    mm = set(int(i) for i in mm_idxs)
    for i, (shape, model_kwargs) in enumerate(batches):
        for t in range(mm_num_repeats if i in mm else 1):
            jobs.append(EvalJob(i, t, tuple(shape), model_kwargs, eval_seed_number(seed, i, t)))
    return jobs


def _mergeable(a: EvalJob, b: EvalJob) -> bool:
    if tuple(a.shape[1:]) != tuple(b.shape[1:]) or set(a.model_kwargs) != set(b.model_kwargs):
        return False
    ya, yb = a.model_kwargs["y"], b.model_kwargs["y"]
    if set(ya) != set(yb):
        return False
    for k in ya:
        va, vb = ya[k], yb[k]
        batched = (torch.is_tensor(va) and va.dim() > 0 and va.shape[0] == a.shape[0]) or \
                  (isinstance(va, (list, tuple)) and len(va) == a.shape[0])
        if batched:
            continue
        if torch.is_tensor(va) or torch.is_tensor(vb):
            if not (torch.is_tensor(va) and torch.is_tensor(vb) and va.shape == vb.shape and torch.equal(va, vb)):
                return False
        elif va != vb:
            return False
    return True


def _cat(values, sizes):
    v0 = values[0]
    if torch.is_tensor(v0) and v0.dim() > 0 and v0.shape[0] == sizes[0]:
        return torch.cat(list(values), dim=0)
    if isinstance(v0, (list, tuple)) and len(v0) == sizes[0]:
        out = []
        for v in values:
            out += list(v)
        return out
    return v0


def merge_jobs(group: Sequence[EvalJob]) -> EvalJob:
    """Concatenate the per-sample entries of several jobs along the batch dimension (non-batched entries must agree)."""
    if len(group) == 1:
        return group[0]
    sizes = [int(j.shape[0]) for j in group]
    kw = {}
    for k in group[0].model_kwargs:
        if k == "y":
            kw["y"] = {kk: _cat([j.model_kwargs["y"][kk] for j in group], sizes) for kk in group[0].model_kwargs["y"]}
        else:
            kw[k] = _cat([j.model_kwargs[k] for j in group], sizes)
    return EvalJob(group[0].batch_index, group[0].repeat, (sum(sizes),) + tuple(group[0].shape[1:]), kw, group[0].seed_number,
                   {"sizes": sizes})


def plan(jobs: Sequence[EvalJob], world: int, merge: int) -> List[List[int]]:
    """Units of work (lists of job indices run as ONE engine batch), in job order; unit u runs on rank u % world."""
    units, cur = [], []
    for idx, job in enumerate(jobs):
        if cur and (len(cur) >= merge or not _mergeable(jobs[cur[0]], job)):
            units.append(cur)
            cur = []
        cur.append(idx)
    if cur:
        units.append(cur)
    return units


def run_eval_jobs(diffusion, model, jobs: Sequence[EvalJob], sampler: str = "p_sample_loop", rng: str = "engine", seed: int = 0,
                  merge: int = 2, group=None, gather: bool = True, fixseed: Optional[Callable[[int], None]] = None,
                  **sampler_kwargs) -> Dict[int, torch.Tensor]:
    """Run every job's sampler call; returns {job index: sample (bs, njoints, nfeats, nframes)} -- all jobs when
    `gather`, else this rank's.

    rng="engine": motion m of job j draws its noise from (seed, first_motion_index(j) + m): independent of `merge` and of
    the world size.  rng="torch": `fixseed(job.seed_number)` (default torch.manual_seed) before each call and torch's
    generator stream inside it, one call per job (merge is forced to 1), as the reference loop does.
    """
    if getattr(diffusion, "window", None) is not None:
        raise NotImplementedError("run_eval_jobs does not run overlapping windows (diffusion.window)")
    world = dist.get_world_size(group) if dist.is_initialized() else 1
    rank = dist.get_rank(group) if dist.is_initialized() else 0
    if rng == "torch":
        merge = 1
    elif rng != "engine":
        raise ValueError("rng must be 'engine' or 'torch'")
    sampler_kwargs.setdefault("clip_denoised", False)  # :346
    units = plan(jobs, world, max(1, int(merge)))
    first_motion, n = [], 0
    for j in jobs:
        first_motion.append(n)
        n += int(j.shape[0])
    prev = (getattr(diffusion, "rng", "torch"), getattr(diffusion, "sample_offset", 0), getattr(diffusion, "engine_seed", None))
    mine: Dict[int, torch.Tensor] = {}
    try:
        for u, unit in enumerate(units):
            if u % world != rank:
                continue
            job = merge_jobs([jobs[i] for i in unit])
            if rng == "engine":
                diffusion.rng, diffusion.engine_seed, diffusion.sample_offset = "engine", int(seed), first_motion[unit[0]]
            else:
                diffusion.rng = "torch"
                (fixseed or torch.manual_seed)(int(job.seed_number))
            out = getattr(diffusion, sampler)(model, tuple(job.shape), model_kwargs=job.model_kwargs, **sampler_kwargs)
            lo = 0
            for i in unit:
                bs = int(jobs[i].shape[0])
                mine[i] = out[lo:lo + bs]
                lo += bs
    finally:
        diffusion.rng, diffusion.sample_offset, diffusion.engine_seed = prev
    if world == 1 or not gather:
        return mine
    # one exchange of finished samples: every rank contributes its jobs, padded to a common count
    per_rank = max(sum(len(unit) for u, unit in enumerate(units) if u % world == r) for r in range(world))
    proto = next(iter(mine.values())) if mine else None
    shapes = [None] * world
    dist.all_gather_object(shapes, None if proto is None else (tuple(proto.shape[1:]), str(proto.dtype)), group=group)
    tail = next(s for s in shapes if s is not None)
    dev = proto.device if proto is not None else (torch.device("cuda", torch.cuda.current_device()) if dist.get_backend(group) == "nccl"
                                                  else torch.device("cpu"))
    max_bs = max(int(j.shape[0]) for j in jobs)
    send = torch.zeros((per_rank, max_bs) + tuple(tail[0]), dtype=getattr(torch, tail[1].split(".")[-1]), device=dev)
    order = [i for u, unit in enumerate(units) if u % world == rank for i in unit]
    for slot, i in enumerate(order):
        send[slot, :mine[i].shape[0]] = mine[i]
    recv = torch.empty((world,) + tuple(send.shape), dtype=send.dtype, device=dev)
    dist.all_gather_into_tensor(recv.view(world * per_rank, *send.shape[1:]), send, group=group)
    out: Dict[int, torch.Tensor] = {}
    for r in range(world):
        order_r = [i for u, unit in enumerate(units) if u % world == r for i in unit]
        for slot, i in enumerate(order_r):
            out[i] = recv[r, slot, :int(jobs[i].shape[0])]
    return out

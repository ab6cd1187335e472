"""Restatement of classifier-free guidance limited to an interval of steps (y['stop_cfg_at'] / y['start_cfg_at'],
cmdi_sample_args.cfg_interval).

At the sampler's step index t (the spaced index under respacing), guidance is active while

    stop_cfg_at <= t <= start_cfg_at          (a missing bound does not limit)

Inside the interval the model call is the guided wrapper in use: CFG (Conditioning.cfg) or keyframe CFG
(keyframe_cfg_oracle.keyframe_cfg), as condmdi_oracle's model call finds it when the block is entered.  Outside it is the
inner model's conditional pass alone, the plain call with cfg off: text and keyframe input are kept and no scale is read.
That is not u + 1 (c - u), which differs from c in fp32.

`cfg_interval(tab, stop, start)` wraps condmdi_oracle's model call (its module-level `_model`), so the restated
p_mean_variance and every sampler restatement built on it (p_sample, ddim_sample, PLMS, DPM-Solver++, UniPC,
SDE-DPM-Solver++, RePaint, DDIM inversion), and the guidance and imputation they apply, see the model the interval
selects at each evaluation.  The model call receives the original timestep tab.timestep_map[t]; the block maps it back to
t (the map is strictly increasing).  oracle/make_golden_cfg_interval.py anchors it to the reference's own loops.
"""
from __future__ import annotations

import contextlib
import dataclasses
from typing import Optional

from oracle import condmdi_oracle as O

_plain_model = O._model  # the unwrapped model call (condmdi_oracle's own)


def active(t: int, stop: Optional[int], start: Optional[int]) -> bool:
    """Whether guidance runs at step index t."""
    return (stop is None or t >= stop) and (start is None or t <= start)


@contextlib.contextmanager
def cfg_interval(tab: O.DiffusionTables, stop: Optional[int] = None, start: Optional[int] = None):
    """Every model call of condmdi_oracle inside the block is the guided wrapper at the steps inside the interval and the
    inner model's conditional pass at the others."""
    guided = O._model
    step_of = {int(m): i for i, m in enumerate(tab.timestep_map)}

    def model(sd, x, t_model, c):
        steps = {step_of[int(v)] for v in t_model.reshape(-1).tolist()}
        assert len(steps) == 1, "the step index is uniform over the batch"
        if active(steps.pop(), stop, start):
            return guided(sd, x, t_model, c)
        return _plain_model(sd, x, t_model, dataclasses.replace(c, cfg=False))

    O._model = model
    try:
        yield
    finally:
        O._model = guided

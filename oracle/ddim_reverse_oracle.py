"""TEST INFRASTRUCTURE -- CPU restatement of the reference's DDIM inversion, built on the restatement of p_mean_variance
in `oracle/condmdi_oracle.py`:

    ddim_reverse_sample        diffusion/gaussian_diffusion.py:1418-1452 (eta = 0)
    ddim_reverse_sample_loop   for i in range(T): x = ddim_reverse_sample(x, [i] * B)["sample"]  (the reference has the
                               step only; this is the loop a user writes around it)

Pinned against the unmodified reference by `oracle/make_golden_ddim_reverse.py`, which writes tests/golden/ddim_reverse.*
that `tests/test_ddim_reverse_oracle.py` re-checks wherever the suite runs.  Like condmdi_oracle, only `tests/` may
import it.
"""
from __future__ import annotations

from typing import Optional

import numpy as np
import torch

from oracle.condmdi_oracle import Conditioning, DiffusionTables, extract, p_mean_variance


def alphas_cumprod_next(tab: DiffusionTables) -> np.ndarray:
    """GaussianDiffusion.__init__ (gaussian_diffusion.py:194): float64, last entry 0."""
    return np.append(tab.alphas_cumprod[1:], 0.0)


def reverse_update(tab: DiffusionTables, x: torch.Tensor, t: torch.Tensor, pred_xstart: torch.Tensor) -> torch.Tensor:
    """The update of ddim_reverse_sample after p_mean_variance (:1442-1450), given its pred_xstart."""
    eps = (extract(tab.sqrt_recip_alphas_cumprod, t, x.shape) * x - pred_xstart) / \
        extract(tab.sqrt_recipm1_alphas_cumprod, t, x.shape)
    alpha_bar_next = extract(alphas_cumprod_next(tab), t, x.shape)
    return pred_xstart * torch.sqrt(alpha_bar_next) + torch.sqrt(1 - alpha_bar_next) * eps


def ddim_reverse_sample(sd, tab: DiffusionTables, x: torch.Tensor, t: torch.Tensor, c: Conditioning, eta: float = 0.0):
    """ddim_reverse_sample (gaussian_diffusion.py:1418-1452): x_t -> x_{t+1}."""
    assert eta == 0.0, "Reverse ODE only for deterministic path"
    out = p_mean_variance(sd, tab, x, t, c)
    return {"sample": reverse_update(tab, x, t, out["pred_xstart"]), "pred_xstart": out["pred_xstart"]}


def ddim_reverse_sample_loop(sd, tab: DiffusionTables, x_start: torch.Tensor, c: Conditioning, t_start: int = 0,
                             max_steps: Optional[int] = None, return_all: bool = False):
    """x_start at step index t_start, inverted step by step up to t = T - 1 (max_steps: stop after that many).
    return_all: every step's dict; otherwise the last sample."""
    x = x_start.clone()
    outs, out = [], None
    with torch.no_grad():
        for k, i in enumerate(range(t_start, tab.num_timesteps)):
            if max_steps is not None and k >= max_steps:
                break
            out = ddim_reverse_sample(sd, tab, x, torch.tensor([i] * x.shape[0]), c)
            if return_all:
                outs.append(out)
            x = out["sample"]
    return outs if return_all else x

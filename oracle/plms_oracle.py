"""TEST INFRASTRUCTURE -- CPU restatement of the reference's PLMS sampler (pseudo linear multistep), built on the
restatement of p_mean_variance in `oracle/condmdi_oracle.py`:

    plms_sample            diffusion/gaussian_diffusion.py:1589-1687 (cond_fn = None)
    plms_sample_loop       :1689-1804 (noise tape instead of the global generator; only tape[0] is drawn)

Pinned against the unmodified reference by `oracle/make_golden_plms.py`, which writes tests/golden/plms.* that
`tests/test_plms_oracle.py` re-checks wherever the suite runs.  Like condmdi_oracle, only `tests/` may import it.
"""
from __future__ import annotations

from typing import List, Optional, Sequence

import torch

from oracle.condmdi_oracle import Conditioning, DiffusionTables, extract, p_mean_variance


def plms_check_order(order) -> None:
    """The argument checks of plms_sample (gaussian_diffusion.py:1608-1609), plus the two orders the reference accepts
    there and then fails on later: order 1 (old_out["old_eps"] on None at the first step, a TypeError) and non-integral
    orders in (1, 4] (the Adams-Bashforth branch has no weights for them)."""
    if not int(order) or not 1 <= order <= 4:
        raise ValueError("order is invalid (should be int from 1-4).")
    if order != int(order):
        raise NotImplementedError(f"PLMS order {order!r} is not an integer")
    if int(order) == 1:
        raise TypeError("PLMS order 1 fails on the first step of the reference ('NoneType' object is not subscriptable)")


def plms_sample(sd, tab: DiffusionTables, x: torch.Tensor, t: torch.Tensor, c: Conditioning, order: int = 2,
                old_eps: Optional[List[torch.Tensor]] = None):
    """plms_sample with cond_fn=None (gaussian_diffusion.py:1589-1687).  old_eps: the previous step's history list, or
    None on the first step of a loop.  The returned "old_eps" is a new list (the reference mutates its list in place)."""
    plms_check_order(order)
    r1, r2 = tab.sqrt_recip_alphas_cumprod, tab.sqrt_recipm1_alphas_cumprod

    def model_eps(x_, t_):
        out = p_mean_variance(sd, tab, x_, t_, c)
        eps = (extract(r1, t_, x_.shape) * x_ - out["pred_xstart"]) / extract(r2, t_, x_.shape)  # :551-555
        return eps, out

    def xstart_from_eps(e):  # :536-541
        return extract(r1, t, x.shape) * x - extract(r2, t, x.shape) * e

    alpha_bar_prev = extract(tab.alphas_cumprod_prev, t, x.shape)
    eps, out = model_eps(x, t)
    if old_eps is None:
        # pseudo improved Euler (:1647-1656); the second evaluation is at t - 1 (at t = 0 that is index -1, the last
        # table entry, as torch indexes it: the result is discarded by the nonzero mask below)
        hist = [eps]
        mean_pred = out["pred_xstart"] * torch.sqrt(alpha_bar_prev) + torch.sqrt(1 - alpha_bar_prev) * eps
        eps_2, _ = model_eps(mean_pred, t - 1)
        eps_prime = (eps + eps_2) / 2
    else:
        # pseudo linear multistep, Adams-Bashforth (:1657-1675)
        hist = list(old_eps) + [eps]
        cur_order = min(order, len(hist))
        if cur_order == 1:
            eps_prime = hist[-1]
        elif cur_order == 2:
            eps_prime = (3 * hist[-1] - hist[-2]) / 2
        elif cur_order == 3:
            eps_prime = (23 * hist[-1] - 16 * hist[-2] + 5 * hist[-3]) / 12
        else:
            eps_prime = (55 * hist[-1] - 59 * hist[-2] + 37 * hist[-3] - 9 * hist[-4]) / 24
    pred_prime = xstart_from_eps(eps_prime)
    mean_pred = pred_prime * torch.sqrt(alpha_bar_prev) + torch.sqrt(1 - alpha_bar_prev) * eps_prime
    if len(hist) >= order:
        hist.pop(0)
    nonzero = (t != 0).float().view(-1, *([1] * (len(x.shape) - 1)))
    sample = mean_pred * nonzero + out["pred_xstart"] * (1 - nonzero)
    return {"sample": sample, "pred_xstart": out["pred_xstart"], "old_eps": hist}


def plms_sample_loop(sd, tab: DiffusionTables, shape: Sequence[int], c: Conditioning, tape: torch.Tensor, order: int = 2,
                     skip_timesteps: int = 0, init_image: Optional[torch.Tensor] = None, max_steps: Optional[int] = None,
                     return_all: bool = False):
    """plms_sample_loop(_progressive) (gaussian_diffusion.py:1689-1804).  tape[0] is the initial randn(*shape) draw; the
    loop draws nothing else.  max_steps (test aid): stop after that many iterations.  return_all: every step's dict."""
    plms_check_order(order)
    img = tape[0].clone()
    if skip_timesteps and init_image is None:
        init_image = torch.zeros_like(img)
    indices = list(range(tab.num_timesteps - skip_timesteps))[::-1]
    if init_image is not None:
        my_t = torch.ones([shape[0]], dtype=torch.long) * indices[0]
        img = extract(tab.sqrt_alphas_cumprod, my_t, img.shape) * init_image + \
            extract(tab.sqrt_one_minus_alphas_cumprod, my_t, img.shape) * img  # q_sample (:311-328)
    outs, out = [], None
    with torch.no_grad():
        for k, i in enumerate(indices):
            if max_steps is not None and k >= max_steps:
                break
            out = plms_sample(sd, tab, img, torch.tensor([i] * shape[0]), c, order, None if out is None else out["old_eps"])
            if return_all:
                outs.append(out)
            img = out["sample"]
    return outs if return_all else out["sample"]

"""TEST INFRASTRUCTURE -- CPU restatement of the engine's SDE-DPM-Solver++ multistep sampler (Lu et al. 2022, "DPM-Solver++:
Fast Solver for Guided Sampling of Diffusion Probabilistic Models"; the SDE solver in data prediction, midpoint form),
built on the restatement of p_mean_variance in `oracle/condmdi_oracle.py`.  The reference has no such sampler; its order 1
is the DDPM posterior step, and `oracle/make_golden_dpm_solver_sde.py` pins that against the reference's p_sample_loop.

    step grid      the spaced steps s = T' - 1 - skip_timesteps, ..., 0; the step at s moves from abar_s = alphas_cumprod[s]
                   to abar_u = alphas_cumprod_prev[s]
    x0             m0 = pred_xstart of p_mean_variance at (x_s, s): CFG, keyframe input, imputation, guidance
    update         alpha = sqrt(abar), sigma = sqrt(1 - abar), lambda = log alpha - log sigma, h = lambda_u - lambda_s,
                   e = 1 - exp(-2h) = -expm1(-2h), z the step's standard normal draw
                     order 1: x_u = (sigma_u / sigma_s) exp(-h) x_s + alpha_u e m0 + sigma_u sqrt(e) z
                     order 2: ... + alpha_u e D1_0 / 2,  D1_0 = (m0 - m1) / r0,  r0 = (lambda_s - lambda_{s+1}) / h
    order          min(order, k + 1, s + 1) at loop iteration k; the last step (abar_u = 1) returns m0
    noise          p_sample_loop's: tape[0] is x_T, tape[1 + k] the draw of loop iteration k (drawn at every step,
                   the last included, whose value is not used)

The loop folds each step into x_u = A x_s + B0 m0 + B1 m1 + Cn z with a float64 table rounded to fp32, as the engine
does.  Like condmdi_oracle, only `tests/` and `oracle/` may import it.
"""
from __future__ import annotations

from typing import Optional, Sequence

import numpy as np
import torch

from oracle.condmdi_oracle import Conditioning, DiffusionTables, extract, p_mean_variance
from oracle.dpm_solver_oracle import effective_order, lambdas


def check_order(order) -> None:
    if isinstance(order, bool) or not isinstance(order, (int, np.integer)) or int(order) not in (1, 2):
        raise ValueError(f"SDE-DPM-Solver++ order must be an int in {{1, 2}}, got {order!r}")


def unfolded_update(tab: DiffusionTables, s: int, eff: int, x, m0, m1=None, z=None):
    """One step from the formulas as the module docstring states them (float64 in, float64 out)."""
    if s == 0:
        return m0
    lam = lambdas(tab)
    acp_s, acp_u = tab.alphas_cumprod[s], tab.alphas_cumprod_prev[s]
    alpha_u, sigma_u, sigma_s = np.sqrt(acp_u), np.sqrt(1.0 - acp_u), np.sqrt(1.0 - acp_s)
    h = lam[s - 1] - lam[s]
    e = -np.expm1(-2.0 * h)
    x_u = (sigma_u / sigma_s) * np.exp(-h) * x + alpha_u * e * m0 + sigma_u * np.sqrt(e) * z
    if eff == 1:
        return x_u
    r0 = (lam[s] - lam[s + 1]) / h
    return x_u + 0.5 * alpha_u * e * (m0 - m1) / r0


def coefficient_table(tab: DiffusionTables, t_start: int, order: int) -> np.ndarray:
    """[T', 4] float64 (A, B0, B1, Cn) per step index of a history started at t_start; rows above t_start are zero."""
    check_order(order)
    lam = lambdas(tab)
    out = np.zeros((tab.num_timesteps, 4))
    for s in range(t_start + 1):
        if s == 0:
            out[s] = (0.0, 1.0, 0.0, 0.0)
            continue
        eff = effective_order(order, t_start - s, s)
        acp_u = tab.alphas_cumprod_prev[s]
        alpha_u, sigma_u = np.sqrt(acp_u), np.sqrt(1.0 - acp_u)
        h = lam[s - 1] - lam[s]
        e = -np.expm1(-2.0 * h)
        A = sigma_u / np.sqrt(1.0 - tab.alphas_cumprod[s]) * np.exp(-h)
        B0, B1 = alpha_u * e, 0.0
        if eff == 2:
            c = 0.5 * alpha_u * e / ((lam[s] - lam[s + 1]) / h)
            B0, B1 = B0 + c, -c
        out[s] = (A, B0, B1, sigma_u * np.sqrt(e))
    return out


def dpm_solver_sde_sample_loop(sd, tab: DiffusionTables, shape: Sequence[int], c: Conditioning, tape: torch.Tensor,
                               order: int = 2, skip_timesteps: int = 0, init_image: Optional[torch.Tensor] = None,
                               max_steps: Optional[int] = None, return_all: bool = False):
    """The engine's dpm_solver_sde_sample_loop(_progressive).  tape[0] is x_T, tape[1 + k] the draw of iteration k;
    skip_timesteps / init_image as p_sample_loop (q_sample with x_T as the noise).  max_steps: stop after that many
    iterations.  return_all: every step's {"sample", "pred_xstart"}."""
    check_order(order)
    img = tape[0].clone()
    if skip_timesteps and init_image is None:
        init_image = torch.zeros_like(img)
    t_start = tab.num_timesteps - 1 - skip_timesteps
    if init_image is not None:
        my_t = torch.ones([shape[0]], dtype=torch.long) * t_start
        img = extract(tab.sqrt_alphas_cumprod, my_t, img.shape) * init_image + \
            extract(tab.sqrt_one_minus_alphas_cumprod, my_t, img.shape) * img  # q_sample (:311-328)
    coef = torch.from_numpy(coefficient_table(tab, t_start, order)).to(img.dtype)
    m1, outs = None, []
    with torch.no_grad():
        for k, s in enumerate(range(t_start, -1, -1)):
            if max_steps is not None and k >= max_steps:
                break
            m0 = p_mean_variance(sd, tab, img, torch.tensor([s] * shape[0]), c)["pred_xstart"]
            A, B0, B1, Cn = coef[s]
            x = A * img + B0 * m0
            if effective_order(order, k, s) >= 2:
                x = x + B1 * m1
            x = x + Cn * tape[1 + k] if s > 0 else m0
            m1, img = m0, x
            if return_all:
                outs.append({"sample": img, "pred_xstart": m0})
    return outs if return_all else img


def gaussian_std_error(tab: DiffusionTables, order: int, data_std: float, data_mean: float = 0.5) -> float:
    """|std(x0) - data_std| of the loop's samples, exactly, for data x0 ~ N(data_mean, data_std^2) per element and the
    exact denoiser m(x_s) = E[x0 | x_s] = a_s x_s + b_s (a_s = alpha_s d^2 / (alpha_s^2 d^2 + sigma_s^2), b_s = mu (1 - a_s
    alpha_s)).  Every step is linear in (x_s, m1) plus independent noise, so the law of the state stays Gaussian: its
    mean and 2 x 2 covariance are propagated through the folded table, from x_T ~ N(0, 1).  Float64; no sampling."""
    coef = coefficient_table(tab, tab.num_timesteps - 1, order)
    acp = tab.alphas_cumprod
    d2 = data_std ** 2
    mean, cov = np.zeros(2), np.diag([1.0, 0.0])  # (x_s, m1)
    for s in range(tab.num_timesteps - 1, -1, -1):
        al, si2 = np.sqrt(acp[s]), 1.0 - acp[s]
        a = al * d2 / (acp[s] * d2 + si2)
        b = data_mean * (1.0 - a * al)
        if s == 0:
            return abs(abs(a) * np.sqrt(cov[0, 0]) - data_std)  # the sample is m0
        A, B0, B1, Cn = coef[s]
        M = np.array([[A + B0 * a, B1], [a, 0.0]])
        mean = M @ mean + np.array([B0 * b, b])
        cov = M @ cov @ M.T + np.diag([Cn ** 2, 0.0])
    raise AssertionError("unreachable")

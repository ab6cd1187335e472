"""Foot-contact guidance, restated for the tests: p_mean_variance of `oracle/joint_guidance_oracle.py` with a third loss
against foot sliding.  The reference uses foot contacts only at training time (its `fc` term); this is the sampling-time
semantics the engine implements (include/condmdi_b200.h, cmdi_sample_args.foot_contact):

    P(x0_hat)      = recover_from_ric(x0_hat^T * std + mean, 22, abs_3d)                      (B, L, 22, 3)
    kappa(b, f, k) = [channel 259 + k of x0_hat^T * std + mean > 0.5]                         a constant, J = (7, 10, 8, 11)
    L_c            = sum_{b, f <= L - 2, k} kappa(b, f, k) m(b, f) m(b, f + 1) |P_{J_k}(f + 1) - P_{J_k}(f)|^2
    c_c(t)         = w_c[t] * weight * sqrt(alpha_bar_t) / 2                                  0 while t < stop_footcontact_at
    x0_tilde       = x0_hat - ~M * (c_r(t) dL_r/dz + c_j(t) dL_j/dz + c_c(t) dL_c/dz)

with m = y['mask'] (the valid frames), L_r, c_r and M reconstruction guidance's and L_j, c_j joint guidance's (both 0
when off).  Channel 259 + k at frame f is the label foot_detect computes from the move f -> f + 1, so it weights that
displacement.  Every tensor stays on the caller's device and dtype.  `foot_contact_guided(fc, j)` routes condmdi_oracle's
samplers through it.
"""
from __future__ import annotations

import contextlib
from dataclasses import dataclass
from typing import Optional

import torch

from oracle import condmdi_oracle as O
from oracle import joint_guidance_oracle as J

FOOT_JOINTS = (7, 10, 8, 11)   # feet_l (7, 10), feet_r (8, 11): motion_process.py's foot_detect order
CONTACT_CHANNEL = 259          # channels 259 .. 262 of the 263-d HumanML3D vector

_P_MEAN_VARIANCE = O.p_mean_variance


def contact_weights(x0: torch.Tensor, mean: torch.Tensor, std: torch.Tensor, valid: Optional[torch.Tensor]) -> torch.Tensor:
    """kappa(b, f, k) m(b, f) m(b, f + 1) for f = 0 .. L - 2: (B, L - 1, 4) in x0's dtype, with no gradient.
    x0 (B, 263, 1, L) normalised; valid (B, L) (any layout with B * L entries) or None: every frame valid."""
    B, L = x0.shape[0], x0.shape[-1]
    data = x0.detach()[:, CONTACT_CHANNEL:CONTACT_CHANNEL + 4, 0].transpose(1, 2) * \
        std[CONTACT_CHANNEL:CONTACT_CHANNEL + 4].to(x0) + mean[CONTACT_CHANNEL:CONTACT_CHANNEL + 4].to(x0)
    kappa = data > 0.5                                                       # (B, L, 4)
    m = torch.ones(B, L, dtype=torch.bool, device=x0.device) if valid is None else valid.to(x0.device).reshape(B, L).bool()
    return (kappa[:, :-1] & m[:, :-1, None] & m[:, 1:, None]).to(x0.dtype)


def contact_loss(x0, mean, std, abs_3d, valid=None) -> torch.Tensor:
    """L_c (module docstring)"""
    w = contact_weights(x0, mean, std, valid)
    P = J.joint_positions(x0, mean, std, abs_3d)[:, :, list(FOOT_JOINTS)]   # (B, L, 4, 3)
    return ((P[:, 1:] - P[:, :-1]).square().sum(-1) * w).sum()


def contact_seed(x0, mean, std, abs_3d, valid=None) -> torch.Tensor:
    """dL_c/dx0 by autograd (the engine's cmdi_foot_contact_seed with c_c = 1 and no joint term)"""
    with torch.enable_grad():
        z = x0.detach().requires_grad_(True)
        return torch.autograd.grad(contact_loss(z, mean, std, abs_3d, valid), z)[0]


@dataclass
class FootContactTerm:
    """y['foot_contact_*'] and diffusion.joint_space, reduced to tensors; m is y['mask'] (Conditioning.y_mask)."""
    mean: torch.Tensor                   # (263,)
    std: torch.Tensor
    abs_3d: bool = True
    weight: float = 1.0
    gradient_schedule: Optional[str] = None
    diffusion_steps: int = 1000
    stop_footcontact_at: int = 0


def p_mean_variance(sd, tab: O.DiffusionTables, x: torch.Tensor, t: torch.Tensor, c: O.Conditioning, fc: FootContactTerm,
                    j: Optional[J.JointTerm] = None):
    """condmdi_oracle.p_mean_variance with the foot-contact term and, when j is given, the joint term (module docstring)."""
    need_fc = bool((t >= fc.stop_footcontact_at).all())
    need_jg = j is not None and bool((t >= j.stop_jointguidance_at).all())
    if not need_fc:
        return J.p_mean_variance(sd, tab, x, t, c, j) if j is not None else _P_MEAN_VARIANCE(sd, tab, x, t, c)
    dev = x.device
    t_model = torch.tensor(tab.timestep_map, dtype=t.dtype)[t]
    B, L = x.shape[0], x.shape[-1]
    y_mask = c.y_mask.to(dev) if c.y_mask is not None else torch.ones(B, 1, 1, L, dtype=torch.bool, device=dev)
    keyframes = c.reconstruction_guidance or (c.imputate and c.replacement_distribution == "conditional")
    M = (c.inpainting_mask.to(dev) & y_mask.bool()) if keyframes else torch.zeros_like(x, dtype=torch.bool)
    need_rg = c.reconstruction_guidance and bool((t >= c.stop_recguidance_at).all())
    need_imp = keyframes and c.imputate and bool((t >= c.stop_imputation_at).all())
    with torch.enable_grad():
        z = x.detach().requires_grad_(True)
        hat_x = O._model(sd, z, t_model, c)
        grad = J._coef(fc.gradient_schedule, fc.diffusion_steps, fc.weight, tab, t, x.shape, dev) * torch.autograd.grad(
            contact_loss(hat_x, fc.mean, fc.std, fc.abs_3d, y_mask), z, retain_graph=need_jg or need_rg)[0]
        if need_jg:
            Mj = j.mask.to(dev) & y_mask.reshape(B, L)[:, :, None, None].bool()
            g_j = torch.autograd.grad(J.joint_loss(hat_x, j.target, Mj, j.mean, j.std, j.abs_3d), z, retain_graph=need_rg)[0]
            grad = J._coef(j.gradient_schedule, j.diffusion_steps, j.weight, tab, t, x.shape, dev) * g_j + grad
        if need_rg:
            loss_r = ((c.inpainted_motion.to(dev) - hat_x).square() * M).sum()
            g_r = torch.autograd.grad(loss_r, z)[0]
            grad = J._coef(c.gradient_schedule, c.diffusion_steps, c.reconstruction_weight, tab, t, x.shape, dev) * g_r + grad
    hat_x = hat_x.detach()
    tilde = hat_x - grad * (~M).to(hat_x)
    model_output = (tilde * ~M) + (c.inpainted_motion.to(dev) * M) if need_imp else (tilde * ~M) + (hat_x * M)
    log_variance = O.extract(tab.posterior_log_variance_clipped, t, x.shape).to(dev)
    mean = O.extract(tab.posterior_mean_coef1, t, x.shape).to(dev) * model_output + \
        O.extract(tab.posterior_mean_coef2, t, x.shape).to(dev) * x
    return {"mean": mean, "log_variance": log_variance, "pred_xstart": model_output, "model_output": model_output}


@contextlib.contextmanager
def foot_contact_guided(fc: FootContactTerm, j: Optional[J.JointTerm] = None):
    """condmdi_oracle's samplers (sample_loop, p_sample, ddim_sample; so also repaint_oracle's walk) and
    dpm_solver_oracle's loop with the foot-contact term (and the joint term when j is given) in p_mean_variance"""
    from oracle import dpm_solver_oracle as S
    pmv = lambda sd, tab, x, t, c: p_mean_variance(sd, tab, x, t, c, fc, j)  # noqa: E731
    O.p_mean_variance = S.p_mean_variance = pmv
    try:
        yield
    finally:
        O.p_mean_variance = S.p_mean_variance = _P_MEAN_VARIANCE


def inputs(B: int, L: int = 196, seed: int = 0, contact_rate: float = 0.5):
    """Seeded foot-contact inputs: joint_guidance_oracle.inputs' statistics, with the contact channels' statistics set
    so that a standard-normal x0 marks about `contact_rate` of the frames as in contact (mean 0.5 - std * q, q the
    standard normal's (1 - contact_rate) quantile, std 0.5), and x0 (B, 263, 1, L) standard normal."""
    mean, std, _, _, g = J.inputs(B, L, seed=seed)
    q = torch.distributions.Normal(0.0, 1.0).icdf(torch.tensor(1.0 - contact_rate)).item()
    std[CONTACT_CHANNEL:CONTACT_CHANNEL + 4] = 0.5
    mean[CONTACT_CHANNEL:CONTACT_CHANNEL + 4] = 0.5 - 0.5 * q
    x0 = torch.randn(B, 263, 1, L, generator=g)
    return mean, std, x0, g

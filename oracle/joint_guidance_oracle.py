"""Joint-position guidance, restated for the tests: p_mean_variance of `oracle/condmdi_oracle.py` with a second loss on
world-space joint positions.  The reference has no such guidance; this is the semantics the engine implements
(include/condmdi_b200.h, cmdi_sample_args.joint_guidance):

    P(x0_hat) = recover_from_ric(x0_hat^T * std + mean, 22, abs_3d)                  (B, L, 22, 3)
    L_j       = sum(M_j * (P(x0_hat(z)) - target)^2)                                 M_j = joint mask & y['mask']
    c_j(t)    = w_j[t] * weight * sqrt(alpha_bar_t) / 2                               0 while t < stop_jointguidance_at
    x0_tilde  = x0_hat - ~M * (c_r(t) dL_r/dz + c_j(t) dL_j/dz)

with L_r, c_r and M reconstruction guidance's (c_r = 0 when it is off or t < stop_recguidance_at), then imputation as
before.  The feature keyframes are those p_mean_variance reads: with reconstruction guidance on, or with imputation from
the 'conditional' replacement distribution; otherwise (none given, or imputation from the 'marginal' one, which only
calls the model) M = 0 and nothing is imputed.  Every tensor stays on the caller's device and dtype, so the GPU tests
run it in fp32, under CUDA autocast or in fp64.  `joint_guided(j)` routes condmdi_oracle's samplers through it.
"""
from __future__ import annotations

import contextlib
from dataclasses import dataclass
from typing import Optional

import torch

from oracle import condmdi_oracle as O

JOINTS = 22

_P_MEAN_VARIANCE = O.p_mean_variance


def recover_from_ric(data: torch.Tensor, abs_3d: bool) -> torch.Tensor:
    """condmdi_oracle.recover_from_ric for the 22-joint skeleton in the same operation order, with its intermediates on
    data's device and dtype: (..., frames, 263) de-normalised -> (..., frames, 22, 3)."""
    if abs_3d:
        ang = data[..., 0]
    else:
        ang = torch.zeros_like(data[..., 0])
        ang[..., 1:] = data[..., :-1, 0]
        ang = torch.cumsum(ang, dim=-1)
    cos_a, sin_a = torch.cos(ang), torch.sin(ang)
    root = data.new_zeros(data.shape[:-1] + (3,))
    if abs_3d:
        root[..., 0], root[..., 2] = data[..., 1], data[..., 2]
    else:
        root[..., 1:, 0], root[..., 1:, 2] = data[..., :-1, 1], data[..., :-1, 2]
        root = torch.cumsum(O._rotate_about_y(cos_a, sin_a, root), dim=-2)
    root[..., 1] = data[..., 3]
    local = data[..., 4:(JOINTS - 1) * 3 + 4].reshape(data.shape[:-1] + (JOINTS - 1, 3))
    pos = O._rotate_about_y(cos_a[..., None], sin_a[..., None], local)
    pos = torch.stack((pos[..., 0] + root[..., None, 0], pos[..., 1], pos[..., 2] + root[..., None, 2]), -1)
    return torch.cat((root[..., None, :], pos), dim=-2)


def joint_positions(x0: torch.Tensor, mean: torch.Tensor, std: torch.Tensor, abs_3d: bool) -> torch.Tensor:
    """x0 (B, 263, 1, L) normalised -> world-space joints (B, L, 22, 3)."""
    data = x0[:, :, 0].transpose(1, 2) * std.to(x0) + mean.to(x0)
    return recover_from_ric(data, abs_3d)


def joint_loss(x0, target, mask, mean, std, abs_3d) -> torch.Tensor:
    """sum(mask * (P(x0) - target)^2)"""
    return ((joint_positions(x0, mean, std, abs_3d) - target.to(x0)).square() * mask.to(x0)).sum()


def joint_seed(x0, target, mask, mean, std, abs_3d) -> torch.Tensor:
    """dL_j/dx0 by autograd (the engine's cmdi_joint_guidance_seed)"""
    with torch.enable_grad():
        z = x0.detach().requires_grad_(True)
        return torch.autograd.grad(joint_loss(z, target, mask, mean, std, abs_3d), z)[0]


@dataclass
class JointTerm:
    """y['joint_*'] and diffusion.joint_space, reduced to tensors."""
    target: torch.Tensor                 # (B, L, 22, 3)
    mask: torch.Tensor                   # bool (B, L, 22, 3), y['mask'] not yet folded in
    mean: torch.Tensor                   # (263,)
    std: torch.Tensor
    abs_3d: bool = True
    weight: float = 1.0
    gradient_schedule: Optional[str] = None
    diffusion_steps: int = 1000
    stop_jointguidance_at: int = 0


def _coef(schedule, steps, weight, tab, t, shape, device):
    """w[t] * weight * sqrt(alpha_bar_t) / 2 in fp32, as condmdi_oracle.p_mean_variance forms it"""
    w = O.extract(O.get_gradient_schedule(schedule, steps), t, shape) * weight
    return (w * O.extract(tab.sqrt_alphas_cumprod, t, shape) / 2).to(device)


def p_mean_variance(sd, tab: O.DiffusionTables, x: torch.Tensor, t: torch.Tensor, c: O.Conditioning, j: JointTerm):
    """condmdi_oracle.p_mean_variance with the joint term (module docstring)."""
    need_jg = bool((t >= j.stop_jointguidance_at).all())
    if not need_jg:
        return _P_MEAN_VARIANCE(sd, tab, x, t, c)
    dev = x.device
    t_model = torch.tensor(tab.timestep_map, dtype=t.dtype)[t]
    B, L = x.shape[0], x.shape[-1]
    y_mask = c.y_mask.to(dev) if c.y_mask is not None else torch.ones(B, 1, 1, L, dtype=torch.bool, device=dev)
    keyframes = c.reconstruction_guidance or (c.imputate and c.replacement_distribution == "conditional")
    M = (c.inpainting_mask.to(dev) & y_mask.bool()) if keyframes else torch.zeros_like(x, dtype=torch.bool)
    Mj = j.mask.to(dev) & y_mask.reshape(B, L)[:, :, None, None].bool()
    need_rg = c.reconstruction_guidance and bool((t >= c.stop_recguidance_at).all())
    need_imp = keyframes and c.imputate and bool((t >= c.stop_imputation_at).all())
    with torch.enable_grad():
        z = x.detach().requires_grad_(True)
        hat_x = O._model(sd, z, t_model, c)
        grad = _coef(j.gradient_schedule, j.diffusion_steps, j.weight, tab, t, x.shape, dev) * torch.autograd.grad(
            joint_loss(hat_x, j.target, Mj, j.mean, j.std, j.abs_3d), z, retain_graph=need_rg)[0]
        if need_rg:
            loss_r = ((c.inpainted_motion.to(dev) - hat_x).square() * M).sum()
            g_r = torch.autograd.grad(loss_r, z)[0]
            grad = _coef(c.gradient_schedule, c.diffusion_steps, c.reconstruction_weight, tab, t, x.shape, dev) * g_r + grad
    hat_x = hat_x.detach()
    tilde = hat_x - grad * (~M).to(hat_x)
    model_output = (tilde * ~M) + (c.inpainted_motion.to(dev) * M) if need_imp else (tilde * ~M) + (hat_x * M)
    log_variance = O.extract(tab.posterior_log_variance_clipped, t, x.shape).to(dev)
    mean = O.extract(tab.posterior_mean_coef1, t, x.shape).to(dev) * model_output + \
        O.extract(tab.posterior_mean_coef2, t, x.shape).to(dev) * x
    return {"mean": mean, "log_variance": log_variance, "pred_xstart": model_output, "model_output": model_output}


@contextlib.contextmanager
def joint_guided(j: JointTerm):
    """condmdi_oracle's samplers (sample_loop, p_sample, ddim_sample; so also repaint_oracle's walk) and
    dpm_solver_oracle's loop with the joint term in p_mean_variance"""
    from oracle import dpm_solver_oracle as S
    pmv = lambda sd, tab, x, t, c: p_mean_variance(sd, tab, x, t, c, j)  # noqa: E731
    O.p_mean_variance = S.p_mean_variance = pmv
    try:
        yield
    finally:
        O.p_mean_variance = S.p_mean_variance = _P_MEAN_VARIANCE


def inputs(B: int, L: int = 196, seed: int = 0):
    """Seeded joint-guidance inputs: statistics (mean, std) of dataset-like size, a random target and a sparse mask: the
    pelvis XZ on every frame, and all joints on every (L // 4)-th frame."""
    g = torch.Generator().manual_seed(seed)
    mean = torch.randn(263, generator=g) * 0.1
    std = 0.05 + torch.rand(263, generator=g) * 0.5
    mask = torch.zeros(B, L, 22, 3, dtype=torch.bool)
    mask[:, :, 0, 0] = mask[:, :, 0, 2] = True
    mask[:, ::max(1, L // 4), :, :] = True
    target = torch.randn(B, L, 22, 3, generator=g)
    return mean, std, target, mask, g

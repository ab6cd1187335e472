"""Obstacle-avoidance guidance, restated for the tests: p_mean_variance of `oracle/foot_contact_oracle.py` with a fourth
loss that keeps chosen joints out of vertical cylinders.  This is GMD's collision term (the reference's
sample/gmd/condition.py, CondKeyLocationsWithSdf: `dist = clamp(rad - |trajec[:, :, [0, 2]] - cent|, min=0)`,
`loss_colli += dist.sum() / trajec.shape[1]`) over the whole motion, generalised to per-sample obstacles, any joint set
and ragged masks; the semantics the engine implements (include/condmdi_b200.h, cmdi_sample_args.obstacle_guidance):

    P(x0_hat) = recover_from_ric(x0_hat^T * std + mean, 22, abs_3d)                                  (B, L, 22, 3)
    L_o       = sum_b (1 / L) sum_{f, j in S, k} m(b, f) max(r_k - |(P_j^x, P_j^z)(b, f) - (c_x, c_z)_k|, 0)
    c_o(t)    = w_o[t] * weight * sqrt(alpha_bar_t) / 2                             0 while t < stop_obstacleguidance_at
    x0_tilde  = x0_hat - ~M * (c_r(t) dL_r/dz + c_j(t) dL_j/dz + c_c(t) dL_c/dz + c_o(t) dL_o/dz)

with obstacles o_k = (c_x, c_z, r_k) per sample ((B, K, 3); r = 0 rows are padding), S the joint set (GMD: {0}, the
pelvis), m = y['mask'], and the other terms those of foot_contact_oracle (0 when off).  GMD's w_colli and
classifiler_scale fold into the weight.  The gradient is torch's: at distance 0 the norm's backward gives 0, at distance
r the clamp passes it.  Every tensor stays on the caller's device and dtype.  `obstacle_guided(ob, fc, j)` routes
condmdi_oracle's samplers through it.
"""
from __future__ import annotations

import contextlib
from dataclasses import dataclass
from typing import Optional, Sequence

import torch

from oracle import condmdi_oracle as O
from oracle import foot_contact_oracle as FC
from oracle import joint_guidance_oracle as J

MAX_OBSTACLES = 16

_P_MEAN_VARIANCE = O.p_mean_variance


def obstacles_from_list(obs_list, B: int) -> torch.Tensor:
    """GMD's obs_list [((c_x, c_z), r), ...], shared by the batch, as the (B, K, 3) fp32 tensor form"""
    rows = [[float(cx), float(cz), float(r)] for (cx, cz), r in obs_list]
    return torch.tensor(rows, dtype=torch.float32).reshape(1, len(rows), 3).expand(B, -1, -1).contiguous()


def obstacle_loss(x0, mean, std, abs_3d, obstacles, joints: Sequence[int] = (0,), valid=None) -> torch.Tensor:
    """L_o (module docstring); x0 (B, 263, 1, L) normalised, obstacles (B, K, 3), valid (B, L) (any layout with B * L
    entries) or None: every frame valid"""
    B, L = x0.shape[0], x0.shape[-1]
    P = J.joint_positions(x0, mean, std, abs_3d)[:, :, list(joints)][..., [0, 2]]          # (B, L, |S|, 2)
    obs = obstacles.to(x0)
    dist = torch.norm(P[:, :, :, None, :] - obs[:, None, None, :, :2], dim=-1)             # (B, L, |S|, K)
    pen = torch.clamp(obs[:, None, None, :, 2] - dist, min=0.0)
    m = torch.ones(B, L, dtype=x0.dtype, device=x0.device) if valid is None else \
        valid.to(x0.device).reshape(B, L).to(x0.dtype)
    return (pen.sum((-1, -2)) * m).sum() / L


def obstacle_seed(x0, mean, std, abs_3d, obstacles, joints=(0,), valid=None) -> torch.Tensor:
    """dL_o/dx0 by autograd (the engine's cmdi_obstacle_seed with c_o = 1 and no other term)"""
    with torch.enable_grad():
        z = x0.detach().requires_grad_(True)
        return torch.autograd.grad(obstacle_loss(z, mean, std, abs_3d, obstacles, joints, valid), z)[0]


def joint_mask(joints: Sequence[int]) -> int:
    """the engine's bit mask of a joint set"""
    m = 0
    for j in joints:
        m |= 1 << int(j)
    return m


@dataclass
class ObstacleTerm:
    """y['obstacle_*'] and diffusion.joint_space, reduced to tensors; m is y['mask'] (Conditioning.y_mask)."""
    mean: torch.Tensor                   # (263,)
    std: torch.Tensor
    obstacles: torch.Tensor              # (B, K, 3)
    joints: Sequence[int] = (0,)
    abs_3d: bool = True
    weight: float = 1.0
    gradient_schedule: Optional[str] = None
    diffusion_steps: int = 1000
    stop_obstacleguidance_at: int = 0


def p_mean_variance(sd, tab: O.DiffusionTables, x: torch.Tensor, t: torch.Tensor, c: O.Conditioning, ob: ObstacleTerm,
                    fc: Optional[FC.FootContactTerm] = None, j: Optional[J.JointTerm] = None):
    """condmdi_oracle.p_mean_variance with the obstacle term and, when given, the foot-contact and joint terms (module
    docstring)."""
    need_ob = bool((t >= ob.stop_obstacleguidance_at).all())
    if not need_ob:
        if fc is not None:
            return FC.p_mean_variance(sd, tab, x, t, c, fc, j)
        return J.p_mean_variance(sd, tab, x, t, c, j) if j is not None else _P_MEAN_VARIANCE(sd, tab, x, t, c)
    dev = x.device
    t_model = torch.tensor(tab.timestep_map, dtype=t.dtype)[t]
    B, L = x.shape[0], x.shape[-1]
    y_mask = c.y_mask.to(dev) if c.y_mask is not None else torch.ones(B, 1, 1, L, dtype=torch.bool, device=dev)
    keyframes = c.reconstruction_guidance or (c.imputate and c.replacement_distribution == "conditional")
    M = (c.inpainting_mask.to(dev) & y_mask.bool()) if keyframes else torch.zeros_like(x, dtype=torch.bool)
    need_fc = fc is not None and bool((t >= fc.stop_footcontact_at).all())
    need_jg = j is not None and bool((t >= j.stop_jointguidance_at).all())
    need_rg = c.reconstruction_guidance and bool((t >= c.stop_recguidance_at).all())
    need_imp = keyframes and c.imputate and bool((t >= c.stop_imputation_at).all())
    with torch.enable_grad():
        z = x.detach().requires_grad_(True)
        hat_x = O._model(sd, z, t_model, c)
        grad = J._coef(ob.gradient_schedule, ob.diffusion_steps, ob.weight, tab, t, x.shape, dev) * torch.autograd.grad(
            obstacle_loss(hat_x, ob.mean, ob.std, ob.abs_3d, ob.obstacles, ob.joints, y_mask), z,
            retain_graph=need_fc or need_jg or need_rg)[0]
        if need_fc:
            g_c = torch.autograd.grad(FC.contact_loss(hat_x, fc.mean, fc.std, fc.abs_3d, y_mask), z,
                                      retain_graph=need_jg or need_rg)[0]
            grad = J._coef(fc.gradient_schedule, fc.diffusion_steps, fc.weight, tab, t, x.shape, dev) * g_c + grad
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
def obstacle_guided(ob: ObstacleTerm, fc: Optional[FC.FootContactTerm] = None, j: Optional[J.JointTerm] = None):
    """condmdi_oracle's samplers (sample_loop, p_sample, ddim_sample; so also repaint_oracle's walk) and
    dpm_solver_oracle's loop with the obstacle term (and the foot-contact / joint terms when given) in p_mean_variance"""
    from oracle import dpm_solver_oracle as S
    pmv = lambda sd, tab, x, t, c: p_mean_variance(sd, tab, x, t, c, ob, fc, j)  # noqa: E731
    O.p_mean_variance = S.p_mean_variance = pmv
    try:
        yield
    finally:
        O.p_mean_variance = S.p_mean_variance = _P_MEAN_VARIANCE


def obstacles_near(x0, mean, std, abs_3d, K: int, joints=(0,), g: Optional[torch.Generator] = None,
                   pad: int = 0) -> torch.Tensor:
    """(B, K + pad, 3) obstacles that the joints of x0 run into: obstacle k of sample b is centred near the XZ position of
    a random joint of `joints` at a random frame, with a radius between 0.5 and 1.5 times the median step of that joint,
    so that it covers a few frames; then `pad` padding rows (r = 0) at random centres."""
    g = g if g is not None else torch.Generator().manual_seed(0)
    P = J.joint_positions(x0.double(), mean.double(), std.double(), abs_3d)[..., [0, 2]]         # (B, L, 22, 2)
    B, L = P.shape[:2]
    out = torch.zeros(B, K + pad, 3, dtype=torch.float64)
    for b in range(B):
        for k in range(K):
            jt = joints[int(torch.randint(len(joints), (1,), generator=g))]
            f = int(torch.randint(L, (1,), generator=g))
            step = (P[b, 1:, jt] - P[b, :-1, jt]).norm(dim=-1).median().clamp_min(1e-3)
            out[b, k, :2] = P[b, f, jt] + 0.3 * step * torch.randn(2, generator=g, dtype=torch.float64)
            out[b, k, 2] = step * (0.5 + torch.rand(1, generator=g, dtype=torch.float64))
        out[b, K:, :2] = torch.randn(pad, 2, generator=g, dtype=torch.float64)
    return out.float()


def inputs(B: int, L: int = 196, seed: int = 0, K: int = 4, joints=(0,), abs_3d: bool = True, pad: int = 0):
    """Seeded obstacle inputs: joint_guidance_oracle.inputs' statistics, x0 (B, 263, 1, L) standard normal, and
    obstacles_near(x0) (B, K + pad, 3)."""
    mean, std, _, _, g = J.inputs(B, L, seed=seed)
    x0 = torch.randn(B, 263, 1, L, generator=g)
    return mean, std, x0, obstacles_near(x0, mean, std, abs_3d, K, joints, g, pad), g

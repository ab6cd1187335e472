"""Restatement of overlapping-window sampling (GaussianDiffusion.window, DESIGN.md "Overlapping windows").

A motion of N frames runs as K windows of F frames: window k starts at global frame f0(k) = min(k (F - O), N - F),
K = 1 + ceil((N - F) / (F - O)) (1 when N <= F).  Window b*K + k is row k of sample b in a batch of B*K sequences.  At
every step the x0 of each element (after CFG, guidance and imputation) of a frame g that several windows cover becomes
sum_k w_k(g) x0_k(g) / sum_k w_k(g) over them in ascending k, in fp32, with w_k(g) = 1 + min(g - f0(k), f0(k) + F - 1 - g);
a frame covered by one window keeps its x0.  Noise is drawn in the global layout and cropped.

`blended(f0, N)` wraps the restated p_mean_variance (condmdi_oracle's, and the name the PLMS, DPM-Solver++, UniPC and
SDE-DPM-Solver++ restatements import), as make_golden_unet_guidance.model_calls_under wraps its model call: the blend
replaces pred_xstart and the posterior mean is recomputed from it (q_posterior_mean_variance,
gaussian_diffusion.py:330-349).  oracle/make_golden_windowed.py anchors it to the reference's own steps.
"""
from __future__ import annotations

import contextlib
from typing import List, Optional

import torch

from oracle import condmdi_oracle as O


def placement(n: int, frames: int, overlap: int) -> List[int]:
    """First global frame of each window."""
    if n <= frames:
        return [0]
    step = frames - overlap
    k = 1 + (n - frames + step - 1) // step
    return [min(i * step, n - frames) for i in range(k)]


def weights(f0: List[int], frames: int) -> torch.Tensor:
    """(K, F) fp32 tent weights w_k of each window's frames: 1 at its ends, rising by 1 per frame inwards."""
    l = torch.arange(frames)
    w = 1 + torch.minimum(l, frames - 1 - l)
    return w.to(torch.float32).expand(len(f0), frames).clone()


def crop(x: torch.Tensor, f0: List[int], frames: int) -> torch.Tensor:
    """(B, ..., N) -> (B * K, ..., F)"""
    parts = [x[..., f:f + frames] for f in f0]
    return torch.stack(parts, 1).reshape(x.shape[0] * len(f0), *x.shape[1:-1], frames)


def gather(xw: torch.Tensor, f0: List[int], n: int) -> torch.Tensor:
    """(B * K, ..., F) -> (B, ..., N), each frame from the first window covering it"""
    K, F = len(f0), xw.shape[-1]
    xw = xw.reshape(xw.shape[0] // K, K, *xw.shape[1:])
    out = torch.empty(*xw.shape[:1], *xw.shape[2:-1], n, dtype=xw.dtype)
    for g in range(n):
        k = next(i for i in range(K) if f0[i] + F > g)
        out[..., g] = xw[:, k, ..., g - f0[k]]
    return out


def blend(x0w: torch.Tensor, f0: List[int], n: int) -> torch.Tensor:
    """The blended x0 of every window row: fp32, ascending k, products and sums rounded one at a time."""
    K, F = len(f0), x0w.shape[-1]
    w = weights(f0, F)
    xw = x0w.reshape(x0w.shape[0] // K, K, *x0w.shape[1:])
    out = xw.clone()
    for g in range(n):
        cover = [k for k in range(K) if f0[k] <= g < f0[k] + F]
        if len(cover) < 2:
            continue
        acc, wsum = None, torch.tensor(0.0)
        for k in cover:
            term = w[k, g - f0[k]] * xw[:, k, ..., g - f0[k]]
            acc = term if acc is None else acc + term
            wsum = wsum + w[k, g - f0[k]]
        v = acc / wsum
        for k in cover:
            out[:, k, ..., g - f0[k]] = v
    return out.reshape(x0w.shape)


# the sampler restatements that import p_mean_variance by name (they call it through their own module globals)
_PMV_USERS = ("oracle.plms_oracle", "oracle.dpm_solver_oracle", "oracle.unipc_oracle", "oracle.dpm_solver_sde_oracle")


@contextlib.contextmanager
def blended(f0: List[int], n: int):
    """Every p_mean_variance of condmdi_oracle and of the sampler restatements that import it (PLMS, DPM-Solver++,
    UniPC, SDE-DPM-Solver++) inside the block returns the window-blended pred_xstart and the posterior mean of it; one
    window: unchanged."""
    import importlib
    plain = O.p_mean_variance
    users = [importlib.import_module(m) for m in _PMV_USERS]
    if len(f0) > 1:
        def wrapped(sd, tab, x, t, c):
            out = dict(plain(sd, tab, x, t, c))
            pred = blend(out["pred_xstart"], f0, n)
            out["pred_xstart"] = pred
            out["mean"] = O.extract(tab.posterior_mean_coef1, t, x.shape) * pred + O.extract(tab.posterior_mean_coef2, t, x.shape) * x
            return out
        O.p_mean_variance = wrapped
        for u in users:
            u.p_mean_variance = wrapped
    try:
        yield
    finally:
        O.p_mean_variance = plain
        for u in users:
            u.p_mean_variance = plain


# ---------------------------------------------------------------------------------------------------
# the configurations of tests/golden/windowed.* (oracle/make_golden_windowed.py drives the reference on them)
# ---------------------------------------------------------------------------------------------------
B_FIX = 2
# name: (global frames N, window frames F, overlap O, sampler, respacing, skip_timesteps, guided, unet)
FIXTURES = {
    "text_k2": (300, 196, 48, "ddpm", "ddim50", 45, False, False),     # per-window prompts, CFG 2.5 + imputation, K = 2
    "guided_k3": (200, 120, 60, "ddim", "ddim50", 46, True, False),    # + reconstruction guidance w = 20, K = 3, 3-way frames
    "unet_k3": (200, 120, 60, "ddpm", "ddim50", 46, False, True),      # UNet xl, CFG 2.5 + keyframe input, K = 3
}


def fixture_inputs(name: str):
    """Seeded inputs of a fixture configuration, in the global layout: x_obs, keyframe mask, per-window text
    embeddings (B * K, 512), text_scale, and the tape (x_T, then one draw per step)."""
    N, F, O_, _, respacing, skip, _, _ = FIXTURES[name]
    K = len(placement(N, F, O_))
    g = torch.Generator().manual_seed(sorted(FIXTURES).index(name) + 500)
    x_obs = torch.randn(B_FIX, 263, 1, N, generator=g)
    kf = torch.rand(B_FIX, 263, 1, N, generator=g) < 0.2
    cond_w = torch.randn(B_FIX * K, 512, generator=g)
    scale = torch.tensor([2.5, 0.7])
    steps = O.make_tables(respacing).num_timesteps - skip
    tape = torch.randn(1 + steps, B_FIX, 263, 1, N, generator=g)
    return x_obs, kf, cond_w, scale, tape


def fixture_conditioning(name: str, x_obs, kf, scale) -> O.Conditioning:
    """The global conditioning of a fixture (cond_emb is passed per window)"""
    N, _, _, _, _, _, guided, unet = FIXTURES[name]
    kw = dict(cfg=True, text_scale=scale, y_mask=torch.ones(B_FIX, 1, 1, N, dtype=torch.bool))
    if unet:
        kw.update(obs_x0=x_obs, obs_mask=kf)
    else:
        kw.update(imputate=True, stop_imputation_at=1, inpainted_motion=x_obs, inpainting_mask=kf)
    if guided:
        kw.update(reconstruction_guidance=True, reconstruction_weight=20.0, stop_recguidance_at=2)
    return O.Conditioning(**kw)


def fixture_restatement(name: str, sd):
    """The restated windowed loop of a fixture configuration, global (B, 263, 1, N)"""
    N, F, O_, sampler, respacing, skip, _, _ = FIXTURES[name]
    x_obs, kf, cond_w, scale, tape = fixture_inputs(name)
    c = fixture_conditioning(name, x_obs, kf, scale)
    return sample_loop(sd, O.make_tables(respacing), (B_FIX, 263, 1, N), c, tape, placement(N, F, O_), F, sampler=sampler,
                       skip_timesteps=skip, init_image=x_obs, cond_emb=cond_w)


def window_conditioning(c: O.Conditioning, f0: List[int], frames: int, cond_emb: Optional[torch.Tensor] = None) -> O.Conditioning:
    """Conditioning in the global layout -> the windows': tensors over frames cropped, per-sample ones repeated per
    window; cond_emb (B * K, 512) replaces the repeated one (per-window prompts)."""
    K = len(f0)
    rep = lambda t: None if t is None else t.repeat_interleave(K, 0)  # noqa: E731
    cr = lambda t: None if t is None else crop(t, f0, frames)  # noqa: E731
    return O.Conditioning(cond_emb=cond_emb if cond_emb is not None else rep(c.cond_emb), cfg=c.cfg, text_scale=rep(c.text_scale),
                          y_mask=cr(c.y_mask), imputate=c.imputate, stop_imputation_at=c.stop_imputation_at,
                          replacement_distribution=c.replacement_distribution, inpainted_motion=cr(c.inpainted_motion),
                          inpainting_mask=cr(c.inpainting_mask), reconstruction_guidance=c.reconstruction_guidance,
                          reconstruction_weight=c.reconstruction_weight, gradient_schedule=c.gradient_schedule,
                          diffusion_steps=c.diffusion_steps, stop_recguidance_at=c.stop_recguidance_at, obs_x0=cr(c.obs_x0),
                          obs_mask=cr(c.obs_mask))


def sample_loop(sd, tab: O.DiffusionTables, shape, c: O.Conditioning, tape: torch.Tensor, f0: List[int], frames: int,
                sampler: str = "ddpm", skip_timesteps: int = 0, init_image: Optional[torch.Tensor] = None,
                cond_emb: Optional[torch.Tensor] = None, windows: bool = False, loop=None):
    """condmdi_oracle.sample_loop on overlapping windows: shape, c, tape and init_image in the global layout, the result
    gathered to (B, D, 1, N) (windows=True: the window rows (B * K, D, 1, F)).  loop: another restated loop with
    sample_loop's leading arguments (sd, tab, shape, c, tape, skip_timesteps=, init_image=), e.g.
    plms_oracle.plms_sample_loop with its order bound; `sampler` is then unused."""
    n = int(shape[-1])
    wshape = (shape[0] * len(f0),) + tuple(shape[1:-1]) + (frames,)
    wtape = torch.stack([crop(tape[i], f0, frames) for i in range(tape.shape[0])])
    wc = window_conditioning(c, f0, frames, cond_emb)
    init = None if init_image is None else crop(init_image, f0, frames)
    with blended(f0, n):
        if loop is None:
            xw = O.sample_loop(sd, tab, wshape, wc, wtape, sampler=sampler, skip_timesteps=skip_timesteps, init_image=init)
        else:
            xw = loop(sd, tab, wshape, wc, wtape, skip_timesteps=skip_timesteps, init_image=init)
    return xw if windows else gather(xw, f0, n)

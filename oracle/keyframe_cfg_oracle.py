"""Restatement of classifier-free guidance over keyframes (condmdi_b200.KeyframeClassifierFreeSampleModel).

Per sample b, with obs = (obs_x0, obs_mask) of a keyframe-conditioned MDM_UNET:

    c = m(x, text_b, obs)     u = m(x, no text, obs)     n = m(x, no text, obs_mask = 0)
    text model (Conditioning.cfg):  x0 = (n + w_k (u - n)) + w_t (c - u)      w_t = text_scale[b], w_k = keyframe_scale[b]
    no_cond model:                  x0 = n + w_k (c - n)

every operation an fp32 tensor op (round to nearest), in that order.  `keyframe_cfg(w_k)` wraps condmdi_oracle's model
call (its module-level `_model`), as windowed_oracle wraps p_mean_variance, so the restated p_mean_variance, p_sample,
ddim_sample and sample_loop (and the PLMS restatement, which calls p_mean_variance) apply imputation and reconstruction
guidance to this x0 exactly as they do to CFG's output.  oracle/make_golden_keyframe_cfg.py anchors it to the
reference's own MDM_UNET and loops.
"""
from __future__ import annotations

import contextlib

import torch

from oracle import condmdi_oracle as O


def combine(c: torch.Tensor, u: torch.Tensor, n: torch.Tensor, text_scale, keyframe_scale: torch.Tensor) -> torch.Tensor:
    """The guided output from the passes; u None: the two-pass form n + w_k (c - n)."""
    wk = keyframe_scale.view(-1, 1, 1, 1)
    if u is None:
        return n + wk * (c - n)
    a = n + wk * (u - n)
    return a + text_scale.view(-1, 1, 1, 1) * (c - u)


def passes(sd, x, t_model, c: O.Conditioning):
    """(c, u, n): the passes of the guided model; u is None without text CFG."""
    free_mask = torch.zeros_like(c.obs_mask)
    cc = O.unet_forward(sd, x, t_model, c.cond_emb, False, c.obs_x0, c.obs_mask)
    uu = O.unet_forward(sd, x, t_model, c.cond_emb, True, c.obs_x0, c.obs_mask) if c.cfg else None
    nn = O.unet_forward(sd, x, t_model, c.cond_emb, True, c.obs_x0, free_mask)
    return cc, uu, nn


def model(sd, x, t_model, c: O.Conditioning, keyframe_scale: torch.Tensor) -> torch.Tensor:
    assert O.is_unet(sd) and c.obs_x0 is not None, "keyframe CFG needs a keyframe-conditioned MDM_UNET and its keyframes"
    cc, uu, nn = passes(sd, x, t_model, c)
    return combine(cc, uu, nn, c.text_scale, keyframe_scale)


@contextlib.contextmanager
def keyframe_cfg(keyframe_scale: torch.Tensor):
    """Every model call of condmdi_oracle (its `_model`) becomes the keyframe-guided model with w_k = keyframe_scale."""
    plain = O._model
    O._model = lambda sd, x, t_model, c: model(sd, x, t_model, c, keyframe_scale)
    try:
        yield
    finally:
        O._model = plain

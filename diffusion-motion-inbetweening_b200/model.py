"""Drop-in mirror of the reference's denoiser interface, backed by the native H100 engine.

    MDM                          model/mdm.py:10-315   (arch='trans_enc', data_rep='hml_vec', cond_mode no_cond|text)
    ClassifierFreeSampleModel    model/cfg_sampler.py:5-35
    KeyframeClassifierFreeSampleModel   classifier-free guidance over the keyframes of a keyframe-conditioned MDM_UNET
                                        (y['keyframe_scale']), which the reference's scripts set and never read

`MDM` owns fp32 parameters under the reference's state-dict keys (so `load_state_dict` of a reference checkpoint
works, utils/model_util.py:19-23) and evaluates through `cmdi_model_forward`; there is no PyTorch math path.
`resolve_model` also accepts the REFERENCE's own `MDM` / `ClassifierFreeSampleModel` instances (duck-typed), which
is how the engine drops in under sample/synthesize.py etc. without touching them (see INTEGRATION.md).
"""
from __future__ import annotations

import math
import types
from copy import deepcopy
from typing import Dict, Optional, Tuple

import numpy as np
import torch
import torch.nn as nn

from . import capi
from .engine import Engine


def _positional_encoding(d_model: int, max_len: int = 5000) -> torch.Tensor:
    """PositionalEncoding buffer (mdm.py:322-330)."""
    pe = torch.zeros(max_len, d_model)
    position = torch.arange(0, max_len, dtype=torch.float).unsqueeze(1)
    div_term = torch.exp(torch.arange(0, d_model, 2).float() * (-np.log(10000.0) / d_model))
    pe[:, 0::2] = torch.sin(position * div_term)
    pe[:, 1::2] = torch.cos(position * div_term)
    return pe.unsqueeze(0).transpose(0, 1)


def _state_fingerprint(module: nn.Module) -> Tuple:
    return tuple((k, v.data_ptr(), v._version) for k, v in module.state_dict(keep_vars=True).items()
                 if not k.startswith("clip_model."))


def engine_for(self, device: torch.device, max_batch: int = 64, precision: int = capi.PRECISION_BF16X3,
               nframes: Optional[int] = None) -> Engine:
    """Engine holding this module's weights on `device` (created once, re-uploaded when parameters change)."""
    device = torch.device(device)
    cache: Dict = self.__dict__.setdefault("_condmdi_engines", {})
    nframes = int(nframes if nframes is not None else getattr(self, "max_frames", 196))
    key = (str(device), precision, nframes)
    eng = cache.get(key)
    sd = None
    if eng is None or eng.max_batch < max_batch:
        sd = {k: v for k, v in self.state_dict().items() if not k.startswith("clip_model.")}
        if eng is not None:
            eng.close()
        if "unet.time_mlp.0.weight" in sd:
            # MDM_UNET (model/mdm_unet.py): geometry read off the state dict
            levels = 1 + max(int(k.split(".")[2]) for k in sd if k.startswith("unet.downs."))
            d = sd["unet.time_mlp.0.weight"].shape[1]
            mults = [sd[f"unet.downs.{l}.0.blocks.0.block1.0.weight"].shape[0] // d for l in range(levels)]
            njoints = sd["unet.final_conv.1.weight"].shape[0]
            in_ch = sd["unet.downs.0.0.blocks.0.block1.0.weight"].shape[1]
            if in_ch not in (njoints, 2 * njoints) or "unet.downs.0.0.blocks.0.block.0.weight" in sd:
                raise NotImplementedError("the engine implements MDM_UNET with adagn=True and input_feats or 2 * input_feats channels")
            eng = Engine(device, njoints=njoints, nframes=nframes, latent_dim=d, max_batch=max_batch, has_text="embed_text.weight" in sd,
                         precision=precision, arch=capi.ARCH_UNET, unet_dim_mults=mults, keyframe_conditioned=in_ch == 2 * njoints)
        else:
            num_layers = 1 + max(int(k.split(".")[2]) for k in sd if k.startswith("seqTransEncoder.layers."))
            ff = sd["seqTransEncoder.layers.0.linear1.weight"].shape[0]
            d = sd["input_process.poseEmbedding.weight"].shape[0]
            njoints = sd["input_process.poseEmbedding.weight"].shape[1]
            eng = Engine(device, njoints=njoints, nframes=nframes, latent_dim=d, ff_size=ff, num_layers=num_layers,
                         num_heads=int(getattr(self, "num_heads", 4)), max_batch=max_batch,
                         has_text="embed_text.weight" in sd, precision=precision)
        eng._fingerprint = None
        cache[key] = eng
    fp = _state_fingerprint(self)
    if eng._fingerprint != fp:
        if sd is None:
            sd = {k: v for k, v in self.state_dict().items() if not k.startswith("clip_model.")}
        eng.load_state_dict(sd)
        eng._fingerprint = fp
    return eng


class MDM(nn.Module):
    """Motion diffusion transformer encoder (reference: model/mdm.py:10), inference only, engine-backed."""

    def __init__(self, modeltype="", njoints=263, nfeats=1, num_actions=1, translation=True, pose_rep="rot6d", glob=True,
                 glob_rot=True, latent_dim=512, ff_size=1024, num_layers=8, num_heads=4, dropout=0.1, ablation=None,
                 activation="gelu", legacy=False, data_rep="hml_vec", dataset="humanml", clip_dim=512, arch="trans_enc",
                 emb_trans_dec=False, clip_version=None, **kargs):
        super().__init__()
        if arch != "trans_enc" or activation != "gelu" or nfeats != 1:
            raise NotImplementedError("the engine implements arch='trans_enc', activation='gelu', nfeats=1")
        self.modeltype, self.njoints, self.nfeats, self.num_actions = modeltype, njoints, nfeats, num_actions
        self.data_rep, self.dataset, self.pose_rep, self.glob, self.glob_rot = data_rep, dataset, pose_rep, glob, glob_rot
        self.translation, self.latent_dim, self.ff_size, self.num_layers = translation, latent_dim, ff_size, num_layers
        self.num_heads, self.dropout, self.activation, self.clip_dim, self.arch = num_heads, dropout, activation, clip_dim, arch
        self.input_feats = njoints * nfeats
        self.cond_mode = kargs.get("cond_mode", "no_cond")
        self.cond_mask_prob = kargs.get("cond_mask_prob", 0.)
        self.keyframe_conditioned = kargs.get("keyframe_conditioned", False)
        self.max_frames = kargs.get("max_frames", 196)
        self.rot2xyz = None  # identity for hml_vec / 'xyz' (model/rotation2xyz.py:20-21); SMPL is out of scope
        d, ff = latent_dim, ff_size
        P = nn.Parameter

        def lin(prefix, out_f, in_f):
            bound = 1.0 / math.sqrt(in_f)
            self.register_parameter_path(prefix + ".weight", P((torch.rand(out_f, in_f) * 2 - 1) * bound))
            self.register_parameter_path(prefix + ".bias", P((torch.rand(out_f) * 2 - 1) * bound))

        lin("input_process.poseEmbedding", d, self.input_feats)
        self.register_buffer_path("sequence_pos_encoder.pe", _positional_encoding(d))
        lin("embed_timestep.time_embed.0", d, d)
        lin("embed_timestep.time_embed.2", d, d)
        # the reference's TimestepEmbedder holds the same PositionalEncoding module (mdm.py:147-148): same alias key
        self._modules["embed_timestep"].add_module("sequence_pos_encoder", self._modules["sequence_pos_encoder"])
        for i in range(num_layers):
            p = f"seqTransEncoder.layers.{i}."
            bound = math.sqrt(6.0 / (d + 3 * d))
            self.register_parameter_path(p + "self_attn.in_proj_weight", P((torch.rand(3 * d, d) * 2 - 1) * bound))
            self.register_parameter_path(p + "self_attn.in_proj_bias", P(torch.zeros(3 * d)))
            lin(p + "self_attn.out_proj", d, d)
            lin(p + "linear1", ff, d)
            lin(p + "linear2", d, ff)
            for n in ("norm1", "norm2"):
                self.register_parameter_path(p + n + ".weight", P(torch.ones(d)))
                self.register_parameter_path(p + n + ".bias", P(torch.zeros(d)))
        lin("output_process.poseFinal", self.input_feats, d)
        if "text" in self.cond_mode:
            lin("embed_text", d, clip_dim)
        for prm in self.parameters():
            prm.requires_grad_(False)

    # parameters are stored in nested containers so state_dict() yields exactly the reference's dotted keys
    def _container(self, path: str) -> Tuple[nn.Module, str]:
        mod = self
        parts = path.split(".")
        for part in parts[:-1]:
            if part not in mod._modules:
                mod.add_module(part, nn.Module())
            mod = mod._modules[part]
        return mod, parts[-1]

    def register_parameter_path(self, path: str, p: nn.Parameter) -> None:
        mod, leaf = self._container(path)
        mod.register_parameter(leaf, p)

    def register_buffer_path(self, path: str, t: torch.Tensor) -> None:
        mod, leaf = self._container(path)
        mod.register_buffer(leaf, t)

    engine_for = engine_for

    def encode_text(self, raw_text):
        """mdm.py:211-237 runs CLIP; CLIP is not part of this repo. Attach a callable returning (B, 512) fp32."""
        raise NotImplementedError("attach a text encoder: model.encode_text = lambda texts: <(B,512) float tensor>")

    def mask_cond(self, cond, force_mask=False):
        """mdm.py:188-198, eval mode."""
        return torch.zeros_like(cond) if force_mask else cond

    def parameters_wo_clip(self):
        return [p for name, p in self.named_parameters() if not name.startswith("clip_model.")]

    def forward(self, x, timesteps, y=None, cond_val=None, cond_mask=None):
        """mdm.py:239-306. `cond_val`/`cond_mask` (obs_x0/obs_mask under the CFG wrapper) are accepted and ignored,
        exactly like the reference's trans_enc path without 'better_cond' (SURVEY.md 8(b) note 2)."""
        return _forward_any(self, x, timesteps, y, cfg=False)


class MDM_UNET(nn.Module):
    """The UNet denoiser of the published CondMDI checkpoints (reference: model/mdm_unet.py:561-849; arch='unet',
    adagn, no attention), inference only, engine-backed.  Parameters live under the reference's state-dict keys."""

    def __init__(self, modeltype="", njoints=263, nfeats=1, num_actions=1, translation=True, pose_rep="rot6d", glob=True,
                 glob_rot=True, latent_dim=512, dim_mults=(2, 2, 2, 2), attention=False, ablation=None, legacy=False,
                 data_rep="hml_vec", dataset="humanml", clip_dim=512, emb_trans_dec=False, clip_version=None, adagn=True,
                 zero=True, arch="unet", unet_out_mult=8, xz_only=False, train_keypoint_mask="none", keyframe_conditioned=False,
                 keyframe_selection_scheme="in-between", zero_keyframe_loss=False, **kwargs):
        super().__init__()
        if arch != "unet" or attention or not adagn or xz_only or train_keypoint_mask != "none" or nfeats != 1:
            raise NotImplementedError("the engine implements MDM_UNET arch='unet', adagn=True, attention=False")
        if len(set(dim_mults)) != 1 or not 2 <= len(dim_mults) <= 4:
            raise NotImplementedError("dim_mults must be 2..4 equal multipliers (every published configuration)")
        self.njoints, self.nfeats, self.latent_dim, self.dim_mults = njoints, nfeats, latent_dim, tuple(dim_mults)
        self.data_rep, self.dataset, self.arch, self.translation = data_rep, dataset, arch, translation
        self.keyframe_conditioned = keyframe_conditioned
        self.cond_mode = kwargs.get("cond_mode", "no_cond")
        self.cond_mask_prob = kwargs.get("cond_mask_prob", 0.)
        self.input_feats = njoints * nfeats
        self.max_frames = kwargs.get("max_frames", 196)
        self.rot2xyz = None
        P, d = nn.Parameter, latent_dim
        g = torch.Generator().manual_seed(0)

        def uni(shape, bound):
            return (torch.rand(*shape, generator=g) * 2 - 1) * bound

        def put(key, t):
            mod, leaf = self._container(key)
            mod.register_parameter(leaf, P(t))

        def conv(key, co, ci, k, transposed=False, zero_=False):
            bound = 1.0 / math.sqrt(ci * k)
            w = uni((ci, co, k) if transposed else (co, ci, k), bound)
            put(key + ".weight", torch.zeros_like(w) if zero_ else w)
            put(key + ".bias", torch.zeros(co) if zero_ else uni((co,), bound))

        def lin(key, co, ci, zero_=False):
            bound = 1.0 / math.sqrt(ci)
            put(key + ".weight", torch.zeros(co, ci) if zero_ else uni((co, ci), bound))
            put(key + ".bias", torch.zeros(co) if zero_ else uni((co,), bound))

        def rtb(pre, ci, co):
            conv(pre + "blocks.0.block1.0", co, ci, 5)
            put(pre + "blocks.0.block1.2.weight", torch.ones(co)); put(pre + "blocks.0.block1.2.bias", torch.zeros(co))
            conv(pre + "blocks.1.block.0", co, co, 5, zero_=zero)      # mdm_unet.py:53-56
            put(pre + "blocks.1.block.2.weight", torch.ones(co)); put(pre + "blocks.1.block.2.bias", torch.zeros(co))
            lin(pre + "time_mlp.1", 2 * co, d, zero_=True)             # :190-193
            if ci != co:
                conv(pre + "residual_conv", co, ci, 1)

        lin("unet.time_mlp.0", 4 * d, d)
        lin("unet.time_mlp.2", d, 4 * d)
        dims = [self.input_feats] + [int(d * m) for m in dim_mults]
        added = self.input_feats if keyframe_conditioned else 0
        n = len(dim_mults)
        for l in range(n):
            rtb(f"unet.downs.{l}.0.", dims[l] + (added if l == 0 else 0), dims[l + 1])
            rtb(f"unet.downs.{l}.1.", dims[l + 1], dims[l + 1])
            if l + 1 < n:
                conv(f"unet.downs.{l}.3.conv", dims[l + 1], dims[l + 1], 3)
        rtb("unet.mid_block1.", dims[-1], dims[-1])
        rtb("unet.mid_block2.", dims[-1], dims[-1])
        for i, l in enumerate(range(n - 1, 0, -1)):
            rtb(f"unet.ups.{i}.0.", dims[l + 1] * 2, dims[l])
            rtb(f"unet.ups.{i}.1.", dims[l], dims[l])
            conv(f"unet.ups.{i}.3.conv", dims[l], dims[l], 4, transposed=True)
        conv("unet.final_conv.0.block.0", dims[1], dims[1], 5)
        put("unet.final_conv.0.block.2.weight", torch.ones(dims[1])); put("unet.final_conv.0.block.2.bias", torch.zeros(dims[1]))
        conv("unet.final_conv.1", self.input_feats, dims[1], 1, zero_=zero)
        mod, leaf = self._container("sequence_pos_encoder.pe")
        mod.register_buffer(leaf, _positional_encoding(d))
        lin("embed_timestep.time_embed.0", d, d)
        lin("embed_timestep.time_embed.2", d, d)
        self._modules["embed_timestep"].add_module("sequence_pos_encoder", self._modules["sequence_pos_encoder"])
        if "text" in self.cond_mode:
            lin("embed_text", d, clip_dim)
        for prm in self.parameters():
            prm.requires_grad_(False)

    def _container(self, path: str):
        mod = self
        parts = path.split(".")
        for part in parts[:-1]:
            if part not in mod._modules:
                mod.add_module(part, nn.Module())
            mod = mod._modules[part]
        return mod, parts[-1]

    engine_for = engine_for

    def encode_text(self, raw_text):
        raise NotImplementedError("attach a text encoder: model.encode_text = lambda texts: <(B,512) float tensor>")

    def mask_cond(self, cond, force_mask=False):
        return torch.zeros_like(cond) if force_mask else cond

    def parameters_wo_clip(self):
        return [p for name, p in self.named_parameters() if not name.startswith("clip_model.")]

    def forward(self, x, timesteps, y=None, obs_x0=None, obs_mask=None):
        """mdm_unet.py:765-783."""
        assert (obs_x0 is None) == (obs_mask is None), 'with spatial-conditioning, both obs_x0 and obs_mask must be provided'
        return _forward_any(self, x, timesteps, y, cfg=False, obs_x0=obs_x0, obs_mask=obs_mask)


def _forward_any(inner, x, timesteps, y, cfg: bool, text_scale=None, obs_x0=None, obs_mask=None, keyframe_scale=None):
    y = {} if y is None else y
    if not x.is_cuda:
        raise RuntimeError("condmdi_b200 runs on CUDA tensors only (no CPU fallback)")
    ts = timesteps.reshape(-1)
    t0 = int(ts[0].item())
    if not bool((ts == t0).all()):
        # per-sample timesteps (not produced by the sampling loops): evaluate per distinct value
        out = torch.empty_like(x, dtype=torch.float32)
        for tv in ts.unique().tolist():
            idx = (ts == tv).nonzero().reshape(-1)
            ysub = dict(y)
            if "text" in ysub:
                ysub["text"] = [ysub["text"][i] for i in idx.tolist()]
            if text_scale is not None:
                ysub["text_scale"] = y["text_scale"][idx]
            out[idx] = _forward_any(inner, x[idx], ts[idx], ysub, cfg, None if text_scale is None else text_scale[idx],
                                    None if obs_x0 is None else obs_x0[idx], None if obs_mask is None else obs_mask[idx],
                                    None if keyframe_scale is None else keyframe_scale[idx])
        return out
    B = x.shape[0]
    eng = inner.engine_for(x.device, max_batch=B if keyframe_scale is None else keyframe_cfg_max_batch(B, cfg), nframes=x.shape[-1])
    cond_emb = None
    if "text" in getattr(inner, "cond_mode", "no_cond"):
        cond_emb = inner.encode_text(y["text"]).to(device=x.device, dtype=torch.float32)
    if eng.arch != capi.ARCH_UNET:
        obs_x0 = obs_mask = None  # the transformer accepts and ignores them (SURVEY 8b note 2)
    return eng.forward(x, t0, cond_emb=cond_emb, uncond=bool(y.get("uncond", False)), cfg=cfg, text_scale=text_scale,
                       obs_x0=obs_x0, obs_mask=obs_mask, keyframe_scale=keyframe_scale)


class ClassifierFreeSampleModel(nn.Module):
    """model/cfg_sampler.py:5-35; the cond and uncond passes run as one batch-doubled native pass."""

    def __init__(self, model):
        super().__init__()
        self.model = model
        assert self.model.cond_mask_prob > 0, \
            'Cannot run a guided diffusion on a model that has not been trained with no conditions'
        self.rot2xyz = self.model.rot2xyz
        self.translation = self.model.translation
        self.njoints = self.model.njoints
        self.nfeats = self.model.nfeats
        self.data_rep = self.model.data_rep
        self.cond_mode = self.model.cond_mode
        self.keyframe_conditioned = self.model.keyframe_conditioned
        self.mask_value = -2.0

    def forward(self, x, timesteps, y=None, obs_x0=None, obs_mask=None, **kwargs):
        cond_mode = self.model.cond_mode
        assert cond_mode in ['text', 'action']
        # the caller's y is never mutated (the reference deep-copies it, cfg_sampler.py:28)
        return _forward_any(self.model, x, timesteps, y, cfg=True, text_scale=y['text_scale'].reshape(-1), obs_x0=obs_x0,
                            obs_mask=obs_mask)


def keyframe_cfg_max_batch(batch: int, text_cfg: bool) -> int:
    """The engine max_batch keyframe CFG needs for `batch` sequences: its passes (3 with text CFG, else 2) must fit the
    2 * max_batch sequences the engine's buffers hold."""
    return ((3 if text_cfg else 2) * batch + 1) // 2


def _is_keyframe_unet(model) -> bool:
    """A keyframe-conditioned MDM_UNET (this package's or the reference's), recognised by its state dict as engine_for
    reads it: the first convolution takes 2 * input_feats channels."""
    if not isinstance(model, nn.Module):
        return False
    sd = model.state_dict()
    if "unet.time_mlp.0.weight" not in sd:
        return False
    return sd["unet.downs.0.0.blocks.0.block1.0.weight"].shape[1] == 2 * sd["unet.final_conv.1.weight"].shape[0]


def check_keyframe_cfg_scales(y, text: bool) -> None:
    """Keyframe CFG reads y['keyframe_scale'], and for a text model y['text_scale'] too (w_t = 1: text conditioning
    without text guidance)."""
    for key in ("keyframe_scale",) + (("text_scale",) if text else ()):
        if y is None or key not in y:
            raise ValueError(f"KeyframeClassifierFreeSampleModel needs y[{key!r}]"
                             + (" (a text model's w_t; 1 for no text guidance)" if key == "text_scale" else ""))


class KeyframeClassifierFreeSampleModel(nn.Module):
    """Classifier-free guidance over the keyframes of a keyframe-conditioned MDM_UNET, nested inside text CFG (the
    two-condition guidance of InstructPix2Pix, Brooks et al. 2023, eq. 3, keyframes the inner condition).  Per sample b:

        c = m(x, text_b, obs)    u = m(x, no text, obs)    n = m(x, no text, obs_mask = 0)
        text model:     x0 = n + w_k (u - n) + w_t (c - u)    w_t = y['text_scale'][b], w_k = y['keyframe_scale'][b]
        no_cond model:  x0 = n + w_k (c - n)

    n is the keyframe-dropped input the published checkpoints were trained on (keyframe_mask_prob).  In fp32 each
    operation rounds to nearest in the order a = n + w_k (u - n), x0 = a + w_t (c - u); at w_k = 1 it is
    ClassifierFreeSampleModel up to that rounding.  The passes run as one batch-stacked native pass; y['uncond'] makes
    the text passes unconditional as it does for CFG.  A text model needs y['text_scale'] as ClassifierFreeSampleModel
    does (1 for keyframe guidance alone).  Every sampler of the package accepts it in place of the model."""

    def __init__(self, model):
        super().__init__()
        if not _is_keyframe_unet(model):
            raise ValueError("KeyframeClassifierFreeSampleModel needs a keyframe-conditioned MDM_UNET "
                             f"(got {type(model).__name__} without keyframe input)")
        self.model = model
        self.rot2xyz = getattr(model, "rot2xyz", None)
        self.translation = model.translation
        self.njoints = model.njoints
        self.nfeats = model.nfeats
        self.data_rep = model.data_rep
        self.cond_mode = model.cond_mode
        self.keyframe_conditioned = model.keyframe_conditioned
        self.mask_value = -2.0

    def forward(self, x, timesteps, y=None, obs_x0=None, obs_mask=None, **kwargs):
        text = "text" in self.model.cond_mode
        check_keyframe_cfg_scales(y, text)
        inner, _ = resolve_model(self.model)
        return _forward_any(inner, x, timesteps, y, cfg=text, text_scale=y["text_scale"].reshape(-1) if text else None,
                            obs_x0=obs_x0, obs_mask=obs_mask, keyframe_scale=y["keyframe_scale"].reshape(-1))


def is_keyframe_cfg(model) -> bool:
    """Whether `model` (or the model a _WrappedModel holds) is a KeyframeClassifierFreeSampleModel."""
    while type(model).__name__ == "_WrappedModel" and isinstance(getattr(model, "model", None), nn.Module):
        model = model.model
    return isinstance(model, KeyframeClassifierFreeSampleModel)


def resolve_model(model) -> Tuple[nn.Module, bool]:
    """(inner MDM-like module, is_cfg).  Accepts this package's classes and the reference's (duck-typed).  For a
    KeyframeClassifierFreeSampleModel is_cfg says whether text CFG runs with keyframe CFG (a text model)."""
    if isinstance(model, KeyframeClassifierFreeSampleModel):
        inner, _ = resolve_model(model.model)
        return inner, "text" in getattr(inner, "cond_mode", "no_cond")
    is_cfg = False
    inner = model
    if hasattr(inner, "model") and isinstance(getattr(inner, "model"), nn.Module) and \
            type(inner).__name__ in ("ClassifierFreeSampleModel", "_WrappedModel"):
        if type(inner).__name__ == "_WrappedModel":
            return resolve_model(inner.model)
        is_cfg = True
        inner = inner.model
    arch = getattr(inner, "arch", "trans_enc")
    if arch not in ("trans_enc", "unet"):
        raise NotImplementedError(f"the engine implements MDM arch='trans_enc' and MDM_UNET arch='unet' (got {arch!r})")
    if not hasattr(inner, "engine_for"):
        keys = inner.state_dict().keys()
        if "seqTransEncoder.layers.0.self_attn.in_proj_weight" not in keys and "unet.time_mlp.0.weight" not in keys:
            raise NotImplementedError(f"{type(inner).__name__} is neither an MDM transformer encoder nor an MDM_UNET")
        inner.engine_for = types.MethodType(engine_for, inner)  # reference model: attach the engine accessor
    return inner, is_cfg

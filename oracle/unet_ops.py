"""MDM_UNET op by op: the fp64 module each op of the engine's UNet op lists implements, looked up by the op's name (the
state-dict prefix of the module, "^T" for its input-VJP), and the model's forward order of those names.

unet_forward_by_ops composes these per-op references in that order and must be unet_forward itself; the GPU tests hold
every engine op to the reference of its name, so the names are what ties each op to the model.
"""
from __future__ import annotations

from typing import Dict, List, Optional

import torch
import torch.nn.functional as F

from .condmdi_oracle import unet_levels_of

FRAMES = 224  # the reference right-pads every input to 224 frames (mdm_unet.py:817)


def block_prefixes(levels: int) -> List[str]:
    """ResidualTemporalBlocks in forward order (the order of the engine's time_mlp.1 concatenation)."""
    out = []
    for l in range(levels):
        out += [f"unet.downs.{l}.0.", f"unet.downs.{l}.1."]
    out += ["unet.mid_block1.", "unet.mid_block2."]
    for i in range(levels - 1):
        out += [f"unet.ups.{i}.0.", f"unet.ups.{i}.1."]
    return out


def ada_columns(sd) -> Dict[str, int]:
    """the first column of each block's [scale | shift] in the concatenated time_mlp.1 output"""
    col, out = 0, {}
    for pre in block_prefixes(unet_levels_of(sd)):
        out[pre] = col
        col += sd[pre + "time_mlp.1.weight"].shape[0]
    return out


def weight_bias(sd, name: str):
    """(weight, bias) of the linear / convolution `name`; "*.time_mlp.1" is every block's time_mlp.1 stacked"""
    name = name.removesuffix("^T")
    if name == "*.time_mlp.1":
        pres = block_prefixes(unet_levels_of(sd))
        return (torch.cat([sd[p + "time_mlp.1.weight"] for p in pres]), torch.cat([sd[p + "time_mlp.1.bias"] for p in pres]))
    return sd[name + ".weight"], sd[name + ".bias"]


def is_gn(name: str) -> bool:
    n = name.removesuffix("^T")
    return n.endswith(".block1.2") or n.endswith(".block.2")


def gemm_forward(name: str, x: torch.Tensor, w: torch.Tensor, b: Optional[torch.Tensor]) -> torch.Tensor:
    """the convolution / linear layer `name` without its activation: x (nseq, C_in, P) or (nseq, K) for the time MLP"""
    if ".time_mlp." in name:
        return F.linear(x, w, b)
    if name.startswith("unet.downs.") and name.endswith(".3.conv"):
        return F.conv1d(x, w, b, stride=2, padding=1)                       # Downsample1d (mdm_unet.py:15-21)
    if name.startswith("unet.ups.") and name.endswith(".3.conv"):
        return F.conv_transpose1d(x, w, b, stride=2, padding=1)             # Upsample1d (:24-30)
    return F.conv1d(x, w, b, padding=w.shape[-1] // 2)


def is_upsample(name: str) -> bool:
    name = name.removesuffix("^T")
    return name.startswith("unet.ups.") and name.endswith(".3.conv")


def gemm_act(name: str) -> bool:
    """time_mlp.0's output goes through Mish, and so does time_mlp.2's (every block's time_mlp starts with Mish)"""
    return name in ("unet.time_mlp.0", "unet.time_mlp.2")


def gemm_vjp(name: str, dout: torch.Tensor, w: torch.Tensor, in_len: int) -> torch.Tensor:
    """d/dx of <gemm_forward(name, x), dout> for x of `in_len` positions (autograd of the forward module)"""
    cin = w.shape[0] if is_upsample(name) else w.shape[1]
    x = torch.zeros(dout.shape[0], cin, in_len, dtype=dout.dtype, device=dout.device, requires_grad=True)
    with torch.enable_grad():
        y = gemm_forward(name.removesuffix("^T"), x, w, None)
        return torch.autograd.grad(y, x, dout)[0]


def gn_mish(y: torch.Tensor, gamma, beta, scale=None, shift=None, res=None, one_plus_scale=None) -> torch.Tensor:
    """GroupNorm(8) -> [* (1 + scale) + shift] -> Mish -> [+ res] (Conv1dAdaGNBlock / ResidualTemporalBlock, mdm_unet.py:
    33-100, :163-218); one_plus_scale: a rounding of 1 + scale (autocast computes it in fp16)"""
    h = F.group_norm(y, 8, gamma, beta, 1e-5)
    if scale is not None:
        ops = 1 + scale
        if one_plus_scale is not None:
            ops = one_plus_scale(ops)
        h = h * ops[..., None] + shift[..., None]
    h = F.mish(h)
    return h if res is None else h + res


def gn_mish_vjp(y, dout, gamma, beta, scale=None, shift=None, one_plus_scale=None) -> torch.Tensor:
    y = y.detach().requires_grad_(True)
    with torch.enable_grad():
        return torch.autograd.grad(gn_mish(y, gamma, beta, scale, shift, one_plus_scale=one_plus_scale), y, dout)[0]


def forward_names(sd) -> List[str]:
    """the names of the ops of one engine pass, in the model's forward order"""
    levels = unet_levels_of(sd)
    out = ["input", "emb", "unet.time_mlp.0", "unet.time_mlp.2", "*.time_mlp.1"]

    def rtb(pre):
        out.extend([pre + "blocks.0.block1.0", pre + "blocks.0.block1.2", pre + "blocks.1.block.0"]
                   + ([pre + "residual_conv"] if pre + "residual_conv.weight" in sd else []) + [pre + "blocks.1.block.2"])

    for l in range(levels):
        rtb(f"unet.downs.{l}.0.")
        rtb(f"unet.downs.{l}.1.")
        if l + 1 < levels:
            out.append(f"unet.downs.{l}.3.conv")
    rtb("unet.mid_block1.")
    rtb("unet.mid_block2.")
    for i in range(levels - 1):
        rtb(f"unet.ups.{i}.0.")
        rtb(f"unet.ups.{i}.1.")
        out.append(f"unet.ups.{i}.3.conv")
    out += ["unet.final_conv.0.block.0", "unet.final_conv.0.block.2", "unet.final_conv.1"]
    return out


def unet_forward_by_ops(sd: Dict[str, torch.Tensor], x: torch.Tensor, timesteps: torch.Tensor, cond_emb=None, uncond=False,
                        obs_x0=None, obs_mask=None) -> torch.Tensor:
    """condmdi_oracle.unet_forward, as the per-op references of forward_names composed in that order: each op reads the
    tensors the ops before it produced, the way the engine's buffers pass them on"""
    levels = unet_levels_of(sd)
    skip_blocks = {f"unet.downs.{l}.1." for l in range(levels)}
    if obs_x0 is not None:
        x = torch.cat([obs_x0 * obs_mask + x * (~obs_mask), obs_mask.to(x.dtype)], dim=1)
    bs, nj, nf, L = x.shape
    pe = sd["sequence_pos_encoder.pe"] if "sequence_pos_encoder.pe" in sd else sd["embed_timestep.sequence_pos_encoder.pe"]
    state: Dict[str, torch.Tensor] = {}
    ada = ada_columns(sd)
    skips: List[torch.Tensor] = []
    block_in: Optional[torch.Tensor] = None
    for name in forward_names(sd):
        if name == "input":
            h = F.pad(x.reshape(bs, nj * nf, L), (0, FRAMES - L))
        elif name == "emb":
            emb = F.linear(F.silu(F.linear(pe[timesteps].reshape(bs, -1), sd["embed_timestep.time_embed.0.weight"], sd["embed_timestep.time_embed.0.bias"])),
                           sd["embed_timestep.time_embed.2.weight"], sd["embed_timestep.time_embed.2.bias"])
            if cond_emb is not None:
                emb = emb + F.linear(torch.zeros_like(cond_emb) if uncond else cond_emb, sd["embed_text.weight"], sd["embed_text.bias"])
            state["t"] = emb
        elif ".time_mlp." in name:
            w, b = weight_bias(sd, name)
            v = gemm_forward(name, state["t"], w, b)
            state["t"] = F.mish(v) if gemm_act(name) else v
            if name == "*.time_mlp.1":
                state["ada"] = state.pop("t")
        elif name.endswith("blocks.0.block1.0"):
            pre = name[: -len("blocks.0.block1.0")]
            if pre.startswith("unet.ups.") and pre.endswith(".0."):
                h = torch.cat((h, skips.pop()), dim=1)
            block_in = h
            w, b = weight_bias(sd, name)
            state["y"] = gemm_forward(name, h, w, b)
        elif name.endswith("blocks.1.block.0") or name == "unet.final_conv.0.block.0":
            w, b = weight_bias(sd, name)
            state["y"] = gemm_forward(name, h if name.startswith("unet.final") else state["t1"], w, b)
        elif name.endswith("residual_conv"):
            w, b = weight_bias(sd, name)
            state["r"] = gemm_forward(name, block_in, w, b)
        elif is_gn(name):
            g, bt = sd[name + ".weight"], sd[name + ".bias"]
            if name.endswith("blocks.0.block1.2"):
                pre = name[: -len("blocks.0.block1.2")]
                co = g.shape[0]
                a = state["ada"][:, ada[pre]: ada[pre] + 2 * co]
                state["t1"] = gn_mish(state["y"], g, bt, a[:, :co], a[:, co:])
            elif name.startswith("unet.final"):
                h = gn_mish(state["y"], g, bt)
            else:
                h = gn_mish(state["y"], g, bt, res=state.pop("r") if "r" in state else block_in)
                if name[: -len("blocks.1.block.2")] in skip_blocks:
                    skips.append(h)
        else:  # Downsample / Upsample / final_conv.1
            w, b = weight_bias(sd, name)
            h = gemm_forward(name, h, w, b)
    out = h[..., :L]
    return out.reshape(bs, out.shape[1], 1, L)

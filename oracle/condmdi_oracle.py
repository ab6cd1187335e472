"""TEST INFRASTRUCTURE -- CPU restatement of the reference's sampling hot path (the parity oracle).

Only `tests/`, `__graft_entry__.smoke()` and `bench.py`'s cpu-baseline legs may import this module; the
product path (condmdi_b200.*) never does and has no CPU fallback.

Every function restates one piece of setarehc/diffusion-motion-inbetweening (paths below are relative to
that repository) in plain torch-CPU / numpy, in the reference's operation order and dtypes:

    cosine_betas, DiffusionTables   diffusion/gaussian_diffusion.py:24-71, :183-217
    space_timesteps, respace        diffusion/respace.py:9-62, :74-91
    mdm_forward                     model/mdm.py:239-306 (+ :317-353 PE / timestep MLP, :356-372, :397-423) and
                                    torch.nn.TransformerEncoderLayer post-norm semantics (norm_first=False)
    cfg_forward                     model/cfg_sampler.py:25-35
    p_mean_variance                 diffusion/gaussian_diffusion.py:352-534 (START_X, FIXED_SMALL)
    p_sample / ddim_sample          :656-713 / :1358-1416
    p_sample_loop / ddim_sample_loop :1149-1297 / :1454-1587 (noise tape instead of the global generator)
    get_keyframes_mask              utils/editing_util.py:30-44, :56-100 + data_loaders/humanml_utils.py:68-91
    get_gradient_schedule           utils/editing_util.py:299-322

PINNING: the reference has no tests or golden vectors of its own (SURVEY.md section 4).  This restatement is
pinned against the reference ITSELF, imported on CPU in the build container (oracle/reference_harness.py):
`oracle/make_golden.py` checks every function here against the reference on seeded inputs and writes the
fixtures under tests/golden/ that `tests/test_oracle_golden.py` re-checks wherever the suite runs.
"""
from __future__ import annotations

import math
from dataclasses import dataclass
from typing import Dict, List, Optional, Sequence

import numpy as np
import torch
import torch.nn.functional as F

# ------------------------------------------------------------------------------------------------
# schedules
# ------------------------------------------------------------------------------------------------


def cosine_betas(num_steps: int, max_beta: float = 0.999) -> np.ndarray:
    """get_named_beta_schedule('cosine') -> betas_for_alpha_bar (gaussian_diffusion.py:44-71)."""
    def alpha_bar(t):
        return math.cos((t + 0.008) / 1.008 * math.pi / 2) ** 2

    betas = []
    for i in range(num_steps):
        t1 = i / num_steps
        t2 = (i + 1) / num_steps
        betas.append(min(1 - alpha_bar(t2) / alpha_bar(t1), max_beta))
    return np.array(betas)


def space_timesteps(num_timesteps: int, section_counts) -> set:
    """respace.py:9-62."""
    if isinstance(section_counts, str):
        if section_counts.startswith("ddim"):
            desired = int(section_counts[len("ddim"):])
            for i in range(1, num_timesteps):
                if len(range(0, num_timesteps, i)) == desired:
                    return set(range(0, num_timesteps, i))
            raise ValueError(f"cannot create exactly {num_timesteps} steps with an integer stride")
        section_counts = [int(x) for x in section_counts.split(",")]
    size_per = num_timesteps // len(section_counts)
    extra = num_timesteps % len(section_counts)
    start_idx = 0
    all_steps = []
    for i, section_count in enumerate(section_counts):
        size = size_per + (1 if i < extra else 0)
        if size < section_count:
            raise ValueError(f"cannot divide section of {size} steps into {section_count}")
        frac_stride = 1 if section_count <= 1 else (size - 1) / (section_count - 1)
        cur_idx = 0.0
        taken = []
        for _ in range(section_count):
            taken.append(start_idx + round(cur_idx))
            cur_idx += frac_stride
        all_steps += taken
        start_idx += size
    return set(all_steps)


@dataclass
class DiffusionTables:
    """float64 tables of GaussianDiffusion.__init__ (gaussian_diffusion.py:183-217)."""
    betas: np.ndarray
    timestep_map: List[int]

    def __post_init__(self):
        betas = np.array(self.betas, dtype=np.float64)
        self.betas = betas
        self.num_timesteps = int(betas.shape[0])
        alphas = 1.0 - betas
        self.alphas_cumprod = np.cumprod(alphas, axis=0)
        self.alphas_cumprod_prev = np.append(1.0, self.alphas_cumprod[:-1])
        self.sqrt_alphas_cumprod = np.sqrt(self.alphas_cumprod)
        self.sqrt_one_minus_alphas_cumprod = np.sqrt(1.0 - self.alphas_cumprod)
        self.sqrt_recip_alphas_cumprod = np.sqrt(1.0 / self.alphas_cumprod)
        self.sqrt_recipm1_alphas_cumprod = np.sqrt(1.0 / self.alphas_cumprod - 1)
        self.posterior_variance = betas * (1.0 - self.alphas_cumprod_prev) / (1.0 - self.alphas_cumprod)
        self.posterior_log_variance_clipped = np.log(np.append(self.posterior_variance[1], self.posterior_variance[1:]))
        self.posterior_mean_coef1 = betas * np.sqrt(self.alphas_cumprod_prev) / (1.0 - self.alphas_cumprod)
        self.posterior_mean_coef2 = (1.0 - self.alphas_cumprod_prev) * np.sqrt(alphas) / (1.0 - self.alphas_cumprod)


def make_tables(respacing="", steps: int = 1000) -> DiffusionTables:
    """create_gaussian_diffusion (utils/model_util.py:122-165) -> SpacedDiffusion.__init__ (respace.py:74-91)."""
    base = DiffusionTables(cosine_betas(steps), list(range(steps)))
    use = space_timesteps(steps, respacing if respacing else [steps])
    last = 1.0
    new_betas, tmap = [], []
    for i, acp in enumerate(base.alphas_cumprod):
        if i in use:
            new_betas.append(1 - acp / last)
            last = acp
            tmap.append(i)
    return DiffusionTables(np.array(new_betas), tmap)


def extract(arr: np.ndarray, t: torch.Tensor, shape) -> torch.Tensor:
    """_extract_into_tensor (gaussian_diffusion.py:2215-2228): f64 table -> gather -> .float() -> broadcast."""
    res = torch.from_numpy(arr)[t].float()
    while len(res.shape) < len(shape):
        res = res[..., None]
    return res.expand(shape)


# ------------------------------------------------------------------------------------------------
# denoiser
# ------------------------------------------------------------------------------------------------


def positional_encoding(d_model: int, max_len: int = 5000) -> torch.Tensor:
    """PositionalEncoding.__init__ (mdm.py:322-330) -> (max_len, 1, d)."""
    pe = torch.zeros(max_len, d_model)
    position = torch.arange(0, max_len, dtype=torch.float).unsqueeze(1)
    div_term = torch.exp(torch.arange(0, d_model, 2).float() * (-np.log(10000.0) / d_model))
    pe[:, 0::2] = torch.sin(position * div_term)
    pe[:, 1::2] = torch.cos(position * div_term)
    return pe.unsqueeze(0).transpose(0, 1)


def _encoder_layer(x: torch.Tensor, sd: Dict[str, torch.Tensor], pre: str, num_heads: int) -> torch.Tensor:
    """nn.TransformerEncoderLayer, norm_first=False, activation gelu (erf), eval mode, no masks. x: (S, B, d)."""
    S, B, d = x.shape
    dh = d // num_heads
    qkv = F.linear(x, sd[pre + "self_attn.in_proj_weight"], sd[pre + "self_attn.in_proj_bias"])
    q, k, v = qkv.chunk(3, dim=-1)

    def heads(t):  # (S, B, d) -> (B, H, S, dh)
        return t.reshape(S, B, num_heads, dh).permute(1, 2, 0, 3)

    q, k, v = heads(q), heads(k), heads(v)
    att = torch.softmax(q @ k.transpose(-1, -2) / math.sqrt(dh), dim=-1)
    a = (att @ v).permute(2, 0, 1, 3).reshape(S, B, d)
    a = F.linear(a, sd[pre + "self_attn.out_proj.weight"], sd[pre + "self_attn.out_proj.bias"])
    x = F.layer_norm(x + a, (d,), sd[pre + "norm1.weight"], sd[pre + "norm1.bias"], 1e-5)
    h = F.gelu(F.linear(x, sd[pre + "linear1.weight"], sd[pre + "linear1.bias"]))
    h = F.linear(h, sd[pre + "linear2.weight"], sd[pre + "linear2.bias"])
    return F.layer_norm(x + h, (d,), sd[pre + "norm2.weight"], sd[pre + "norm2.bias"], 1e-5)


def num_layers_of(sd: Dict[str, torch.Tensor]) -> int:
    return 1 + max(int(k.split(".")[2]) for k in sd if k.startswith("seqTransEncoder.layers."))


def mdm_forward(sd: Dict[str, torch.Tensor], x: torch.Tensor, timesteps: torch.Tensor,
                cond_emb: Optional[torch.Tensor] = None, uncond: bool = False, num_heads: int = 4) -> torch.Tensor:
    """MDM.forward for arch='trans_enc' (mdm.py:239-306).

    x (B, njoints, 1, nframes) fp32; timesteps (B,) int64, ORIGINAL-process indices;
    cond_emb (B, 512): what encode_text returns (only for cond_mode='text'); uncond: y['uncond'].
    """
    bs, njoints, nfeats, nframes = x.shape
    pe = sd["sequence_pos_encoder.pe"]
    # TimestepEmbedder (mdm.py:351-353)
    emb = F.linear(F.silu(F.linear(pe[timesteps], sd["embed_timestep.time_embed.0.weight"],
                                   sd["embed_timestep.time_embed.0.bias"])),
                   sd["embed_timestep.time_embed.2.weight"], sd["embed_timestep.time_embed.2.bias"]).permute(1, 0, 2)
    if cond_emb is not None:
        # emb += embed_text(mask_cond(enc_text, force_mask))   (mdm.py:248-251, :188-191)
        c = torch.zeros_like(cond_emb) if uncond else cond_emb
        emb = emb + F.linear(c, sd["embed_text.weight"], sd["embed_text.bias"])
    # InputProcess (mdm.py:366-372)
    h = x.permute(3, 0, 1, 2).reshape(nframes, bs, njoints * nfeats)
    h = F.linear(h, sd["input_process.poseEmbedding.weight"], sd["input_process.poseEmbedding.bias"])
    xseq = torch.cat((emb, h), dim=0)
    xseq = xseq + pe[: xseq.shape[0]]  # dropout is identity in eval
    for i in range(num_layers_of(sd)):
        xseq = _encoder_layer(xseq, sd, f"seqTransEncoder.layers.{i}.", num_heads)
    out = xseq[1:]
    out = F.linear(out, sd["output_process.poseFinal.weight"], sd["output_process.poseFinal.bias"])
    return out.reshape(nframes, bs, njoints, nfeats).permute(1, 2, 3, 0)


def cfg_forward(sd, x, timesteps, cond_emb, text_scale: torch.Tensor, num_heads: int = 4) -> torch.Tensor:
    """ClassifierFreeSampleModel.forward (cfg_sampler.py:25-35)."""
    out = mdm_forward(sd, x, timesteps, cond_emb, uncond=False, num_heads=num_heads)
    out_uncond = mdm_forward(sd, x, timesteps, cond_emb, uncond=True, num_heads=num_heads)
    return out_uncond + (text_scale.view(-1, 1, 1, 1) * (out - out_uncond))


# ------------------------------------------------------------------------------------------------
# MDM_UNET (model/mdm_unet.py): the denoiser of the published CondMDI checkpoints  (SURVEY.md 8f-4, 8f-1)
# ------------------------------------------------------------------------------------------------
def _unrounded(t):
    return t


def _conv_gn(x, sd, conv: str, gn: str, groups: int = 8, q=None):
    """Conv1d(k, padding=k//2) -> GroupNorm(8)   (Conv1dBlock / Conv1dAdaGNBlock.block1, mdm_unet.py:33-88)"""
    q = q or _unrounded
    w = sd[conv + ".weight"]
    x = F.conv1d(q(x), q(w), sd[conv + ".bias"], padding=w.shape[-1] // 2)
    return F.group_norm(x, groups, sd[gn + ".weight"], sd[gn + ".bias"], 1e-5)


def _residual_temporal_block(x, emb_mish, sd, pre: str, q=None):
    """ResidualTemporalBlock with adagn=True (mdm_unet.py:163-218): x (B, C_in, L), emb_mish = Mish(c) (B, 512)"""
    q = q or _unrounded
    cond = F.linear(q(emb_mish), q(sd[pre + "time_mlp.1.weight"]), sd[pre + "time_mlp.1.bias"]).unsqueeze(-1)  # (B, 2*C_out, 1)
    scale, shift = cond.chunk(2, dim=1)
    out = _conv_gn(x, sd, pre + "blocks.0.block1.0", pre + "blocks.0.block1.2", q=q)
    out = F.mish(out * (1 + scale) + shift)                                  # ada_shift_scale (:159-160) then Mish
    out = F.mish(_conv_gn(out, sd, pre + "blocks.1.block.0", pre + "blocks.1.block.2", q=q))
    if pre + "residual_conv.weight" in sd:
        x = F.conv1d(q(x), q(sd[pre + "residual_conv.weight"]), sd[pre + "residual_conv.bias"])
    return out + x


def unet_levels_of(sd) -> int:
    return 1 + max(int(k.split(".")[2]) for k in sd if k.startswith("unet.downs."))


def unet_forward(sd: Dict[str, torch.Tensor], x: torch.Tensor, timesteps: torch.Tensor, cond_emb: Optional[torch.Tensor] = None,
                 uncond: bool = False, obs_x0: Optional[torch.Tensor] = None, obs_mask: Optional[torch.Tensor] = None,
                 q=None) -> torch.Tensor:
    """MDM_UNET.forward + forward_core + TemporalUnet.forward (mdm_unet.py:765-849, :309-350), arch='unet', adagn,
    no attention, hml_vec.  keyframe-conditioned when obs_x0 / obs_mask are given (:778-783).

    q (test aid): a rounding applied to both operands (not the bias) of every convolution and of the time MLPs' linear
    layers, e.g. to bf16 to model one bf16 MMA per product; the timestep and text embeddings stay unrounded.  None: none."""
    q = q or _unrounded
    assert (obs_x0 is None) == (obs_mask is None)
    if obs_x0 is not None:
        x = obs_x0 * obs_mask + x * (~obs_mask)
        x = torch.cat([x, obs_mask.to(x.dtype)], dim=1)
    bs, njoints, nfeats, nframes = x.shape
    pe = sd["sequence_pos_encoder.pe"] if "sequence_pos_encoder.pe" in sd else sd["embed_timestep.sequence_pos_encoder.pe"]
    emb = F.linear(F.silu(F.linear(pe[timesteps], sd["embed_timestep.time_embed.0.weight"], sd["embed_timestep.time_embed.0.bias"])),
                   sd["embed_timestep.time_embed.2.weight"], sd["embed_timestep.time_embed.2.bias"]).permute(1, 0, 2)  # (1, B, d)
    if cond_emb is not None:
        cmask = torch.zeros_like(cond_emb) if uncond else cond_emb
        emb = emb + F.linear(cmask, sd["embed_text.weight"], sd["embed_text.bias"])
    emb = emb.squeeze(0)
    h = x.permute(3, 0, 1, 2).reshape(nframes, bs, njoints * nfeats)
    h = F.pad(h, (0, 0, 0, 0, 0, 224 - nframes), value=0)            # right-pad to the training length (:817)
    h = h.permute(1, 2, 0)                                            # 's b d -> b d s'
    c = F.linear(q(F.mish(F.linear(q(emb), q(sd["unet.time_mlp.0.weight"]), sd["unet.time_mlp.0.bias"]))),
                 q(sd["unet.time_mlp.2.weight"]), sd["unet.time_mlp.2.bias"])
    cm = F.mish(c)                                                    # every block's time_mlp starts with Mish (:183)
    levels = unet_levels_of(sd)
    skips = []
    for l in range(levels):
        h = _residual_temporal_block(h, cm, sd, f"unet.downs.{l}.0.", q)
        h = _residual_temporal_block(h, cm, sd, f"unet.downs.{l}.1.", q)
        skips.append(h)
        if l + 1 < levels:
            h = F.conv1d(q(h), q(sd[f"unet.downs.{l}.3.conv.weight"]), sd[f"unet.downs.{l}.3.conv.bias"], stride=2, padding=1)
    h = _residual_temporal_block(h, cm, sd, "unet.mid_block1.", q)
    h = _residual_temporal_block(h, cm, sd, "unet.mid_block2.", q)
    for i in range(levels - 1):
        h = torch.cat((h, skips.pop()), dim=1)
        h = _residual_temporal_block(h, cm, sd, f"unet.ups.{i}.0.", q)
        h = _residual_temporal_block(h, cm, sd, f"unet.ups.{i}.1.", q)
        h = F.conv_transpose1d(q(h), q(sd[f"unet.ups.{i}.3.conv.weight"]), sd[f"unet.ups.{i}.3.conv.bias"], stride=2, padding=1)
    h = F.mish(_conv_gn(h, sd, "unet.final_conv.0.block.0", "unet.final_conv.0.block.2", q=q))
    h = F.conv1d(q(h), q(sd["unet.final_conv.1.weight"]), sd["unet.final_conv.1.bias"])
    out = h.permute(2, 0, 1)[:nframes]                                # 'b d s -> s b d', drop the padding
    njoints_out = out.shape[-1]
    return out.reshape(nframes, bs, njoints_out, 1).permute(1, 2, 3, 0).float()


def random_unet_state_dict(seed: int = 0, dim: int = 512, mults: Sequence[int] = (2, 2, 2, 2), feats: int = 263,
                           keyframe_conditioned: bool = True, text: bool = False) -> Dict[str, torch.Tensor]:
    """Random weights with the MDM_UNET state-dict key set (arch='unet', adagn) at PyTorch-default-like scales -- every
    tensor non-zero (the reference's `zero=True` init would make a random-init model output zeros)."""
    g = torch.Generator().manual_seed(seed)

    def uni(shape, bound):
        return (torch.rand(*shape, generator=g) * 2 - 1) * bound

    sd: Dict[str, torch.Tensor] = {}

    def conv(key, co, ci, k, transposed=False):
        bound = 1.0 / math.sqrt(ci * k)
        sd[key + ".weight"] = uni((ci, co, k) if transposed else (co, ci, k), bound)
        sd[key + ".bias"] = uni((co,), bound)

    def gn(key, c):
        sd[key + ".weight"] = 1.0 + 0.1 * uni((c,), 1.0)
        sd[key + ".bias"] = 0.1 * uni((c,), 1.0)

    def lin(key, co, ci, gain=1.0):
        bound = gain / math.sqrt(ci)
        sd[key + ".weight"] = uni((co, ci), bound)
        sd[key + ".bias"] = uni((co,), bound)

    def rtb(pre, ci, co):
        conv(pre + "blocks.0.block1.0", co, ci, 5)
        gn(pre + "blocks.0.block1.2", co)
        conv(pre + "blocks.1.block.0", co, co, 5)
        gn(pre + "blocks.1.block.2", co)
        lin(pre + "time_mlp.1", 2 * co, dim, gain=0.5)
        if ci != co:
            conv(pre + "residual_conv", co, ci, 1)

    lin("unet.time_mlp.0", dim * 4, dim)
    lin("unet.time_mlp.2", dim, dim * 4)
    dims = [feats] + [int(dim * m) for m in mults]
    added = feats if keyframe_conditioned else 0
    n = len(mults)
    for l in range(n):
        rtb(f"unet.downs.{l}.0.", dims[l] + (added if l == 0 else 0), dims[l + 1])
        rtb(f"unet.downs.{l}.1.", dims[l + 1], dims[l + 1])
        if l + 1 < n:
            conv(f"unet.downs.{l}.3.conv", dims[l + 1], dims[l + 1], 3)
    rtb("unet.mid_block1.", dims[-1], dims[-1])
    rtb("unet.mid_block2.", dims[-1], dims[-1])
    for i, l in enumerate(range(n - 1, 0, -1)):           # reversed(in_out[1:]): (dim_in, dim_out) = (dims[l], dims[l + 1])
        rtb(f"unet.ups.{i}.0.", dims[l + 1] * 2, dims[l])
        rtb(f"unet.ups.{i}.1.", dims[l], dims[l])
        conv(f"unet.ups.{i}.3.conv", dims[l], dims[l], 4, transposed=True)
    conv("unet.final_conv.0.block.0", dims[1], dims[1], 5)
    gn("unet.final_conv.0.block.2", dims[1])
    conv("unet.final_conv.1", feats, dims[1], 1)
    sd["sequence_pos_encoder.pe"] = positional_encoding(dim)
    sd["embed_timestep.sequence_pos_encoder.pe"] = sd["sequence_pos_encoder.pe"]
    for j in (0, 2):
        lin(f"embed_timestep.time_embed.{j}", dim, dim)
    if text:
        lin("embed_text", dim, 512)
    return sd


# ------------------------------------------------------------------------------------------------
# keyframe masks and guidance schedule
# ------------------------------------------------------------------------------------------------


def hml_incidence_matrices():
    """MAT_POS / MAT_ROT / MAT_VEL / MAT_CNT (data_loaders/humanml_utils.py:68-91): 22 joints x 263 features."""
    pos = np.zeros((22, 263), dtype=bool)
    pos[0, 1:4] = True
    for j in range(1, 22):
        ub = 4 + 3 * j
        pos[j, ub - 3:ub] = True
    rot = np.zeros((22, 263), dtype=bool)
    rot[0, 0] = True
    for j in range(1, 22):
        ub = 4 + 21 * 3 + 6 * j
        rot[j, ub - 6:ub] = True
    vel = np.zeros((22, 263), dtype=bool)
    for j in range(0, 22):
        ub = 4 + 21 * 3 + 21 * 6 + 3 * (j + 1)
        vel[j, ub - 3:ub] = True
    cnt = np.zeros((22, 263), dtype=bool)
    cnt[7, -4] = True
    cnt[10, -3] = True
    cnt[8, -2] = True
    cnt[11, -1] = True
    return pos, rot, vel, cnt


def joint_to_full_mask(joint_mask: torch.Tensor, mode: str = "pos_rot_vel") -> torch.Tensor:
    """editing_util.py:30-44: (B, 22, 1, L) bool -> (B, 263, 1, L) bool."""
    assert mode in ["pos", "pos_rot", "pos_rot_vel"]
    pos, rot, vel, cnt = hml_incidence_matrices()
    jm = joint_mask.permute(2, 3, 0, 1).float()
    comps = [jm @ torch.tensor(pos).float(), jm @ torch.tensor(cnt).float()]
    if mode in ["pos_rot", "pos_rot_vel"]:
        comps.append(jm @ torch.tensor(rot).float())
    if mode == "pos_rot_vel":
        comps.append(jm @ torch.tensor(vel).float())
    mask = torch.stack([c.bool() for c in comps], dim=0).any(dim=0)
    return mask.permute(2, 3, 0, 1)


def get_keyframes_mask(data: torch.Tensor, lengths: torch.Tensor, edit_mode: str = "benchmark_sparse",
                       trans_length: int = 10, feature_mode: str = "pos_rot_vel", get_joint_mask: bool = False):
    """editing_util.py:56-229, inference-time modes benchmark_sparse (:85-91), benchmark_clip (:93-100), uncond."""
    batch_size, n_joints, n_features, n_frames = data.shape
    assert n_joints == 263
    obs_joint_mask = torch.zeros((batch_size, 22, n_features, n_frames), dtype=torch.bool)
    if edit_mode == "benchmark_sparse":
        for i, length in enumerate(lengths.cpu().numpy()):
            gt = np.array(range(int(length))[::trans_length])
            obs_joint_mask[i, :, :, gt] = True
    elif edit_mode == "benchmark_clip":
        for i, length in enumerate(lengths.cpu().numpy()):
            length = int(length)
            end_frame = (length - trans_length) // 2
            gt = np.array(list(range(end_frame)) + list(range(end_frame + trans_length, length)))
            obs_joint_mask[i, :, :, gt] = True
    elif edit_mode == "uncond":
        pass
    else:
        raise NotImplementedError(edit_mode)
    obs_feature_mask = joint_to_full_mask(obs_joint_mask, mode=feature_mode)
    if get_joint_mask:
        return obs_feature_mask, obs_joint_mask
    return obs_feature_mask


def get_gradient_schedule(schedule_name=None, num_diffusion_steps: int = 1000, scale: float = .05) -> np.ndarray:
    """editing_util.py:299-322."""
    if schedule_name is None:
        return np.ones(num_diffusion_steps)
    if schedule_name == "first-half":
        return np.concatenate((np.ones(num_diffusion_steps // 2), np.zeros(num_diffusion_steps - num_diffusion_steps // 2)))
    if schedule_name == "last-half":
        return np.concatenate((np.zeros(num_diffusion_steps // 2), np.ones(num_diffusion_steps // 2)))
    if schedule_name == "exponential":
        ts = np.arange(num_diffusion_steps)[::-1]
        return np.exp(-scale * ts)
    if schedule_name == "sigmoid":
        ts = np.arange(num_diffusion_steps)
        scale /= 5
        return 1 / (1 + np.exp(scale * (-ts + num_diffusion_steps / 2)))
    if schedule_name == "half-sigmoid":
        ts = np.arange(num_diffusion_steps)
        scale /= 5
        return 1 / (1 + np.exp(scale * (-ts)))
    raise NotImplementedError(schedule_name)


# ------------------------------------------------------------------------------------------------
# sampler
# ------------------------------------------------------------------------------------------------


@dataclass
class Conditioning:
    """What the reference passes as model_kwargs['y'] (+ wrapper choice), reduced to tensors."""
    cond_emb: Optional[torch.Tensor] = None      # (B, 512) synthetic encode_text output; None -> cond_mode 'no_cond'
    cfg: bool = False                            # model wrapped in ClassifierFreeSampleModel
    text_scale: Optional[torch.Tensor] = None    # y['text_scale'] (B,)
    y_mask: Optional[torch.Tensor] = None        # y['mask'] (B,1,1,L) bool
    imputate: bool = False
    stop_imputation_at: int = 0
    replacement_distribution: str = "conditional"
    inpainted_motion: Optional[torch.Tensor] = None
    inpainting_mask: Optional[torch.Tensor] = None   # bool (B,263,1,L)
    reconstruction_guidance: bool = False
    reconstruction_weight: float = 20.0
    gradient_schedule: Optional[str] = None
    diffusion_steps: int = 1000
    stop_recguidance_at: int = 0
    # top-level model_kwargs of sample/conditional_synthesis.py:159-162 (consumed by MDM_UNET.forward, ignored by MDM)
    obs_x0: Optional[torch.Tensor] = None
    obs_mask: Optional[torch.Tensor] = None      # bool (B,263,1,L)


def is_unet(sd) -> bool:
    return "unet.time_mlp.0.weight" in sd


def _model(sd, x, t_model, c: Conditioning):
    if is_unet(sd):
        if c.cfg:
            out = unet_forward(sd, x, t_model, c.cond_emb, False, c.obs_x0, c.obs_mask)
            out_u = unet_forward(sd, x, t_model, c.cond_emb, True, c.obs_x0, c.obs_mask)
            return out_u + (c.text_scale.view(-1, 1, 1, 1) * (out - out_u))  # cfg_sampler.py:25-35
        return unet_forward(sd, x, t_model, c.cond_emb, False, c.obs_x0, c.obs_mask)
    if c.cfg:
        return cfg_forward(sd, x, t_model, c.cond_emb, c.text_scale)
    return mdm_forward(sd, x, t_model, c.cond_emb)


def p_mean_variance(sd, tab: DiffusionTables, x: torch.Tensor, t: torch.Tensor, c: Conditioning):
    """gaussian_diffusion.py:352-534 for START_X / FIXED_SMALL through _WrappedModel (respace.py:128-133)."""
    t_model = torch.tensor(tab.timestep_map, dtype=t.dtype)[t]

    def eff_mask():
        m = c.y_mask.float() if c.y_mask is not None else torch.ones(x.shape[0], 1, 1, x.shape[-1])
        return (c.inpainting_mask * m).bool()

    need_rg = c.reconstruction_guidance and bool((t >= c.stop_recguidance_at).all())
    need_imp = c.imputate and bool((t >= c.stop_imputation_at).all())
    if need_rg:
        M = eff_mask()
        with torch.enable_grad():
            z = x.detach().requires_grad_(True)
            hat_x = _model(sd, z, t_model, c)
            loss = ((c.inpainted_motion - hat_x).square() * M).sum()
            grad = torch.autograd.grad(loss, z)[0] * (~M).float()
        hat_x = hat_x.detach()
        ws = get_gradient_schedule(c.gradient_schedule, c.diffusion_steps)
        w_r = extract(ws, t, grad.shape) * c.reconstruction_weight
        sab = extract(tab.sqrt_alphas_cumprod, t, grad.shape)
        tilde = hat_x - (w_r * sab / 2) * grad
        model_output = (tilde * ~M) + (c.inpainted_motion * M) if need_imp else (tilde * ~M) + (hat_x * M)
    elif need_imp:
        if c.replacement_distribution == "conditional":
            M = eff_mask()
            hat_x = _model(sd, x, t_model, c)
            model_output = (hat_x * ~M) + (c.inpainted_motion * M)
        elif c.replacement_distribution == "marginal":
            model_output = _model(sd, x, t_model, c)
        else:
            raise NotImplementedError
    else:
        model_output = _model(sd, x, t_model, c)
    log_variance = extract(tab.posterior_log_variance_clipped, t, x.shape)
    pred_xstart = model_output
    mean = extract(tab.posterior_mean_coef1, t, x.shape) * pred_xstart + extract(tab.posterior_mean_coef2, t, x.shape) * x
    return {"mean": mean, "log_variance": log_variance, "pred_xstart": pred_xstart, "model_output": model_output}


def p_sample(sd, tab, x, t, c: Conditioning, noise: torch.Tensor):
    """gaussian_diffusion.py:656-713."""
    out = p_mean_variance(sd, tab, x, t, c)
    nonzero = (t != 0).float().view(-1, *([1] * (len(x.shape) - 1)))
    sample = out["mean"] + nonzero * torch.exp(0.5 * out["log_variance"]) * noise
    return {"sample": sample, "pred_xstart": out["pred_xstart"]}


def ddim_sample(sd, tab, x, t, c: Conditioning, noise: torch.Tensor, eta: float = 0.0):
    """ddim_sample_with_grad with cond_fn=None (gaussian_diffusion.py:1358-1416); the autograd graph the
    reference builds there is discarded, so it is not restated."""
    out = p_mean_variance(sd, tab, x, t, c)
    x0 = out["pred_xstart"]
    eps = (extract(tab.sqrt_recip_alphas_cumprod, t, x.shape) * x - x0) / extract(tab.sqrt_recipm1_alphas_cumprod, t, x.shape)
    alpha_bar = extract(tab.alphas_cumprod, t, x.shape)
    alpha_bar_prev = extract(tab.alphas_cumprod_prev, t, x.shape)
    sigma = eta * torch.sqrt((1 - alpha_bar_prev) / (1 - alpha_bar)) * torch.sqrt(1 - alpha_bar / alpha_bar_prev)
    mean_pred = x0 * torch.sqrt(alpha_bar_prev) + torch.sqrt(1 - alpha_bar_prev - sigma ** 2) * eps
    nonzero = (t != 0).float().view(-1, *([1] * (len(x.shape) - 1)))
    sample = mean_pred + nonzero * sigma * noise
    return {"sample": sample, "pred_xstart": x0}


def sample_loop(sd, tab: DiffusionTables, shape: Sequence[int], c: Conditioning, tape: torch.Tensor,
                sampler: str = "ddpm", eta: float = 0.0, skip_timesteps: int = 0,
                init_image: Optional[torch.Tensor] = None, dump_steps: Optional[Sequence[int]] = None,
                max_steps: Optional[int] = None, return_all: bool = False):
    """p_sample_loop / ddim_sample_loop (gaussian_diffusion.py:1149-1297, :1454-1587).

    tape[0] is the initial randn(*shape) draw, tape[1 + k] the k-th randn_like draw of the loop.
    max_steps (test aid): stop after that many iterations and return the state reached.
    """
    img = tape[0].clone()
    if skip_timesteps and init_image is None:
        init_image = torch.zeros_like(img)
    indices = list(range(tab.num_timesteps - skip_timesteps))[::-1]
    if init_image is not None:
        my_t = torch.ones([shape[0]], dtype=torch.long) * indices[0]
        img = extract(tab.sqrt_alphas_cumprod, my_t, img.shape) * init_image + \
            extract(tab.sqrt_one_minus_alphas_cumprod, my_t, img.shape) * img  # q_sample (:311-328)
    dump, outs = [], []
    out = None
    with torch.no_grad():
        for k, i in enumerate(indices):
            if max_steps is not None and k >= max_steps:
                break
            t = torch.tensor([i] * shape[0])
            if sampler == "ddpm":
                out = p_sample(sd, tab, img, t, c, tape[1 + k])
            else:
                out = ddim_sample(sd, tab, img, t, c, tape[1 + k], eta)
            if dump_steps is not None and k in dump_steps:
                dump.append(out["pred_xstart"].clone())
            if return_all:
                outs.append(out)
            img = out["sample"]
    if return_all:
        return outs
    if dump_steps is not None:
        return dump
    return out["sample"]


def state_dict_of(module: torch.nn.Module) -> Dict[str, torch.Tensor]:
    return {k: v.detach().clone() for k, v in module.state_dict().items()}


def random_state_dict(seed: int = 0, layers: int = 8, d: int = 512, ff: int = 1024, feats: int = 263,
                      text: bool = False) -> Dict[str, torch.Tensor]:
    """Random weights with the MDM state-dict key set (SURVEY.md 8 a-W) and PyTorch-default-like scales.
    Used where the reference is not importable (GPU box): the parity tests only need SOME fixed weights."""
    g = torch.Generator().manual_seed(seed)

    def lin(out_f, in_f):
        bound = 1.0 / math.sqrt(in_f)
        w = (torch.rand(out_f, in_f, generator=g) * 2 - 1) * bound
        b = (torch.rand(out_f, generator=g) * 2 - 1) * bound
        return w, b

    sd: Dict[str, torch.Tensor] = {}
    sd["input_process.poseEmbedding.weight"], sd["input_process.poseEmbedding.bias"] = lin(d, feats)
    sd["sequence_pos_encoder.pe"] = positional_encoding(d)
    sd["embed_timestep.sequence_pos_encoder.pe"] = sd["sequence_pos_encoder.pe"]
    for j in (0, 2):
        sd[f"embed_timestep.time_embed.{j}.weight"], sd[f"embed_timestep.time_embed.{j}.bias"] = lin(d, d)
    for i in range(layers):
        p = f"seqTransEncoder.layers.{i}."
        bound = math.sqrt(6.0 / (d + 3 * d))  # xavier_uniform on in_proj_weight
        sd[p + "self_attn.in_proj_weight"] = (torch.rand(3 * d, d, generator=g) * 2 - 1) * bound
        sd[p + "self_attn.in_proj_bias"] = (torch.rand(3 * d, generator=g) * 2 - 1) * 0.02
        sd[p + "self_attn.out_proj.weight"], sd[p + "self_attn.out_proj.bias"] = lin(d, d)
        sd[p + "linear1.weight"], sd[p + "linear1.bias"] = lin(ff, d)
        sd[p + "linear2.weight"], sd[p + "linear2.bias"] = lin(d, ff)
        for n in ("norm1", "norm2"):
            sd[p + n + ".weight"] = 1.0 + 0.1 * (torch.rand(d, generator=g) * 2 - 1)
            sd[p + n + ".bias"] = 0.1 * (torch.rand(d, generator=g) * 2 - 1)
    sd["output_process.poseFinal.weight"], sd["output_process.poseFinal.bias"] = lin(feats, d)
    if text:
        sd["embed_text.weight"], sd["embed_text.bias"] = lin(d, 512)
    return sd


def golden_inputs(B: int = 2, D: int = 263, L: int = 196) -> Dict[str, torch.Tensor]:
    """Seeded inputs shared by oracle/make_golden.py (which stores the REFERENCE's outputs for them under
    tests/golden/sampler.npz) and the tests that replay them."""
    g = torch.Generator().manual_seed(1234)
    x = torch.randn(B, D, 1, L, generator=g)
    cond = torch.randn(B, 512, generator=g)
    x_obs = torch.randn(B, D, 1, L, generator=g)
    tape = torch.randn(8, B, D, 1, L, generator=g)
    scale = torch.tensor([2.5, 0.7])
    lengths = torch.tensor([196, 150])
    y_mask = (torch.arange(L)[None, :] < lengths[:, None]).view(B, 1, 1, L)
    kf_mask = get_keyframes_mask(x_obs, lengths, "benchmark_sparse", trans_length=5)
    return dict(x=x, cond=cond, x_obs=x_obs, tape=tape, text_scale=scale, lengths=lengths, y_mask=y_mask, kf_mask=kf_mask)


# ---------------------------------------------------------------------------------------------------
# post-processing: HumanML3D vectors -> joint positions
# (data_loaders/humanml/scripts/motion_process.py:402-441 recover_root_rot_pos, :474-489 recover_from_ric,
#  data_loaders/humanml/common/quaternion.py:16-20 qinv, :54-73 qrot; caller sample/synthesize.py:153-157)
# ---------------------------------------------------------------------------------------------------
def _rotate_about_y(cos_a: torch.Tensor, sin_a: torch.Tensor, v: torch.Tensor) -> torch.Tensor:
    """qrot(qinv(q), v) for q = (cos a, 0, sin a, 0), written out in qrot's operation order
    (v + 2 * (w * cross(u, v) + cross(u, cross(u, v))) with u = (0, -sin a, 0))."""
    uy = -sin_a
    x, y, z = v.unbind(-1)
    uv_x, uv_z = uy * z, -(uy * x)
    uuv_x, uuv_z = uy * uv_z, -(uy * uv_x)
    return torch.stack((x + 2 * (cos_a * uv_x + uuv_x), y, z + 2 * (cos_a * uv_z + uuv_z)), -1)


def recover_from_ric(data: torch.Tensor, joints_num: int, abs_3d: bool = False) -> torch.Tensor:
    """data (..., frames, feats) de-normalised -> (..., frames, joints_num, 3)."""
    data = data.float()
    if abs_3d:
        ang = data[..., 0]
    else:
        ang = torch.zeros_like(data[..., 0])
        ang[..., 1:] = data[..., :-1, 0]
        ang = torch.cumsum(ang, dim=-1)                    # :413-414
    cos_a, sin_a = torch.cos(ang), torch.sin(ang)
    root = torch.zeros(data.shape[:-1] + (3,))
    if abs_3d:
        root[..., 0], root[..., 2] = data[..., 1], data[..., 2]      # :425
    else:
        root[..., 1:, 0], root[..., 1:, 2] = data[..., :-1, 1], data[..., :-1, 2]   # :433
        root = torch.cumsum(_rotate_about_y(cos_a, sin_a, root), dim=-2)             # :434-435
    root[..., 1] = data[..., 3]                              # :437
    local = data[..., 4:(joints_num - 1) * 3 + 4].reshape(data.shape[:-1] + (joints_num - 1, 3))
    pos = _rotate_about_y(cos_a[..., None], sin_a[..., None], local)                # :480
    pos = torch.stack((pos[..., 0] + root[..., None, 0], pos[..., 1], pos[..., 2] + root[..., None, 2]), -1)  # :483-484
    return torch.cat((root[..., None, :], pos), dim=-2)     # :487


def sample_to_joints(sample: torch.Tensor, mean, std, joints_num: int = 22, abs_3d: bool = False) -> torch.Tensor:
    """sample/synthesize.py:153-157: (B, feats, 1, frames) normalised -> (B, joints_num, 3, frames)."""
    x = sample.float().permute(0, 2, 3, 1) * torch.as_tensor(std).float() + torch.as_tensor(mean).float()
    pos = recover_from_ric(x, joints_num, abs_3d)           # (B, 1, frames, J, 3)
    return pos.reshape(-1, *pos.shape[2:]).permute(0, 2, 3, 1)


def postprocess_inputs(B: int = 3, D: int = 263, L: int = 196) -> Dict[str, torch.Tensor]:
    """Seeded sampler-output-like tensors for the post-processing fixtures (tests/golden/postprocess.npz holds the
    dataset statistics used and the REFERENCE's outputs)."""
    g = torch.Generator().manual_seed(4321)
    return dict(sample=torch.randn(B, D, 1, L, generator=g), ragged=torch.randn(2, 1, 57, D, generator=g))


def long_loop_tape(B: int = 2, D: int = 263, L: int = 196, steps: int = 1000) -> torch.Tensor:
    """(1 + steps, B, D, 1, L) seeded noise of the full-length loop fixture (tests/golden/long_loop.npz); 412 MB."""
    return torch.randn(1 + steps, B, D, 1, L, generator=torch.Generator().manual_seed(2024))

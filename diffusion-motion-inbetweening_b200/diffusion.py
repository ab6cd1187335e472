"""Drop-in mirror of the reference's sampler classes, backed by the native H100 engine.

Mirrors (same names, argument meaning and error behaviour; paths relative to the reference repository):
    get_named_beta_schedule / betas_for_alpha_bar   diffusion/gaussian_diffusion.py:24-71
    ModelMeanType / ModelVarType / DiffusionConfig  :74-136
    GaussianDiffusion  (sampling half)              :139-241, :311-349, :1149-1297, :1418-1587, :1589-1804
                                                    + dpm_solver_sample_loop[_progressive] (DPM-Solver++, not in the reference)
                                                    + unipc_sample_loop[_progressive] (UniPC, not in the reference)
                                                    + dpm_solver_sde_sample_loop[_progressive] (SDE-DPM-Solver++,
                                                      not in the reference)
                                                    + repaint_sample_loop[_progressive] (RePaint resampling, not in
                                                      the reference)
    space_timesteps / SpacedDiffusion               diffusion/respace.py:9-62, :65-116
    create_gaussian_diffusion                       utils/model_util.py:122-165

`p_sample_loop` / `ddim_sample_loop` / `plms_sample_loop` / `ddim_reverse_sample_loop` / `dpm_solver_sample_loop` /
`unipc_sample_loop` / `dpm_solver_sde_sample_loop` / `repaint_sample_loop` run the WHOLE loop in one native
call (`cmdi_sample`): no per-step Python, no per-step H2D table copies, no per-step host sync (the reference syncs on
`(t >= stop_imputation_at).all()`, utils/editing_util.py:344).  What the reference computes per step in
`p_mean_variance` / `p_sample` / `ddim_sample_with_grad` / `plms_sample` / `ddim_reverse_sample` is done by the CUDA
kernels in csrc/.

Not accelerated (raise NotImplementedError, like the reference does for its own unsupported branches):
cond_fn / 'gmd' classifier guidance, learned variances, EPSILON/PREVIOUS_X parametrisations,
const_noise.  `reconstruction_guidance` runs a backward pass through the denoiser on the GPU (csrc/backward.cu).
"""
from __future__ import annotations

import enum
import math
from dataclasses import dataclass, field
from typing import List, Optional

import warnings

import numpy as np
import torch

from . import capi
from .editing_util import get_gradient_schedule
from .model import resolve_model


def get_named_beta_schedule(schedule_name, num_diffusion_timesteps, scale_betas=1.):
    if schedule_name == "linear":
        scale = scale_betas * 1000 / num_diffusion_timesteps
        return np.linspace(scale * 0.0001, scale * 0.02, num_diffusion_timesteps, dtype=np.float64)
    elif schedule_name == "cosine":
        return betas_for_alpha_bar(num_diffusion_timesteps, lambda t: math.cos((t + 0.008) / 1.008 * math.pi / 2) ** 2)
    raise NotImplementedError(f"unknown beta schedule: {schedule_name}")


def betas_for_alpha_bar(num_diffusion_timesteps, alpha_bar, max_beta=0.999):
    betas = []
    for i in range(num_diffusion_timesteps):
        t1 = i / num_diffusion_timesteps
        t2 = (i + 1) / num_diffusion_timesteps
        betas.append(min(1 - alpha_bar(t2) / alpha_bar(t1), max_beta))
    return np.array(betas)


class ModelMeanType(enum.Enum):
    PREVIOUS_X = enum.auto()
    START_X = enum.auto()
    EPSILON = enum.auto()


class ModelVarType(enum.Enum):
    LEARNED = enum.auto()
    FIXED_SMALL = enum.auto()
    FIXED_LARGE = enum.auto()
    LEARNED_RANGE = enum.auto()


@dataclass
class DiffusionConfig:
    betas: List = field(default_factory=list)
    model_mean_type: ModelMeanType = ModelMeanType.START_X
    model_var_type: ModelVarType = ModelVarType.FIXED_SMALL
    rescale_timesteps: bool = False
    # accepted for signature compatibility with the reference's DiffusionConfig (training-side options)
    extra: dict = field(default_factory=dict)


@dataclass(frozen=True)
class Window:
    """Sample motions longer than the denoiser's window as overlapping windows (`GaussianDiffusion.window`).

    A motion of N frames is covered by K = 1 + ceil((N - frames) / (frames - overlap)) windows of `frames` frames
    (K = 1 when N <= frames: the plain loop at N frames); window k starts at global frame
    f0(k) = min(k * (frames - overlap), N - frames), so the last one is end-aligned.  At every step the x0 of a frame
    that several windows cover (after CFG, reconstruction guidance and imputation) is replaced by their tent-weighted
    mean, w_k(g) = 1 + min(g - f0(k), f0(k) + frames - 1 - g), so the windows agree on their shared frames (the
    "handshake" of PriorMDM's DoubleTake, MultiDiffusion's averaging).  `frames` must be within the engine's limit for
    the architecture (207 for the transformer, 224 for MDM_UNET); 0 <= overlap <= frames // 2."""
    frames: int
    overlap: int = 0

    def __post_init__(self):
        for name in ("frames", "overlap"):
            v = getattr(self, name)
            if isinstance(v, bool) or not isinstance(v, (int, np.integer)):
                raise ValueError(f"Window {name} must be an int, got {v!r}")
        if self.frames < 1:
            raise ValueError(f"Window frames must be >= 1, got {self.frames}")
        if not 0 <= self.overlap <= self.frames // 2:
            raise ValueError(f"Window overlap must be in [0, frames // 2 = {self.frames // 2}], got {self.overlap}")

    def placement(self, n: int) -> List[int]:
        """First global frame of each window of an n-frame motion."""
        F, O = int(self.frames), int(self.overlap)
        if n <= F:
            return [0]
        K = 1 + -(-(n - F) // (F - O))
        return [min(k * (F - O), n - F) for k in range(K)]


def _crop_windows(x: torch.Tensor, f0: List[int], F: int) -> torch.Tensor:
    """(B, ..., N) in the global layout -> (B * K, ..., F): row b * K + k holds frames [f0[k], f0[k] + F) of sample b."""
    idx = torch.tensor(f0, device=x.device)[:, None] + torch.arange(F, device=x.device)
    return x[..., idx].movedim(-2, 1).reshape(x.shape[0] * len(f0), *x.shape[1:-1], F).contiguous()


def _window_prompts(text, B: int, K: int) -> list:
    """y['text'] of a windowed call as one prompt per window: B lists of K prompts (window k of sample b gets
    text[b][k]), or B prompts (every window of sample b gets text[b])."""
    if len(text) != B:
        raise ValueError(f"y['text'] must hold one entry per sample ({B}), got {len(text)}")
    if all(isinstance(t, (list, tuple)) for t in text):
        if any(len(t) != K for t in text):
            raise ValueError(f"per-window prompts: every sample needs one prompt per window ({K})")
        return [p for t in text for p in t]
    return [t for t in text for _ in range(K)]


def _enum_name(v) -> str:
    return getattr(v, "name", str(v))


class GaussianDiffusion:
    """Sampling half of the reference's GaussianDiffusion (gaussian_diffusion.py:139)."""

    def __init__(self, conf):
        self.conf = conf
        self.model_mean_type = conf.model_mean_type
        self.model_var_type = conf.model_var_type
        self.rescale_timesteps = bool(getattr(conf, "rescale_timesteps", False))
        betas = np.array(conf.betas, dtype=np.float64)
        self.betas = betas
        assert len(betas.shape) == 1, "betas must be 1-D"
        assert (betas > 0).all() and (betas <= 1).all()
        self.num_timesteps = int(betas.shape[0])
        alphas = 1.0 - betas
        self.alphas_cumprod = np.cumprod(alphas, axis=0)
        self.alphas_cumprod_prev = np.append(1.0, self.alphas_cumprod[:-1])
        self.alphas_cumprod_next = np.append(self.alphas_cumprod[1:], 0.0)
        self.sqrt_alphas_cumprod = np.sqrt(self.alphas_cumprod)
        self.sqrt_one_minus_alphas_cumprod = np.sqrt(1.0 - self.alphas_cumprod)
        self.log_one_minus_alphas_cumprod = np.log(1.0 - self.alphas_cumprod)
        self.sqrt_recip_alphas_cumprod = np.sqrt(1.0 / self.alphas_cumprod)
        self.sqrt_recipm1_alphas_cumprod = np.sqrt(1.0 / self.alphas_cumprod - 1)
        self.posterior_variance = betas * (1.0 - self.alphas_cumprod_prev) / (1.0 - self.alphas_cumprod)
        self.posterior_log_variance_clipped = np.log(np.append(self.posterior_variance[1], self.posterior_variance[1:]))
        self.posterior_mean_coef1 = betas * np.sqrt(self.alphas_cumprod_prev) / (1.0 - self.alphas_cumprod)
        self.posterior_mean_coef2 = (1.0 - self.alphas_cumprod_prev) * np.sqrt(alphas) / (1.0 - self.alphas_cumprod)
        if not hasattr(self, "timestep_map"):
            self.timestep_map = list(range(self.num_timesteps))
        # hook attributes the reference's eval code sets (gaussian_diffusion.py:238-241)
        self.data_transform_fn = None
        self.data_inv_transform_fn = None
        self.data_get_mean_fn = None
        self.log_trajectory_fn = None
        # engine options
        # capi.PRECISION_FP16 (MDM_UNET only) samples with CUDA autocast's fp16 arithmetic, as the reference does for
        # checkpoints with use_fp16; it is never chosen from conf.fp16 by itself
        self.precision = capi.PRECISION_BF16X3
        self.max_batch = None          # default: the batch of the first call
        self.noise_tape = None         # test aid: (1 + num_steps, B, njoints, 1, nframes) on the device
        self.use_graph = True
        self.sample_offset = 0         # global index of local sample 0 (multi-GPU sharding)
        # per-step noise: "torch" = the exact stream torch.randn_like would produce on this device from torch's CUDA
        # generator (a reference GPU run with the same seed draws the same noise; the generator is advanced as the
        # reference loop would advance it); "engine" = the engine's own counter-based generator keyed by the global
        # sample index (sharding-independent; used by distributed.sharded_sample)
        self.rng = "torch"
        self.engine_seed = None  # rng="engine": explicit Philox key (sharded_sample broadcasts rank 0's); None = draw one
        # Window(frames, overlap): shapes (B, D, 1, N) of any length run as overlapping windows blended at every step;
        # None = one denoiser window per sequence
        self.window = None

    # ------------------------------------------------------------------------------------------
    def q_sample(self, x_start, t, noise=None):
        """gaussian_diffusion.py:311-328 (host-side torch; the loop's own q_sample runs in the engine)."""
        if noise is None:
            noise = torch.randn_like(x_start)
        assert noise.shape == x_start.shape
        return (_extract_into_tensor(self.sqrt_alphas_cumprod, t, x_start.shape) * x_start +
                _extract_into_tensor(self.sqrt_one_minus_alphas_cumprod, t, x_start.shape) * noise)

    # ------------------------------------------------------------------------------------------
    def _check_supported(self, cond_fn, const_noise, randomize_class, model_kwargs):
        if const_noise:
            raise NotImplementedError()  # gaussian_diffusion.py:698-699, :1480-1481
        if randomize_class:
            raise NotImplementedError("randomize_class is a class-conditional feature the MDM path does not use")
        if _enum_name(self.model_mean_type) != "START_X" or _enum_name(self.model_var_type) != "FIXED_SMALL":
            raise NotImplementedError("the engine implements START_X / FIXED_SMALL (utils/model_util.py:142-148)")
        if self.rescale_timesteps:
            raise NotImplementedError("rescale_timesteps=True is not used by the reference (model_util.py:130)")
        y = model_kwargs["y"]  # the reference indexes it unconditionally (gaussian_diffusion.py:1280)
        if "gmd" in y.keys():
            raise NotImplementedError("'gmd' selects p_sample_with_grad (classifier guidance): out of scope")
        if y.get("reconstruction_guidance", False):
            assert "stop_recguidance_at" in y.keys()  # utils/editing_util.py:329-330
            assert "inpainting_mask" in y.keys() and "inpainted_motion" in y.keys()
        return y

    def _run(self, sampler, model, shape, noise, cond_fn, model_kwargs, device, skip_timesteps, init_image, randomize_class,
             dump_steps, const_noise, eta, progressive=False, order=2, num_steps=0, want_pred_xstart=False,
             variant="bh2", corrector=True, jump_length=10, jump_n_sample=10):
        if model_kwargs is None:
            model_kwargs = {}
        y = self._check_supported(cond_fn, const_noise, randomize_class, model_kwargs)
        plms = sampler == capi.SAMPLER_PLMS
        dpm = sampler == capi.SAMPLER_DPM_SOLVER
        unipc = sampler == capi.SAMPLER_UNIPC
        rev = sampler == capi.SAMPLER_DDIM_REVERSE  # `noise` is the state to invert; skip_timesteps its step index
        if sampler == capi.SAMPLER_DDPM:
            assert cond_fn is None, "only support the case where cond_fn is None"  # gaussian_diffusion.py:685
        elif cond_fn is not None:
            raise NotImplementedError("cond_fn (condition_score_with_grad) is out of scope")
        assert isinstance(shape, (tuple, list))
        inner, is_cfg = resolve_model(model)
        if device is None:
            device = next(model.parameters()).device
        device = torch.device(device)
        B = int(shape[0])
        # overlapping windows: f0 = their first frames, crop = a global-layout tensor -> the windows' rows
        f0 = None
        if self.window is not None:
            if rev or sampler == capi.SAMPLER_REPAINT:
                raise NotImplementedError("DDIM inversion and RePaint do not run on overlapping windows (diffusion.window)")
            if not isinstance(self.window, Window):
                raise TypeError(f"diffusion.window must be a Window or None, got {self.window!r}")
            f0 = self.window.placement(int(shape[-1]))
            f0 = f0 if len(f0) > 1 else None  # one window: the plain loop at N frames
        K, F = (len(f0), self.window.frames) if f0 else (1, int(shape[-1]))
        crop = (lambda t: None if t is None else _crop_windows(t, f0, F)) if f0 else (lambda t: t)
        eng = inner.engine_for(device, max_batch=max(B * K, self.max_batch or 0), precision=self.precision, nframes=F)
        eng.set_schedule(self.betas, self.timestep_map)

        # ---- conditioning ----
        cond_emb, text_scale, uncond = None, None, bool(y.get("uncond", False))
        cond_mode = getattr(inner, "cond_mode", "no_cond")
        if "action" in cond_mode:
            raise NotImplementedError("action conditioning is not on the HumanML3D path")
        if "text" in cond_mode:
            # with a window set, y['text'] may hold one prompt per window, also when one window covers the motion
            text = _window_prompts(y["text"], B, K) if self.window is not None else y["text"]
            cond_emb = inner.encode_text(text).to(device=device, dtype=torch.float32)  # once per loop (mdm.py:249 does it per step)
        if is_cfg:
            assert cond_mode in ["text", "action"]  # cfg_sampler.py:27
            text_scale = y["text_scale"].to(device=device, dtype=torch.float32).reshape(-1).repeat_interleave(K)
        # ---- keyframe imputation (gaussian_diffusion.py:427-442, editing_util.py:336-346) ----
        imputate, stop_at, obs, mask, y_mask = False, 0, None, None, None
        guided_cfg = bool(y.get("reconstruction_guidance", False))
        if "imputate" in y.keys() and y["imputate"]:
            assert "stop_imputation_at" in y.keys()
            assert "inpainting_mask" in y.keys() and "inpainted_motion" in y.keys()
            # the reconstruction-guidance branch (:405-425) imputes whenever requires_imputation() holds and never reads
            # replacement_distribution; only the un-guided branch (:427-442) dispatches on it
            dist = "conditional" if guided_cfg else y["replacement_distribution"]
            if dist == "conditional":
                imputate, stop_at = True, int(y["stop_imputation_at"])
                obs = y["inpainted_motion"].to(device=device, dtype=torch.float32)
                mask = y["inpainting_mask"].to(device=device)
                assert obs.shape == mask.shape == tuple(shape)
                obs, mask, y_mask = crop(obs), crop(mask), crop(y["mask"].to(device=device).reshape(B, -1))
            elif dist == "marginal":
                pass  # the reference's 'marginal' branch only calls the model (:437-439)
            else:
                raise NotImplementedError
        # ---- reconstruction guidance (gaussian_diffusion.py:405-425, editing_util.py:325-333) ----
        recon, stop_rg, coef = False, 0, None
        if y.get("reconstruction_guidance", False):
            recon, stop_rg = True, int(y["stop_recguidance_at"])
            if obs is None:
                obs = y["inpainted_motion"].to(device=device, dtype=torch.float32)
                mask = y["inpainting_mask"].to(device=device)
                assert obs.shape == mask.shape == tuple(shape)  # :414
                obs, mask, y_mask = crop(obs), crop(mask), crop(y["mask"].to(device=device).reshape(B, -1))
            # w_r[t] * sqrt(alpha_bar_t) / 2, in fp32 exactly as the reference forms it (:418-422); the schedule is
            # indexed by the sampler step t like _extract_into_tensor(grad_ws, t, ...) does
            ws = get_gradient_schedule(y["gradient_schedule"], y["diffusion_steps"])
            tt = torch.arange(self.num_timesteps)
            w_r = torch.from_numpy(ws)[tt].float() * y["reconstruction_weight"]
            sab = torch.from_numpy(self.sqrt_alphas_cumprod)[tt].float()
            coef = (w_r * sab / 2).float().cpu().numpy()
        # ---- noise ----
        tape = self.noise_tape  # tape[0]: the initial randn(*shape) draw; tape[1 + k]: the k-th randn_like draw
        engine_rng = tape is None and self.rng != "torch"
        if noise is not None:
            x_T = noise.to(device=device, dtype=torch.float32)
        elif tape is not None:
            x_T = tape[0]
        elif engine_rng:
            # the engine draws x_T itself, keyed by (seed, sample_offset + b): rank r of a sharded run starts its
            # sample i from the x_T a single-GPU run gives global sample r*B/G + i (distributed.sharded_sample)
            x_T = None
        else:
            x_T = torch.randn(*shape, device=device)  # the reference's first draw (:1248)
        if tape is not None:
            tape = tape[1:]
        seed, rng_args = 0, {}
        if plms or rev or dpm or unipc:
            # plms_sample_loop_progressive draws nothing after x_T (:1767-1770): a tape contributes tape[0] only, torch's
            # generator has moved by the one randn(*shape) above, and the engine generator draws x_T when rng="engine".
            # DPM-Solver++ and UniPC behave the same way.  DDIM inversion draws nothing at all: x_T is the caller's state.
            # (SDE-DPM-Solver++ draws like p_sample_loop: the branch below.)
            tape = None
            if x_T is None:
                seed = self.engine_seed if self.engine_seed is not None else int(torch.randint(0, 2 ** 62, (1,)).item())
        elif tape is None:
            # one randn_like per loop iteration (:696, :1407); SDE-DPM-Solver++ draws the same way, RePaint once per op
            # of its walk
            n_draws = self.num_timesteps - skip_timesteps
            if sampler == capi.SAMPLER_REPAINT:
                n_draws = len(_repaint_walk(self.num_timesteps - 1 - skip_timesteps, jump_length, jump_n_sample))
            rng_args = _torch_stream_args(device, int(np.prod(shape)), n_draws, lazy=progressive) if self.rng == "torch" else None
            if rng_args is None:
                if x_T is not None and noise is None:
                    x_T = None  # torch-compatible stream unavailable in this build: fall through to the engine generator
                # per-step noise comes from the engine's counter-based generator, keyed by `engine_seed` (set by
                # sharded_sample: identical on all ranks) or by a draw from torch's global CPU generator, so `fixseed`
                # still makes runs reproducible
                seed = self.engine_seed if self.engine_seed is not None else int(torch.randint(0, 2 ** 62, (1,)).item())
                rng_args = {}
            else:
                seed = rng_args.pop("seed")
        if skip_timesteps and init_image is None and not rev:
            init_image = torch.zeros(tuple(shape), device=device, dtype=torch.float32)
        if init_image is not None:
            init_image = crop(init_image.to(device=device, dtype=torch.float32))
        # keyframe INPUT conditioning (MDM_UNET.forward's obs_x0 / obs_mask): top-level model_kwargs, as
        # sample/conditional_synthesis.py:159-162 passes them; the transformer ignores them
        kf_obs, kf_mask = None, None
        if eng.arch == capi.ARCH_UNET and model_kwargs.get("obs_x0") is not None:
            kf_obs = crop(model_kwargs["obs_x0"].to(device=device, dtype=torch.float32))
            kf_mask = crop(model_kwargs["obs_mask"].to(device=device))
        common = dict(batch=B * K, sampler=sampler, eta=eta, cond_emb=cond_emb, uncond=uncond, cfg=is_cfg, text_scale=text_scale,
                      obs_x0=kf_obs, obs_mask=kf_mask,
                      y_mask=y_mask, imputate=imputate, stop_imputation_at=stop_at, inpainted_motion=obs,
                      inpainting_mask=mask, seed=seed, sample_offset=self.sample_offset, use_graph=self.use_graph,
                      recon_guidance=recon, stop_recguidance_at=stop_rg, recon_coef=coef, **rng_args)
        if plms or dpm or sampler == capi.SAMPLER_DPM_SOLVER_SDE:
            common["plms_order" if plms else "dpm_order"] = int(order)
        if unipc:
            common.update(unipc_order=int(order), unipc_variant=capi.UNIPC_BH1 if variant == "bh1" else capi.UNIPC_BH2,
                          unipc_corrector=bool(corrector))
        if sampler == capi.SAMPLER_REPAINT:
            common.update(repaint_jump_length=int(jump_length), repaint_jump_n_sample=int(jump_n_sample))
        if f0:  # x_T, the noise and the outputs stay global (B, D, 1, N)
            common.update(window_frames0=f0, global_frames=int(shape[-1]))
        if progressive:
            return self._step_generator(eng, x_T, init_image, skip_timesteps, tape, common)
        if rev:
            return eng.sample(skip_timesteps=skip_timesteps, num_steps=num_steps, x_T=x_T, want_pred_xstart=want_pred_xstart,
                              **common)
        if plms or dpm or unipc:
            return eng.sample(skip_timesteps=skip_timesteps, init_image=init_image, x_T=x_T, **common)
        return eng.sample(skip_timesteps=skip_timesteps, init_image=init_image, x_T=x_T,
                          noise_tape=None if tape is None else tape, want_pred_xstart=False, dump_steps=dump_steps, **common)

    def _step_generator(self, eng, x_T, init_image, skip_timesteps, tape, common):
        """Generator form of every sampler: one native call per step (slower than the fused loop; kept for API parity),
        each starting from the previous call's sample and replaying the same step graph.  The multistep samplers
        (PLMS, DPM-Solver++ as ODE and SDE, UniPC) continue the history the engine keeps on the device (UniPC's
        corrected state included), and DDIM inversion draws nothing, so
        their samples equal the fused loop's bit for bit; a caller that stops an inversion early has a partial one.
        PLMS also yields old_eps, the values of the reference's history list at that yield (the reference yields one
        list it keeps mutating).  RePaint makes one call per denoise op, which also runs the undo ops before it, and
        yields the op's position as "t".  On overlapping windows every call crops the global state it starts from,
        which holds the bits every covering window holds, and PLMS yields no old_eps (its history is per window)."""
        common = dict(common)
        common["use_graph"] = 2 if common.get("use_graph", True) else 0  # one native call per step, same step graph every time
        plms = common["sampler"] == capi.SAMPLER_PLMS
        repaint = common["sampler"] == capi.SAMPLER_REPAINT
        unwindowed = "window_frames0" not in common
        torch_rng = common.get("rng_mode", capi.RNG_ENGINE) == capi.RNG_TORCH
        off0, inc = common.pop("aten_offset", 0), common.get("aten_increment", 0)
        T = self.num_timesteps
        # the native calls: (skip_timesteps of the position the call starts from, index of its first draw, its draws,
        # the position of its denoise op)
        calls = [(skip_timesteps + k, k, 1, None) for k in range(T - skip_timesteps)]
        if repaint:
            walk = _repaint_walk(T - 1 - skip_timesteps, common["repaint_jump_length"], common["repaint_jump_n_sample"])
            calls, d0 = [], 0
            for d, (p, undo) in enumerate(walk):
                if not undo:
                    start = walk[d0][0] - 1 if walk[d0][1] else walk[d0][0]
                    calls.append((T - 1 - start, d0, d + 1 - d0, p))
                    d0 = d + 1
        state = x_T
        for k, (skip, d0, n_draws, t) in enumerate(calls):
            call = {}
            if common["sampler"] != capi.SAMPLER_DDIM_REVERSE:  # an inversion has no q_sample and no history to resume
                call.update(resume=(k > 0), init_image=init_image if k == 0 else None)
            if torch_rng:
                call["aten_offset"] = off0 + d0 * inc  # each call starts at its own draw of the stream
            res = eng.sample(skip_timesteps=skip, num_steps=1, x_T=state, want_pred_xstart=True, want_old_eps=plms and unwindowed,
                             noise_tape=None if tape is None else tape[d0:], **call, **common)
            state = res["sample"]
            if torch_rng:
                # torch's generator moves one randn_like at a time, as the reference's loop moves it: a caller that
                # breaks out of the generator early leaves it where the reference would
                _advance_torch_generator(eng.device, n_draws * inc)
            step = {"sample": res["sample"], "pred_xstart": res["pred_xstart"]}
            if plms and unwindowed:
                step["old_eps"] = res["old_eps"]
            if repaint:
                step["t"] = t
            yield step

    # ------------------------------------------------------------------------------------------
    def p_sample_loop(self, model, shape, noise=None, clip_denoised=True, denoised_fn=None, cond_fn=None, model_kwargs=None,
                      device=None, progress=False, skip_timesteps=0, init_image=None, randomize_class=False,
                      cond_fn_with_grad=False, dump_steps=None, const_noise=False):
        """gaussian_diffusion.py:1149-1214. Returns the final sample, or the list of pred_xstart at `dump_steps`."""
        res = self._run(capi.SAMPLER_DDPM, model, shape, noise, cond_fn, model_kwargs, device, skip_timesteps, init_image,
                        randomize_class, dump_steps, const_noise, 0.0)
        if dump_steps is not None:
            return res["dump"]
        return res["sample"]

    def p_sample_loop_progressive(self, model, shape, noise=None, clip_denoised=True, denoised_fn=None, cond_fn=None,
                                  model_kwargs=None, device=None, progress=False, skip_timesteps=0, init_image=None,
                                  randomize_class=False, cond_fn_with_grad=False, const_noise=False):
        """gaussian_diffusion.py:1217-1297.  Returns the step generator; the configuration is validated at the call (the
        reference, a generator function, defers the same checks to the first next())."""
        return self._run(capi.SAMPLER_DDPM, model, shape, noise, cond_fn, model_kwargs, device, skip_timesteps,
                             init_image, randomize_class, None, const_noise, 0.0, progressive=True)

    def ddim_sample_loop(self, model, shape, noise=None, clip_denoised=True, denoised_fn=None, cond_fn=None,
                         model_kwargs=None, device=None, progress=False, eta=0.0, skip_timesteps=0, init_image=None,
                         randomize_class=False, cond_fn_with_grad=False, dump_steps=None, const_noise=False):
        """gaussian_diffusion.py:1454-1512."""
        if const_noise == True:  # noqa: E712  (:1480-1481)
            raise NotImplementedError()
        res = self._run(capi.SAMPLER_DDIM, model, shape, noise, cond_fn, model_kwargs, device, skip_timesteps, init_image,
                        randomize_class, dump_steps, const_noise, eta)
        if dump_steps is not None:
            return res["dump"]
        return res["sample"]

    def ddim_sample_loop_progressive(self, model, shape, noise=None, clip_denoised=True, denoised_fn=None, cond_fn=None,
                                     model_kwargs=None, device=None, progress=False, eta=0.0, skip_timesteps=0,
                                     init_image=None, randomize_class=False, cond_fn_with_grad=False):
        """gaussian_diffusion.py:1514-1587."""
        return self._run(capi.SAMPLER_DDIM, model, shape, noise, cond_fn, model_kwargs, device, skip_timesteps,
                             init_image, randomize_class, None, False, eta, progressive=True)

    def plms_sample_loop(self, model, shape, noise=None, clip_denoised=True, denoised_fn=None, cond_fn=None, model_kwargs=None,
                         device=None, progress=False, skip_timesteps=0, init_image=None, randomize_class=False,
                         cond_fn_with_grad=False, order=2):
        """gaussian_diffusion.py:1689-1736: pseudo linear multistep, deterministic after x_T.  The whole loop is one
        native call; the eps history stays on the device."""
        _check_plms_order(order)
        return self._run(capi.SAMPLER_PLMS, model, shape, noise, cond_fn, model_kwargs, device, skip_timesteps, init_image,
                         randomize_class, None, False, 0.0, order=order)["sample"]

    def plms_sample_loop_progressive(self, model, shape, noise=None, clip_denoised=True, denoised_fn=None, cond_fn=None,
                                     model_kwargs=None, device=None, progress=False, skip_timesteps=0, init_image=None,
                                     randomize_class=False, cond_fn_with_grad=False, order=2):
        """gaussian_diffusion.py:1738-1804.  Yields {"sample", "pred_xstart", "old_eps"} per step; the configuration is
        validated at the call (the reference defers its checks to the first next())."""
        _check_plms_order(order)
        return self._run(capi.SAMPLER_PLMS, model, shape, noise, cond_fn, model_kwargs, device, skip_timesteps, init_image,
                         randomize_class, None, False, 0.0, progressive=True, order=order)

    def dpm_solver_sample_loop(self, model, shape, noise=None, clip_denoised=True, denoised_fn=None, cond_fn=None,
                               model_kwargs=None, device=None, progress=False, skip_timesteps=0, init_image=None,
                               randomize_class=False, cond_fn_with_grad=False, order=2):
        """DPM-Solver++ multistep (Lu et al. 2022, data prediction) on this object's spaced steps, orders 1-3: one
        denoiser pass per step, through the same x0 pipeline as DDIM (CFG, keyframe input, imputation, reconstruction
        guidance).  Order 1 is DDIM at eta = 0.  Deterministic after x_T; the whole loop is one native call and the x0
        history stays on the device.  (The reference has no such sampler.)"""
        _check_dpm_order(order)
        _check_no_denoised_fn(denoised_fn)
        return self._run(capi.SAMPLER_DPM_SOLVER, model, shape, noise, cond_fn, model_kwargs, device, skip_timesteps,
                         init_image, randomize_class, None, False, 0.0, order=order)["sample"]

    def dpm_solver_sample_loop_progressive(self, model, shape, noise=None, clip_denoised=True, denoised_fn=None,
                                           cond_fn=None, model_kwargs=None, device=None, progress=False, skip_timesteps=0,
                                           init_image=None, randomize_class=False, cond_fn_with_grad=False, order=2):
        """Yields {"sample", "pred_xstart"} per step of dpm_solver_sample_loop, one native call per step; the samples
        equal the fused loop's bit for bit.  The configuration is validated at the call."""
        _check_dpm_order(order)
        _check_no_denoised_fn(denoised_fn)
        return self._run(capi.SAMPLER_DPM_SOLVER, model, shape, noise, cond_fn, model_kwargs, device, skip_timesteps,
                         init_image, randomize_class, None, False, 0.0, progressive=True, order=order)

    def dpm_solver_sde_sample_loop(self, model, shape, noise=None, clip_denoised=True, denoised_fn=None, cond_fn=None,
                                   model_kwargs=None, device=None, progress=False, skip_timesteps=0, init_image=None,
                                   randomize_class=False, cond_fn_with_grad=False, const_noise=False, order=2):
        """SDE-DPM-Solver++ multistep (Lu et al. 2022; the SDE solver in data prediction, midpoint form) on this object's
        spaced steps, orders 1-2: one denoiser pass per step, through the same x0 pipeline as p_sample_loop (CFG,
        keyframe input, imputation, reconstruction guidance).  Stochastic, with p_sample_loop's noise: one randn(*shape)
        for x_T, then one randn_like per step including the last, from the same source (`rng`, `noise_tape`).  Order 1 is
        p_sample_loop's posterior step; order 2 is second-order accurate in the step size.  The whole loop is one native
        call and the x0 history stays on the device.  (The reference has no such sampler.)"""
        _check_sde_order(order)
        _check_no_denoised_fn(denoised_fn)
        return self._run(capi.SAMPLER_DPM_SOLVER_SDE, model, shape, noise, cond_fn, model_kwargs, device, skip_timesteps,
                         init_image, randomize_class, None, const_noise, 0.0, order=order)["sample"]

    def dpm_solver_sde_sample_loop_progressive(self, model, shape, noise=None, clip_denoised=True, denoised_fn=None,
                                               cond_fn=None, model_kwargs=None, device=None, progress=False,
                                               skip_timesteps=0, init_image=None, randomize_class=False,
                                               cond_fn_with_grad=False, const_noise=False, order=2):
        """Yields {"sample", "pred_xstart"} per step of dpm_solver_sde_sample_loop, one native call per step; the samples
        equal the fused loop's bit for bit, and torch's generator moves one randn_like per yielded step, as
        p_sample_loop_progressive moves it.  The configuration is validated at the call."""
        _check_sde_order(order)
        _check_no_denoised_fn(denoised_fn)
        return self._run(capi.SAMPLER_DPM_SOLVER_SDE, model, shape, noise, cond_fn, model_kwargs, device, skip_timesteps,
                         init_image, randomize_class, None, const_noise, 0.0, progressive=True, order=order)

    def repaint_sample_loop(self, model, shape, noise=None, clip_denoised=True, denoised_fn=None, cond_fn=None,
                            model_kwargs=None, device=None, progress=False, skip_timesteps=0, init_image=None,
                            randomize_class=False, cond_fn_with_grad=False, const_noise=False, jump_length=10,
                            jump_n_sample=10):
        """RePaint resampling (Lugmayr et al. 2022, "time travel") around p_sample_loop, for in-betweening by imputation
        or reconstruction guidance.  The loop walks the spaced steps: it descends one p_sample at a time, and the first
        time it reaches a step t with t % jump_length == 0 (and jump_length steps above it) it re-noises the state
        jump_length steps up, one forward step q(x_p | x_{p-1}) at a time, and denoises that stretch again, jump_n_sample - 1
        times, so the generated frames can settle into agreement with the keyframes.  Each p_sample is p_sample_loop's
        step (CFG, keyframe input, imputation, guidance decided by its step).  The cost is about jump_n_sample times the
        denoiser passes.  Noise: one randn(*shape) for x_T, then one randn_like per op of the walk (`rng`, `noise_tape`);
        jump_n_sample=1 is p_sample_loop.  The whole walk is one native call.  (The reference has no such sampler.)"""
        _check_repaint_args(jump_length, jump_n_sample)
        _check_no_denoised_fn(denoised_fn)
        return self._run(capi.SAMPLER_REPAINT, model, shape, noise, cond_fn, model_kwargs, device, skip_timesteps,
                         init_image, randomize_class, None, const_noise, 0.0, jump_length=jump_length,
                         jump_n_sample=jump_n_sample)["sample"]

    def repaint_sample_loop_progressive(self, model, shape, noise=None, clip_denoised=True, denoised_fn=None,
                                        cond_fn=None, model_kwargs=None, device=None, progress=False, skip_timesteps=0,
                                        init_image=None, randomize_class=False, cond_fn_with_grad=False,
                                        const_noise=False, jump_length=10, jump_n_sample=10):
        """Yields {"sample", "pred_xstart", "t"} after each p_sample of repaint_sample_loop's walk ("t" its step), one
        native call per p_sample (with the re-noising ops before it); the samples equal the fused loop's bit for bit,
        and torch's generator moves one randn_like per op run.  The configuration is validated at the call."""
        _check_repaint_args(jump_length, jump_n_sample)
        _check_no_denoised_fn(denoised_fn)
        return self._run(capi.SAMPLER_REPAINT, model, shape, noise, cond_fn, model_kwargs, device, skip_timesteps,
                         init_image, randomize_class, None, const_noise, 0.0, progressive=True, jump_length=jump_length,
                         jump_n_sample=jump_n_sample)

    def unipc_sample_loop(self, model, shape, noise=None, clip_denoised=True, denoised_fn=None, cond_fn=None,
                          model_kwargs=None, device=None, progress=False, skip_timesteps=0, init_image=None,
                          randomize_class=False, cond_fn_with_grad=False, order=2, variant="bh2", corrector=True):
        """UniPC (Zhao et al. 2023; multistep, data prediction) on this object's spaced steps, orders 1-3, variant
        "bh1" or "bh2": one denoiser pass per step, through the same x0 pipeline as DDIM (CFG, keyframe input,
        imputation, reconstruction guidance).  With corrector=True each pass's x0 also corrects the state it was
        evaluated at (UniC), which raises the order by one at no extra pass.  Order 1 without the corrector is DDIM at
        eta = 0.  Deterministic after x_T; the whole loop is one native call and the x0 history and corrected state stay
        on the device.  (The reference has no such sampler.)"""
        _check_unipc_args(order, variant, corrector)
        _check_no_denoised_fn(denoised_fn)
        return self._run(capi.SAMPLER_UNIPC, model, shape, noise, cond_fn, model_kwargs, device, skip_timesteps,
                         init_image, randomize_class, None, False, 0.0, order=order, variant=variant,
                         corrector=corrector)["sample"]

    def unipc_sample_loop_progressive(self, model, shape, noise=None, clip_denoised=True, denoised_fn=None, cond_fn=None,
                                      model_kwargs=None, device=None, progress=False, skip_timesteps=0, init_image=None,
                                      randomize_class=False, cond_fn_with_grad=False, order=2, variant="bh2",
                                      corrector=True):
        """Yields {"sample", "pred_xstart"} per step of unipc_sample_loop, one native call per step: "sample" is the
        state the next pass evaluates (uncorrected), "pred_xstart" this pass's x0.  The samples equal the fused loop's
        bit for bit.  The configuration is validated at the call."""
        _check_unipc_args(order, variant, corrector)
        _check_no_denoised_fn(denoised_fn)
        return self._run(capi.SAMPLER_UNIPC, model, shape, noise, cond_fn, model_kwargs, device, skip_timesteps,
                         init_image, randomize_class, None, False, 0.0, progressive=True, order=order, variant=variant,
                         corrector=corrector)

    def ddim_reverse_sample(self, model, x, t, clip_denoised=True, denoised_fn=None, model_kwargs=None, eta=0.0):
        """gaussian_diffusion.py:1418-1452: x_t -> x_{t+1} by the reverse DDIM ODE, one native call.  Returns
        {"sample", "pred_xstart"}.  `t` must hold one step index for the whole batch (the engine's step index is per
        call)."""
        assert eta == 0.0, "Reverse ODE only for deterministic path"
        _check_no_denoised_fn(denoised_fn)
        ts = torch.as_tensor(t).reshape(-1)
        if ts.numel() != x.shape[0] or not bool((ts == ts[0]).all()):
            raise NotImplementedError("ddim_reverse_sample runs one step index for the whole batch: t must be uniform")
        res = self._run(capi.SAMPLER_DDIM_REVERSE, model, tuple(x.shape), x, None, model_kwargs, None, int(ts[0]), None, False,
                        None, False, 0.0, num_steps=1, want_pred_xstart=True)
        return {"sample": res["sample"], "pred_xstart": res["pred_xstart"]}

    def ddim_reverse_sample_loop(self, model, x_start, clip_denoised=True, denoised_fn=None, model_kwargs=None, device=None,
                                 progress=False, eta=0.0):
        """DDIM inversion of x_start: `for i in range(num_timesteps): x = ddim_reverse_sample(model, x, [i] * B)["sample"]`,
        the whole loop in one native call.  Returns x_T, the noise ddim_sample_loop(noise=x_T, ...) regenerates x_start
        from.  (The reference exposes the step only.)"""
        assert eta == 0.0, "Reverse ODE only for deterministic path"
        _check_no_denoised_fn(denoised_fn)
        return self._run(capi.SAMPLER_DDIM_REVERSE, model, tuple(x_start.shape), x_start, None, model_kwargs, device, 0, None,
                         False, None, False, 0.0)["sample"]

    def ddim_reverse_sample_loop_progressive(self, model, x_start, clip_denoised=True, denoised_fn=None, model_kwargs=None,
                                             device=None, progress=False, eta=0.0):
        """Yields ddim_reverse_sample's {"sample", "pred_xstart"} for t = 0, 1, ..., num_timesteps - 1, one native call per
        step; stopping early gives a partial inversion.  The configuration is validated at the call."""
        assert eta == 0.0, "Reverse ODE only for deterministic path"
        _check_no_denoised_fn(denoised_fn)
        return self._run(capi.SAMPLER_DDIM_REVERSE, model, tuple(x_start.shape), x_start, None, model_kwargs, device, 0, None,
                         False, None, False, 0.0, progressive=True)


def _check_no_denoised_fn(denoised_fn) -> None:
    if denoised_fn is not None:
        raise NotImplementedError("denoised_fn (a host callback on every x0) is not run by the engine")


def _check_plms_order(order) -> None:
    """plms_sample's check (gaussian_diffusion.py:1608-1609), and errors at the call for the orders the reference accepts
    there but cannot run: order 1 (its first step reads old_out["old_eps"] from None) and non-integral orders (the
    Adams-Bashforth branch has no weights for them)."""
    if not int(order) or not 1 <= order <= 4:
        raise ValueError("order is invalid (should be int from 1-4).")
    if order != int(order):
        raise NotImplementedError(f"PLMS order {order!r} is not an integer")
    if int(order) == 1:
        raise TypeError("PLMS order 1 fails on the reference's first step ('NoneType' object is not subscriptable)")


def _check_dpm_order(order) -> None:
    """DPM-Solver++'s multistep orders are 1, 2 and 3 (an int; bools and floats are refused)."""
    if isinstance(order, bool) or not isinstance(order, (int, np.integer)) or int(order) not in (1, 2, 3):
        raise ValueError(f"DPM-Solver++ order must be an int in {{1, 2, 3}}, got {order!r}")


def _check_sde_order(order) -> None:
    """SDE-DPM-Solver++'s multistep orders are 1 and 2 (an int; bools and floats are refused)."""
    if isinstance(order, bool) or not isinstance(order, (int, np.integer)) or int(order) not in (1, 2):
        raise ValueError(f"SDE-DPM-Solver++ order must be an int in {{1, 2}}, got {order!r}")


def _check_repaint_args(jump_length, jump_n_sample) -> None:
    """RePaint's jump_length and jump_n_sample are ints >= 1 (bools and floats are refused)."""
    for name, v in (("jump_length", jump_length), ("jump_n_sample", jump_n_sample)):
        if isinstance(v, bool) or not isinstance(v, (int, np.integer)) or int(v) < 1:
            raise ValueError(f"RePaint {name} must be an int >= 1, got {v!r}")


def _repaint_walk(t0: int, jump_length: int, jump_n_sample: int) -> list:
    """The engine's RePaint walk from position t0 (csrc/engine.cu, repaint_walk) as [(p, undo)]: a denoise op at p
    (p -> p - 1) or an undo op into p (p - 1 -> p).  The generators need it to split the walk into one call per denoise
    op and to count each call's draws."""
    walk = []
    for p in range(t0, -1, -1):
        if p % jump_length == 0 and p + jump_length <= t0:
            for _ in range(jump_n_sample - 1):
                walk += [(u, True) for u in range(p + 1, p + jump_length + 1)]
                walk += [(u, False) for u in range(p + jump_length, p, -1)]
        walk.append((p, False))
    return walk


def _check_unipc_args(order, variant, corrector) -> None:
    """UniPC's multistep orders are 1, 2 and 3 (an int; bools and floats are refused), its variants "bh1" and "bh2",
    and corrector a bool."""
    if isinstance(order, bool) or not isinstance(order, (int, np.integer)) or int(order) not in (1, 2, 3):
        raise ValueError(f"UniPC order must be an int in {{1, 2, 3}}, got {order!r}")
    if not isinstance(variant, str) or variant not in ("bh1", "bh2"):
        raise ValueError(f"UniPC variant must be 'bh1' or 'bh2', got {variant!r}")
    if not isinstance(corrector, (bool, np.bool_)):
        raise ValueError(f"UniPC corrector must be a bool, got {corrector!r}")


def space_timesteps(num_timesteps, section_counts):
    """respace.py:9-62."""
    if isinstance(section_counts, str):
        if section_counts.startswith("ddim"):
            desired_count = int(section_counts[len("ddim"):])
            for i in range(1, num_timesteps):
                if len(range(0, num_timesteps, i)) == desired_count:
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
        taken_steps = []
        for _ in range(section_count):
            taken_steps.append(start_idx + round(cur_idx))
            cur_idx += frac_stride
        all_steps += taken_steps
        start_idx += size
    return set(all_steps)


class SpacedDiffusion(GaussianDiffusion):
    """respace.py:65-116: keeps `use_timesteps` of the base process; the engine applies timestep_map on the device."""

    def __init__(self, use_timesteps, conf):
        self.use_timesteps = set(use_timesteps)
        self.timestep_map = []
        self.original_num_steps = len(conf.betas)
        base = GaussianDiffusion.__new__(GaussianDiffusion)
        GaussianDiffusion.__init__(base, conf)
        last_alpha_cumprod = 1.0
        new_betas = []
        for i, alpha_cumprod in enumerate(base.alphas_cumprod):
            if i in self.use_timesteps:
                new_betas.append(1 - alpha_cumprod / last_alpha_cumprod)
                last_alpha_cumprod = alpha_cumprod
                self.timestep_map.append(i)
        new_conf = DiffusionConfig(betas=np.array(new_betas), model_mean_type=conf.model_mean_type,
                                   model_var_type=conf.model_var_type,
                                   rescale_timesteps=bool(getattr(conf, "rescale_timesteps", False)))
        super().__init__(new_conf)


def create_gaussian_diffusion(noise_schedule="cosine", steps=1000, use_ddim=False, timestep_respacing=None,
                              predict_xstart=True, sigma_small=True):
    """utils/model_util.py:122-165 (the sampling-relevant arguments)."""
    if timestep_respacing is None:
        timestep_respacing = "ddim100" if use_ddim else ""
    betas = get_named_beta_schedule(noise_schedule, steps, 1.)
    if not timestep_respacing:
        timestep_respacing = [steps]
    return SpacedDiffusion(
        use_timesteps=space_timesteps(steps, timestep_respacing),
        conf=DiffusionConfig(betas=betas,
                             model_mean_type=ModelMeanType.START_X if predict_xstart else ModelMeanType.EPSILON,
                             model_var_type=ModelVarType.FIXED_SMALL if sigma_small else ModelVarType.FIXED_LARGE,
                             rescale_timesteps=False))


def from_reference_diffusion(ref_diffusion) -> SpacedDiffusion:
    """Build the engine-backed sampler from a reference GaussianDiffusion/SpacedDiffusion instance."""
    d = SpacedDiffusion.__new__(SpacedDiffusion)
    d.timestep_map = list(getattr(ref_diffusion, "timestep_map", range(ref_diffusion.num_timesteps)))
    d.use_timesteps = set(d.timestep_map)
    d.original_num_steps = getattr(ref_diffusion, "original_num_steps", ref_diffusion.num_timesteps)
    GaussianDiffusion.__init__(d, DiffusionConfig(betas=np.array(ref_diffusion.betas, dtype=np.float64),
                                                  model_mean_type=ref_diffusion.model_mean_type,
                                                  model_var_type=ref_diffusion.model_var_type,
                                                  rescale_timesteps=ref_diffusion.rescale_timesteps))
    for hook in ("data_transform_fn", "data_inv_transform_fn", "data_get_mean_fn", "log_trajectory_fn"):
        setattr(d, hook, getattr(ref_diffusion, hook, None))
    return d


_warned_policy = False
_policy_ok = {}


def aten_policy(numel: int, num_sms: int, max_threads_per_sm: int) -> tuple:
    """(threads, philox offset increment) of ATen's CUDA `normal_` kernel for `numel` elements
    (aten/src/ATen/native/cuda/DistributionTemplates.h: calc_execution_policy, block 256, unroll 4): the grid is
    min(SMs * resident blocks per SM, ceil(numel / 256)) blocks, every thread makes ceil(numel / (threads * 4)) calls
    of curand_normal4 and each call advances the generator offset by 4."""
    blocks = min(num_sms * (max_threads_per_sm // 256), (numel + 255) // 256)
    threads = 256 * blocks
    return threads, ((numel - 1) // (threads * 4) + 1) * 4


def aten_launch_policy(numel: int, device) -> tuple:
    prop = torch.cuda.get_device_properties(device)
    return aten_policy(numel, prop.multi_processor_count, prop.max_threads_per_multi_processor)


def _cuda_rng_state(device) -> tuple:
    st = torch.cuda.get_rng_state(device)
    if st.numel() != 16:
        raise NotImplementedError("unexpected CUDA generator state layout")
    raw = bytes(st.tolist())
    return int.from_bytes(raw[:8], "little"), int.from_bytes(raw[8:], "little")


def _advance_torch_generator(device, n_offsets: int) -> None:
    seed, off = _cuda_rng_state(device)
    new_state = torch.tensor(list(seed.to_bytes(8, "little") + (off + n_offsets).to_bytes(8, "little")), dtype=torch.uint8)
    torch.cuda.set_rng_state(new_state, device)


def _torch_stream_args(device, numel: int, n_draws: int, lazy: bool = False):
    """Engine arguments that continue torch's CUDA generator stream for `n_draws` randn_like draws of `numel`
    elements, and advance torch's generator past them.  None (with one warning) if this torch build's launch policy
    is not the one `aten_launch_policy` models -- verified by drawing one element block and watching the offset."""
    global _warned_policy
    key = (str(device), numel)
    try:
        threads, inc = aten_launch_policy(numel, device)
        seed, off = _cuda_rng_state(device)
        if key not in _policy_ok:
            probe = torch.cuda.get_rng_state(device)
            torch.empty(numel, device=device).normal_()
            _policy_ok[key] = _cuda_rng_state(device) == (seed, off + inc)
            torch.cuda.set_rng_state(probe, device)
        ok = _policy_ok[key]
    except Exception:  # noqa: BLE001  (state layout / property names differ in this torch build)
        ok = False
    if not ok or off % 4:
        if not _warned_policy:
            warnings.warn("torch-compatible noise stream unavailable for this torch build; using the engine generator")
            _warned_policy = True
        return None
    if not lazy:  # the fused loop consumes all its draws inside one native call; the generators advance per yielded step
        _advance_torch_generator(device, n_draws * inc)
    return dict(seed=seed, rng_mode=capi.RNG_TORCH, aten_offset=off, aten_increment=inc, aten_threads=threads)


def _extract_into_tensor(arr, timesteps, broadcast_shape):
    """gaussian_diffusion.py:2215-2228."""
    res = torch.from_numpy(arr).to(device=timesteps.device)[timesteps].float()
    while len(res.shape) < len(broadcast_shape):
        res = res[..., None]
    return res.expand(broadcast_shape)

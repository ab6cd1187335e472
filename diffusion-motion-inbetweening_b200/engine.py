"""Python handle of the native sampling engine (thin: torch supplies device memory and streams only)."""
from __future__ import annotations

import ctypes
from typing import Dict, Optional, Sequence

import numpy as np
import torch

from . import capi


def _ptr(t: Optional[torch.Tensor]) -> Optional[int]:
    return None if t is None else t.data_ptr()


def _stream_ptr(device: torch.device) -> int:
    return torch.cuda.current_stream(device).cuda_stream


class Engine:
    """One native engine per (device, weight set). See include/condmdi_b200.h for the C ABI it drives."""

    def __init__(self, device: torch.device, njoints: int = 263, nframes: int = 196, latent_dim: int = 512,
                 ff_size: int = 1024, num_layers: int = 8, num_heads: int = 4, max_batch: int = 64, has_text: bool = False,
                 precision: int = capi.PRECISION_BF16X3, arch: int = capi.ARCH_TRANS_ENC, unet_dim_mults: Sequence[int] = (),
                 keyframe_conditioned: bool = False):
        device = torch.device(device)
        if device.type != "cuda":
            raise RuntimeError("condmdi_b200 runs on CUDA devices only (no CPU fallback)")
        if not torch.cuda.is_available():
            raise RuntimeError("no CUDA device available: condmdi_b200 has no CPU fallback")
        self.lib = capi.load()
        self.device = torch.device("cuda", device.index if device.index is not None else torch.cuda.current_device())
        mults = (ctypes.c_int32 * 4)(*([int(m) for m in unet_dim_mults] + [0] * (4 - len(unet_dim_mults))))
        self.cfg = capi.ModelCfg(njoints, nframes, latent_dim, ff_size, num_layers, num_heads, max_batch, int(has_text),
                                 precision, int(arch), len(unet_dim_mults), mults, int(keyframe_conditioned))
        self.arch = int(arch)
        self.njoints, self.nframes, self.max_batch, self.has_text, self.precision = njoints, nframes, max_batch, has_text, precision
        handle = ctypes.c_void_p()
        capi.check(self.lib.cmdi_engine_create(ctypes.byref(self.cfg), self.device.index, ctypes.byref(handle)),
                   "cmdi_engine_create")
        self._h = handle
        self.schedule_key = None
        self._plms_steps = 0  # iterations of the engine's running PLMS history (mirrors the native side)

    def close(self):
        if getattr(self, "_h", None):
            self.lib.cmdi_engine_destroy(self._h)
            self._h = None

    def __del__(self):  # pragma: no cover
        try:
            self.close()
        except Exception:  # noqa: BLE001
            pass

    @property
    def launch_count(self) -> int:
        return int(self.lib.cmdi_launch_count(self._h))

    # ------------------------------------------------------------------------------------------
    def load_state_dict(self, sd: Dict[str, torch.Tensor]) -> None:
        """Upload an MDM.state_dict() (SURVEY.md 8 a-W). clip_model.* and the PE alias are ignored."""
        keep, descs = [], []
        for k, v in sd.items():
            if k.startswith("clip_model.") or k == "embed_timestep.sequence_pos_encoder.pe":
                continue
            t = v.detach().to(dtype=torch.float32).contiguous()
            keep.append(t)
            descs.append(capi.TensorDesc(k.encode(), t.data_ptr(), t.numel(), 0 if t.is_cuda else 1))
        arr = (capi.TensorDesc * len(descs))(*descs)
        with torch.cuda.device(self.device):
            capi.check(self.lib.cmdi_load_weights(self._h, arr, len(descs)), "cmdi_load_weights")
        del keep

    def set_schedule(self, betas: np.ndarray, timestep_map: Sequence[int]) -> None:
        betas = np.ascontiguousarray(np.asarray(betas, dtype=np.float64))
        tmap = np.ascontiguousarray(np.asarray(list(timestep_map), dtype=np.int64))
        key = (betas.tobytes(), tmap.tobytes())
        if key == self.schedule_key:
            return
        capi.check(self.lib.cmdi_set_schedule(self._h, betas.ctypes.data_as(ctypes.POINTER(ctypes.c_double)), len(betas),
                                              tmap.ctypes.data_as(ctypes.POINTER(ctypes.c_int64))), "cmdi_set_schedule")
        self.schedule_key = key
        self.num_timesteps = len(betas)

    # ------------------------------------------------------------------------------------------
    def forward(self, x: torch.Tensor, timestep: int, cond_emb: Optional[torch.Tensor] = None, uncond: bool = False,
                cfg: bool = False, text_scale: Optional[torch.Tensor] = None, obs_x0: Optional[torch.Tensor] = None,
                obs_mask: Optional[torch.Tensor] = None, keyframe_scale: Optional[torch.Tensor] = None) -> torch.Tensor:
        """MDM.forward / ClassifierFreeSampleModel.forward for a batch sharing one (original) timestep; keyframe_scale
        (B,): keyframe classifier-free guidance (cmdi_forward_args.keyframe_scale)."""
        host = not x.is_cuda
        x = x.to(torch.float32).contiguous()
        B = x.shape[0]
        out = torch.empty_like(x)

        def prep(t):
            if t is None:
                return None
            t = t.to(torch.float32).contiguous()
            return t.cpu() if host else t.to(self.device)

        cond_emb, text_scale, obs_x0, keyframe_scale = prep(cond_emb), prep(text_scale), prep(obs_x0), prep(keyframe_scale)
        if obs_mask is not None:
            obs_mask = obs_mask.to(torch.uint8).contiguous()
            obs_mask = obs_mask.cpu() if host else obs_mask.to(self.device)
        a = capi.ForwardArgs(B, _ptr(x), int(timestep), _ptr(cond_emb), int(uncond), int(cfg), _ptr(text_scale), int(host),
                             _ptr(obs_x0), _ptr(obs_mask), _ptr(keyframe_scale))
        with torch.cuda.device(self.device):
            capi.check(self.lib.cmdi_model_forward(self._h, ctypes.byref(a), out.data_ptr(), _stream_ptr(self.device)),
                       "cmdi_model_forward")
        return out

    def sample(self, batch: int, sampler: int = capi.SAMPLER_DDPM, eta: float = 0.0, skip_timesteps: int = 0,
               num_steps: int = 0, resume: bool = False, uncond: bool = False,
               init_image: Optional[torch.Tensor] = None, x_T: Optional[torch.Tensor] = None,
               noise_tape: Optional[torch.Tensor] = None, seed: int = 0, sample_offset: int = 0,
               rng_mode: int = capi.RNG_ENGINE, aten_offset: int = 0, aten_increment: int = 0, aten_threads: int = 0,
               cond_emb: Optional[torch.Tensor] = None, cfg: bool = False, text_scale: Optional[torch.Tensor] = None,
               y_mask: Optional[torch.Tensor] = None, imputate: bool = False, stop_imputation_at: int = 0,
               inpainted_motion: Optional[torch.Tensor] = None, inpainting_mask: Optional[torch.Tensor] = None,
               recon_guidance: bool = False, stop_recguidance_at: int = 0, recon_coef: Optional[Sequence[float]] = None,
               want_pred_xstart: bool = False, dump_steps: Optional[Sequence[int]] = None, host_buffers: bool = False,
               use_graph: bool = True, out: Optional[torch.Tensor] = None, obs_x0: Optional[torch.Tensor] = None,
               obs_mask: Optional[torch.Tensor] = None, plms_order: int = 2, want_old_eps: bool = False,
               dpm_order: int = 2, unipc_order: int = 2, unipc_variant: int = capi.UNIPC_BH2, unipc_corrector: bool = True,
               repaint_jump_length: int = 10, repaint_jump_n_sample: int = 10,
               window_frames0: Optional[Sequence[int]] = None, global_frames: int = 0, want_window_out: bool = False,
               joint_guidance: bool = False, stop_jointguidance_at: int = 0, joint_coef: Optional[Sequence[float]] = None,
               joint_target: Optional[torch.Tensor] = None, joint_mask: Optional[torch.Tensor] = None,
               joint_mean: Optional[torch.Tensor] = None, joint_std: Optional[torch.Tensor] = None, joint_abs3d: bool = False,
               keyframe_scale: Optional[torch.Tensor] = None, foot_contact: bool = False, stop_footcontact_at: int = 0,
               foot_contact_coef: Optional[Sequence[float]] = None, foot_contact_mask: Optional[torch.Tensor] = None,
               obstacle_guidance: bool = False, stop_obstacleguidance_at: int = 0,
               obstacle_coef: Optional[Sequence[float]] = None, obstacles: Optional[torch.Tensor] = None,
               obstacle_joints: int = 1, obstacle_mask: Optional[torch.Tensor] = None,
               stop_cfg_at: Optional[int] = None, start_cfg_at: Optional[int] = None):
        """The whole sampling loop in one native call. Tensors are in the reference layout (B, njoints, 1, nframes).

        host_buffers=False: every tensor must live on this engine's device; the result is a device tensor and the
        call is stream-ordered.  host_buffers=True: every tensor must be a CPU tensor (pinned for best speed); the
        H2D/D2H copies happen inside the call and the result is a CPU tensor valid on return.
        sampler=SAMPLER_PLMS: `plms_order` is plms_sample's order; want_old_eps adds result["old_eps"], the eps history
        list after the last step (oldest first), as plms_sample_loop_progressive yields it.
        sampler=SAMPLER_DDIM_REVERSE: DDIM inversion from the state x_T, ascending from t = skip_timesteps; plms_order
        is not sent.
        sampler=SAMPLER_DPM_SOLVER: DPM-Solver++ multistep of order `dpm_order` (1-3); resume continues its x0 history.
        sampler=SAMPLER_DPM_SOLVER_SDE: SDE-DPM-Solver++ of order `dpm_order` (1-2), with DDPM's per-step draws
        (noise_tape, seed / rng_mode); resume continues its x0 history.
        dpm_order is sent for these two samplers only, plms_order for the others.
        sampler=SAMPLER_UNIPC: UniPC of order `unipc_order` (1-3), variant `unipc_variant` (UNIPC_BH1 / UNIPC_BH2), with
        or without the corrector; resume continues its x0 history and corrected state.  The unipc_* fields are sent
        for this sampler only.
        sampler=SAMPLER_REPAINT: RePaint resampling around DDPM with `repaint_jump_length` / `repaint_jump_n_sample`
        (sent for this sampler only), one draw per op of its walk (noise_tape, seed / rng_mode); num_steps counts
        denoise ops, and resume continues the walk from the position it has reached (skip_timesteps = T - 1 - that
        position).
        window_frames0 / global_frames: overlapping windows (cmdi_sample_args.window_count): `batch` counts windows, row
        s * K + k is window k of global sample s and covers global frames [window_frames0[k], window_frames0[k] + nframes)
        of global_frames.  x_T, noise_tape and the outputs are global (batch // K, njoints, 1, global_frames); the other
        tensors are per window.  want_window_out adds result["windows"], the windows' final states.
        joint_*: joint-position guidance (cmdi_sample_args.joint_guidance): joint_target (batch, nframes, 22, 3) fp32,
        joint_mask of the same shape (y['mask'] folded in), joint_mean / joint_std (njoints,), joint_coef one entry per
        sampler step.
        keyframe_scale (batch,): keyframe classifier-free guidance (cmdi_sample_args.keyframe_scale), one entry per
        window under windows.
        foot_contact*: foot-contact guidance (cmdi_sample_args.foot_contact): foot_contact_coef one entry per sampler
        step, foot_contact_mask (batch, nframes) the valid frames or None; it reads joint_mean / joint_std / joint_abs3d,
        and joint_target / joint_mask only with joint_guidance.
        obstacle_*: obstacle-avoidance guidance (cmdi_sample_args.obstacle_guidance): obstacle_coef one entry per sampler
        step, obstacles (batch, K, 3) fp32 (c_x, c_z, r) with K <= capi.MAX_OBSTACLES, obstacle_joints the bit mask of
        the joint set, obstacle_mask (batch, nframes) the valid frames or None; it reads joint_mean / joint_std /
        joint_abs3d, and joint_target / joint_mask only with joint_guidance.
        stop_cfg_at / start_cfg_at: the CFG interval (cmdi_sample_args.cfg_interval): with cfg or keyframe_scale, either or
        both limit guidance to the steps stop_cfg_at <= t <= start_cfg_at; the other steps run the conditional pass alone.
        """
        shape = (batch, self.njoints, 1, self.nframes)
        K = 0 if window_frames0 is None else len(window_frames0)
        gshape = (batch // K, self.njoints, 1, int(global_frames)) if K else shape
        dev = torch.device("cpu") if host_buffers else self.device

        def prep(t, dtype=torch.float32, shp=None):
            if t is None:
                return None
            t = t.to(dtype)
            if shp is not None:
                t = t.reshape(shp)
            t = t.contiguous()
            if t.device != dev:
                raise ValueError(f"tensor on {t.device}, expected {dev} (host_buffers={host_buffers})")
            return t

        init_image, x_T = prep(init_image, shp=shape), prep(x_T, shp=gshape)
        cond_emb, text_scale = prep(cond_emb, shp=(batch, 512)), prep(text_scale, shp=(batch,))
        keyframe_scale = prep(keyframe_scale, shp=(batch,))
        y_mask = prep(y_mask, torch.uint8, (batch, self.nframes))
        inpainted_motion = prep(inpainted_motion, shp=shape)
        inpainting_mask = prep(inpainting_mask, torch.uint8, shape)
        obs_x0, obs_mask = prep(obs_x0, shp=shape), prep(obs_mask, torch.uint8, shape)
        if noise_tape is not None:
            noise_tape = noise_tape.to(torch.float32).contiguous()
            if noise_tape.device != self.device:
                raise ValueError("noise_tape must live on the engine's device")
        if out is None:
            out = torch.empty(gshape, dtype=torch.float32, device=dev, pin_memory=host_buffers)
        pred = torch.empty(gshape, dtype=torch.float32, device=dev, pin_memory=host_buffers) if want_pred_xstart else None
        windows = torch.empty(shape, dtype=torch.float32, device=dev, pin_memory=host_buffers) if want_window_out else None
        f0_arr = (ctypes.c_int32 * max(K, 1))(*[int(f) for f in (window_frames0 or [])])
        dump, dump_arr, n_dump = None, None, 0
        if dump_steps is not None:
            # one entry per loop iteration that matches, like the reference's `if i in dump_steps` (:1208-1213):
            # duplicates collapse and iterations the loop never reaches are dropped
            n_iter = self.num_timesteps - int(skip_timesteps)
            if num_steps:
                n_iter = min(n_iter, int(num_steps))
            steps_sorted = sorted({int(s) for s in dump_steps if 0 <= int(s) < n_iter})
            n_dump = len(steps_sorted)
            dump_arr = (ctypes.c_int32 * max(n_dump, 1))(*steps_sorted)
            dump = torch.empty((max(n_dump, 1),) + gshape, dtype=torch.float32, device=dev, pin_memory=host_buffers)
        coef_arr = None
        if recon_guidance:
            coef = np.ascontiguousarray(np.asarray(recon_coef, dtype=np.float32))
            if coef.shape != (self.num_timesteps,):
                raise ValueError(f"recon_coef must have one entry per sampler step ({self.num_timesteps})")
            coef_arr = coef.ctypes.data_as(ctypes.POINTER(ctypes.c_float))
        jcoef_arr = None
        if joint_guidance:
            jcoef = np.ascontiguousarray(np.asarray(joint_coef, dtype=np.float32))
            if jcoef.shape != (self.num_timesteps,):
                raise ValueError(f"joint_coef must have one entry per sampler step ({self.num_timesteps})")
            jcoef_arr = jcoef.ctypes.data_as(ctypes.POINTER(ctypes.c_float))
            joint_target = prep(joint_target, shp=(batch, self.nframes, 22, 3))
            joint_mask = prep(joint_mask, torch.uint8, (batch, self.nframes, 22, 3))
            joint_mean, joint_std = prep(joint_mean, shp=(self.njoints,)), prep(joint_std, shp=(self.njoints,))
        fcoef_arr = None
        if foot_contact:
            fcoef = np.ascontiguousarray(np.asarray(foot_contact_coef, dtype=np.float32))
            if fcoef.shape != (self.num_timesteps,):
                raise ValueError(f"foot_contact_coef must have one entry per sampler step ({self.num_timesteps})")
            fcoef_arr = fcoef.ctypes.data_as(ctypes.POINTER(ctypes.c_float))
            foot_contact_mask = prep(foot_contact_mask, torch.uint8, (batch, self.nframes))
            joint_mean, joint_std = prep(joint_mean, shp=(self.njoints,)), prep(joint_std, shp=(self.njoints,))
        ocoef_arr, n_obstacles = None, 0
        if obstacle_guidance:
            ocoef = np.ascontiguousarray(np.asarray(obstacle_coef, dtype=np.float32))
            if ocoef.shape != (self.num_timesteps,):
                raise ValueError(f"obstacle_coef must have one entry per sampler step ({self.num_timesteps})")
            ocoef_arr = ocoef.ctypes.data_as(ctypes.POINTER(ctypes.c_float))
            if obstacles is None or obstacles.dim() != 3 or obstacles.shape[0] != batch or obstacles.shape[2] != 3:
                raise ValueError(f"obstacles must be ({batch}, K, 3), got {tuple(getattr(obstacles, 'shape', ()))}")
            n_obstacles = int(obstacles.shape[1])
            obstacles = prep(obstacles) if n_obstacles else None
            obstacle_mask = prep(obstacle_mask, torch.uint8, (batch, self.nframes))
            joint_mean, joint_std = prep(joint_mean, shp=(self.njoints,)), prep(joint_std, shp=(self.njoints,))
        n_iter = self.num_timesteps - int(skip_timesteps)
        if num_steps:
            n_iter = min(n_iter, int(num_steps))
        plms_steps = n_iter + (self._plms_steps if resume else 0)  # iterations of the PLMS history after this call
        old_eps, n_old = None, 0
        if want_old_eps and sampler == capi.SAMPLER_PLMS:
            n_old = min(plms_steps, int(plms_order) - 1)  # the length of the reference's list after that many steps
            old_eps = torch.empty((max(n_old, 1),) + shape, dtype=torch.float32, device=dev, pin_memory=host_buffers)
        a = capi.SampleArgs(
            batch=batch, sampler=sampler, eta=float(eta), skip_timesteps=int(skip_timesteps), num_steps=int(num_steps),
            resume=int(resume), init_image=_ptr(init_image), x_T=_ptr(x_T), noise_tape=_ptr(noise_tape),
            seed=int(seed) & (2 ** 64 - 1), sample_offset=int(sample_offset), rng_mode=int(rng_mode),
            aten_offset=int(aten_offset), aten_increment=int(aten_increment), aten_threads=int(aten_threads),
            cond_emb=_ptr(cond_emb), uncond=int(uncond), cfg=int(cfg), text_scale=_ptr(text_scale), y_mask=_ptr(y_mask),
            imputate=int(imputate), stop_imputation_at=int(stop_imputation_at), inpainted_motion=_ptr(inpainted_motion),
            inpainting_mask=_ptr(inpainting_mask), recon_guidance=int(recon_guidance),
            stop_recguidance_at=int(stop_recguidance_at), recon_coef=coef_arr, pred_xstart_out=_ptr(pred),
            dump_xstart=_ptr(dump), dump_steps=dump_arr, n_dump=n_dump, host_buffers=int(host_buffers),
            use_graph=int(use_graph), obs_x0=_ptr(obs_x0), obs_mask=_ptr(obs_mask), plms_old_eps_out=_ptr(old_eps),
            window_count=K, window_frames0=f0_arr if K else None, global_frames=int(global_frames), window_out=_ptr(windows),
            joint_guidance=int(joint_guidance), stop_jointguidance_at=int(stop_jointguidance_at), joint_coef=jcoef_arr,
            joint_target=_ptr(joint_target), joint_mask=_ptr(joint_mask), joint_mean=_ptr(joint_mean),
            joint_std=_ptr(joint_std), joint_abs3d=int(joint_abs3d), keyframe_scale=_ptr(keyframe_scale),
            foot_contact=int(foot_contact), stop_footcontact_at=int(stop_footcontact_at), foot_contact_coef=fcoef_arr)
        # the sampler-specific fields go only to their sampler (the engine refuses them elsewhere)
        dpm = sampler in (capi.SAMPLER_DPM_SOLVER, capi.SAMPLER_DPM_SOLVER_SDE)
        if not dpm and sampler not in (capi.SAMPLER_DDIM_REVERSE, capi.SAMPLER_UNIPC, capi.SAMPLER_REPAINT):
            a.plms_order = int(plms_order)
        if dpm:
            a.dpm_order = int(dpm_order)
        if sampler == capi.SAMPLER_UNIPC:
            a.unipc_order, a.unipc_variant, a.unipc_corrector = int(unipc_order), int(unipc_variant), int(unipc_corrector)
        if sampler == capi.SAMPLER_REPAINT:
            a.repaint_jump_length, a.repaint_jump_n_sample = int(repaint_jump_length), int(repaint_jump_n_sample)
        if foot_contact:
            a.foot_contact_mask = _ptr(foot_contact_mask)
        if obstacle_guidance:
            a.obstacle_guidance, a.stop_obstacleguidance_at, a.obstacle_coef = 1, int(stop_obstacleguidance_at), ocoef_arr
            a.obstacles, a.n_obstacles, a.obstacle_joints = _ptr(obstacles), n_obstacles, int(obstacle_joints)
            a.obstacle_mask = _ptr(obstacle_mask)
        if stop_cfg_at is not None or start_cfg_at is not None:
            # a missing bound is one no step index reaches; the engine compares int32 step indices
            lo, hi = -2 ** 31, 2 ** 31 - 1
            a.cfg_interval = 1
            a.stop_cfg_at = lo if stop_cfg_at is None else min(max(int(stop_cfg_at), lo), hi)
            a.start_cfg_at = hi if start_cfg_at is None else min(max(int(start_cfg_at), lo), hi)
        with torch.cuda.device(self.device):
            capi.check(self.lib.cmdi_sample(self._h, ctypes.byref(a), out.data_ptr(), _stream_ptr(self.device)),
                       "cmdi_sample")
        result = {"sample": out}
        if sampler == capi.SAMPLER_PLMS:
            self._plms_steps = plms_steps
            if old_eps is not None:
                result["old_eps"] = [old_eps[i] for i in range(n_old)]
        if pred is not None:
            result["pred_xstart"] = pred
        if windows is not None:
            result["windows"] = windows
        if dump is not None:
            result["dump"] = [dump[i] for i in range(n_dump)]
        return result

    def profile_pass(self, batch: int, cfg: bool = False, repeats: int = 10):
        """[(kernel name, device ms)] for every launch of one denoiser pass (CUDA events between plain launches)."""
        cap = 2 + 7 * self.cfg.num_layers + 1
        ms = (ctypes.c_float * cap)()
        count = ctypes.c_int(0)
        with torch.cuda.device(self.device):
            capi.check(self.lib.cmdi_profile_pass(self._h, batch, int(cfg), int(repeats), ms, cap, ctypes.byref(count), _stream_ptr(self.device)),
                       "cmdi_profile_pass")
        nl = self.cfg.num_layers
        if count.value == 3 + 2 * nl:  # chained path: token rows, frame embedding, QKV_0, then {attention, chain} per layer
            names = ["token_rows", "frame_embed", "qkv"]
            for l in range(nl):
                names += ["attention", "chain" if l + 1 < nl else "chain_last"]
        else:
            fused = count.value == 2 + 5 * nl + 1
            per_layer = ["qkv", "attention", "out_proj_ln1", "ffn1", "ffn2_ln2"] if fused else \
                ["qkv", "attention", "out_proj", "ln1", "ffn1", "ffn2", "ln2"]
            names = ["token_rows", "frame_embed"]
            for _ in range(nl):
                names += per_layer
            names += ["out_head"]
        return list(zip(names, [ms[i] for i in range(count.value)]))

    # kernel-level entry points for the parity tests -------------------------------------------------
    def test_step(self, sampler, eta, t, model_out_c, model_out_u, text_scale, x_t, noise, impute, stop_at, x_obs, mask):
        B = x_t.shape[0]
        x_next = torch.empty_like(x_t)
        pred = torch.empty_like(x_t)
        with torch.cuda.device(self.device):
            capi.check(self.lib.cmdi_test_step(self._h, sampler, float(eta), int(t), B, _ptr(model_out_c), _ptr(model_out_u),
                                               _ptr(text_scale), _ptr(x_t), _ptr(noise), int(impute), int(stop_at), _ptr(x_obs),
                                               _ptr(mask), x_next.data_ptr(), pred.data_ptr(), _stream_ptr(self.device)),
                       "cmdi_test_step")
        return x_next, pred

    def test_input_vjp(self, x, timestep, inpainted_motion, inpainting_mask, cond_emb=None, uncond=False, cfg=False,
                       text_scale=None, obs_x0=None, obs_mask=None, keyframe_scale=None) -> torch.Tensor:
        """One guided evaluation and its input-VJP (cmdi_test_input_vjp): (passes, B, njoints, 1, nframes), the
        gradient of sum((inpainted_motion - x0_hat)^2 * inpainting_mask) w.r.t. x through each pass, cond pass first
        (passes = 1 + cfg + (keyframe_scale is not None), the keyframe-free pass last)."""
        dev = lambda t, dt=torch.float32: None if t is None else t.to(self.device, dt).contiguous()  # noqa: E731
        x = dev(x)
        B = x.shape[0]
        cond_emb, text_scale, obs_x0, inpainted_motion = dev(cond_emb), dev(text_scale), dev(obs_x0), dev(inpainted_motion)
        obs_mask, inpainting_mask, keyframe_scale = dev(obs_mask, torch.uint8), dev(inpainting_mask, torch.uint8), dev(keyframe_scale)
        passes = 1 + int(bool(cfg)) + int(keyframe_scale is not None)
        grad = torch.empty((passes,) + tuple(x.shape), dtype=torch.float32, device=self.device)
        a = capi.ForwardArgs(B, _ptr(x), int(timestep), _ptr(cond_emb), int(uncond), int(cfg), _ptr(text_scale), 0,
                             _ptr(obs_x0), _ptr(obs_mask), _ptr(keyframe_scale))
        with torch.cuda.device(self.device):
            capi.check(self.lib.cmdi_test_input_vjp(self._h, ctypes.byref(a), _ptr(inpainted_motion), _ptr(inpainting_mask),
                                                    grad.data_ptr(), _stream_ptr(self.device)), "cmdi_test_input_vjp")
        return grad

    def test_joint_input_vjp(self, x, timestep, joint_target, joint_mask, joint_mean, joint_std, joint_abs3d, c_j,
                             inpainted_motion=None, inpainting_mask=None, c_r=0.0, cond_emb=None, uncond=False, cfg=False,
                             text_scale=None, obs_x0=None, obs_mask=None, keyframe_scale=None) -> torch.Tensor:
        """test_input_vjp of the joint-guided seed (cmdi_test_joint_input_vjp): the gradient of
        c_r sum((inpainted_motion - x0_hat)^2 * inpainting_mask) + c_j sum(joint_mask * (P(x0_hat) - joint_target)^2)
        w.r.t. x through each pass, (passes, B, njoints, 1, nframes) as test_input_vjp returns it.  inpainted_motion
        None: the joint term alone."""
        dev = lambda t, dt=torch.float32: None if t is None else t.to(self.device, dt).contiguous()  # noqa: E731
        x = dev(x)
        B = x.shape[0]
        cond_emb, text_scale, obs_x0, inpainted_motion = dev(cond_emb), dev(text_scale), dev(obs_x0), dev(inpainted_motion)
        obs_mask, inpainting_mask = dev(obs_mask, torch.uint8), dev(inpainting_mask, torch.uint8)
        joint_target, joint_mask = dev(joint_target), dev(joint_mask, torch.uint8)
        joint_mean, joint_std, keyframe_scale = dev(joint_mean), dev(joint_std), dev(keyframe_scale)
        passes = 1 + int(bool(cfg)) + int(keyframe_scale is not None)
        grad = torch.empty((passes,) + tuple(x.shape), dtype=torch.float32, device=self.device)
        a = capi.ForwardArgs(B, _ptr(x), int(timestep), _ptr(cond_emb), int(uncond), int(cfg), _ptr(text_scale), 0,
                             _ptr(obs_x0), _ptr(obs_mask), _ptr(keyframe_scale))
        with torch.cuda.device(self.device):
            capi.check(self.lib.cmdi_test_joint_input_vjp(
                self._h, ctypes.byref(a), _ptr(inpainted_motion), _ptr(inpainting_mask), float(c_r), _ptr(joint_target),
                _ptr(joint_mask), _ptr(joint_mean), _ptr(joint_std), int(joint_abs3d), float(c_j), grad.data_ptr(),
                _stream_ptr(self.device)), "cmdi_test_joint_input_vjp")
        return grad

    def test_foot_contact_input_vjp(self, x, timestep, joint_mean, joint_std, joint_abs3d, c_c, valid=None, joint_target=None,
                                    joint_mask=None, c_j=0.0, inpainted_motion=None, inpainting_mask=None, c_r=0.0,
                                    cond_emb=None, uncond=False, cfg=False, text_scale=None, obs_x0=None, obs_mask=None,
                                    keyframe_scale=None) -> torch.Tensor:
        """test_joint_input_vjp with foot-contact guidance (cmdi_test_foot_contact_input_vjp): the gradient of
        c_r L_r + c_j L_j + c_c L_c w.r.t. x through each pass, (passes, B, njoints, 1, nframes).  valid (B, nframes): the
        valid frames (None: all).  joint_target None: no joint term; inpainted_motion None: no reconstruction term."""
        dev = lambda t, dt=torch.float32: None if t is None else t.to(self.device, dt).contiguous()  # noqa: E731
        x = dev(x)
        B = x.shape[0]
        cond_emb, text_scale, obs_x0, inpainted_motion = dev(cond_emb), dev(text_scale), dev(obs_x0), dev(inpainted_motion)
        obs_mask, inpainting_mask = dev(obs_mask, torch.uint8), dev(inpainting_mask, torch.uint8)
        joint_target, joint_mask, valid = dev(joint_target), dev(joint_mask, torch.uint8), dev(valid, torch.uint8)
        joint_mean, joint_std, keyframe_scale = dev(joint_mean), dev(joint_std), dev(keyframe_scale)
        if valid is not None:
            valid = valid.reshape(B, -1).contiguous()
        passes = 1 + int(bool(cfg)) + int(keyframe_scale is not None)
        grad = torch.empty((passes,) + tuple(x.shape), dtype=torch.float32, device=self.device)
        a = capi.ForwardArgs(B, _ptr(x), int(timestep), _ptr(cond_emb), int(uncond), int(cfg), _ptr(text_scale), 0,
                             _ptr(obs_x0), _ptr(obs_mask), _ptr(keyframe_scale))
        with torch.cuda.device(self.device):
            capi.check(self.lib.cmdi_test_foot_contact_input_vjp(
                self._h, ctypes.byref(a), _ptr(inpainted_motion), _ptr(inpainting_mask), float(c_r), _ptr(joint_target),
                _ptr(joint_mask), _ptr(joint_mean), _ptr(joint_std), int(joint_abs3d), float(c_j), _ptr(valid), float(c_c),
                grad.data_ptr(), _stream_ptr(self.device)), "cmdi_test_foot_contact_input_vjp")
        return grad

    @staticmethod
    def foot_contact_seed(*args, **kwargs) -> torch.Tensor:
        """foot_contact_seed (cmdi_foot_contact_seed), the seed kernel alone"""
        return foot_contact_seed(*args, **kwargs)

    def test_obstacle_input_vjp(self, x, timestep, joint_mean, joint_std, joint_abs3d, obstacles, c_o, obstacle_joints=1,
                                valid=None, foot_contact=False, c_c=0.0, joint_target=None, joint_mask=None, c_j=0.0,
                                inpainted_motion=None, inpainting_mask=None, c_r=0.0, cond_emb=None, uncond=False, cfg=False,
                                text_scale=None, obs_x0=None, obs_mask=None, keyframe_scale=None) -> torch.Tensor:
        """test_foot_contact_input_vjp with obstacle-avoidance guidance (cmdi_test_obstacle_input_vjp): the gradient of
        c_r L_r + c_j L_j + c_c L_c + c_o L_o w.r.t. x through each pass, (passes, B, njoints, 1, nframes).  obstacles
        (B, K, 3); obstacle_joints the bit mask of the joint set; valid (B, nframes): the valid frames of both the obstacle
        and the foot-contact term (None: all); foot_contact False: no contact term; joint_target None: no joint term;
        inpainted_motion None: no reconstruction term."""
        dev = lambda t, dt=torch.float32: None if t is None else t.to(self.device, dt).contiguous()  # noqa: E731
        x = dev(x)
        B = x.shape[0]
        cond_emb, text_scale, obs_x0, inpainted_motion = dev(cond_emb), dev(text_scale), dev(obs_x0), dev(inpainted_motion)
        obs_mask, inpainting_mask = dev(obs_mask, torch.uint8), dev(inpainting_mask, torch.uint8)
        joint_target, joint_mask, valid = dev(joint_target), dev(joint_mask, torch.uint8), dev(valid, torch.uint8)
        joint_mean, joint_std, keyframe_scale, obstacles = dev(joint_mean), dev(joint_std), dev(keyframe_scale), dev(obstacles)
        if valid is not None:
            valid = valid.reshape(B, -1).contiguous()
        K = int(obstacles.shape[1])
        passes = 1 + int(bool(cfg)) + int(keyframe_scale is not None)
        grad = torch.empty((passes,) + tuple(x.shape), dtype=torch.float32, device=self.device)
        a = capi.ForwardArgs(B, _ptr(x), int(timestep), _ptr(cond_emb), int(uncond), int(cfg), _ptr(text_scale), 0,
                             _ptr(obs_x0), _ptr(obs_mask), _ptr(keyframe_scale))
        with torch.cuda.device(self.device):
            capi.check(self.lib.cmdi_test_obstacle_input_vjp(
                self._h, ctypes.byref(a), _ptr(inpainted_motion), _ptr(inpainting_mask), float(c_r), _ptr(joint_target),
                _ptr(joint_mask), _ptr(joint_mean), _ptr(joint_std), int(joint_abs3d), float(c_j), _ptr(valid),
                int(bool(foot_contact)), float(c_c), _ptr(obstacles) if K else None, K, int(obstacle_joints), float(c_o),
                grad.data_ptr(), _stream_ptr(self.device)), "cmdi_test_obstacle_input_vjp")
        return grad

    @staticmethod
    def obstacle_seed(*args, **kwargs) -> torch.Tensor:
        """obstacle_seed (cmdi_obstacle_seed), the seed kernel alone"""
        return obstacle_seed(*args, **kwargs)

    def test_unet_ops(self, hook, x, timestep, cond_emb=None, uncond=False, cfg=False, text_scale=None, obs_x0=None,
                      obs_mask=None, inpainted_motion=None, inpainting_mask=None) -> torch.Tensor:
        """MDM_UNET (cmdi_test_unet_ops): the forward Engine.forward runs, or with inpainted_motion / inpainting_mask the
        guided forward and input-VJP Engine.test_input_vjp runs, calling hook(list, op, phase, info) on the host before
        (phase 0) and after (phase 1) each op is enqueued on the current stream; info is a capi.UnetOpInfo.  Returns what
        the wrapped call returns.  An exception the hook raises is re-raised after the call."""
        dev = lambda t, dt=torch.float32: None if t is None else t.to(self.device, dt).contiguous()  # noqa: E731
        x = dev(x)
        B = x.shape[0]
        vjp = inpainted_motion is not None
        cond_emb, text_scale, obs_x0, inpainted_motion = dev(cond_emb), dev(text_scale), dev(obs_x0), dev(inpainted_motion)
        obs_mask, inpainting_mask = dev(obs_mask, torch.uint8), dev(inpainting_mask, torch.uint8)
        out = torch.empty(((2 if cfg else 1,) if vjp else ()) + tuple(x.shape), dtype=torch.float32, device=self.device)
        errors = []

        def call(lst, op, phase, info, _user):
            if errors:
                return
            try:
                hook(lst, op, phase, info.contents)
            except BaseException as ex:  # noqa: BLE001 (ctypes would swallow it)
                errors.append(ex)

        cb = capi.UNET_OP_HOOK(call)
        a = capi.ForwardArgs(B, _ptr(x), int(timestep), _ptr(cond_emb), int(uncond), int(cfg), _ptr(text_scale), 0,
                             _ptr(obs_x0), _ptr(obs_mask))
        with torch.cuda.device(self.device):
            capi.check(self.lib.cmdi_test_unet_ops(self._h, ctypes.byref(a), int(vjp), _ptr(inpainted_motion), _ptr(inpainting_mask),
                                                   out.data_ptr(), cb, None, _stream_ptr(self.device)), "cmdi_test_unet_ops")
        if errors:
            raise errors[0]
        return out


def joint_guidance_seed(x0: torch.Tensor, target: torch.Tensor, mask: torch.Tensor, mean: torch.Tensor, std: torch.Tensor,
                        abs_3d: bool, ld: int = 0, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """cmdi_joint_guidance_seed: d/dx0 of sum(mask * (recover_from_ric(x0 * std + mean, 22, abs_3d) - target)^2) on a CUDA
    device; target / mask (B, L, 22, 3); mean / std (D,).  ld = 0: x0 in the reference layout (B, D, 1, L); ld >= D: x0
    frame-major (B, L, ld) with its first D columns the features (the engine's layout).  out: the result tensor (x0's
    shape), or None for a new one."""
    lib = capi.load()
    dev = x0.device
    if dev.type != "cuda":
        raise RuntimeError("joint_guidance_seed runs on CUDA devices only (no CPU fallback)")
    f = lambda t, dt=torch.float32: t.to(dev, dt).contiguous()  # noqa: E731
    x0, target, mask, mean, std = f(x0), f(target), f(mask, torch.uint8), f(mean), f(std)
    B, D = x0.shape[0], mean.shape[0]
    L = x0.shape[1] if ld else x0.shape[-1]
    want = (B, L, ld) if ld else (B, D, 1, L)
    if tuple(x0.shape) != want or target.shape != (B, L, 22, 3) or mask.shape != (B, L, 22, 3) or std.shape != (D,):
        raise ValueError("joint_guidance_seed: x0 must be (B, D, 1, L) (ld = 0) or (B, L, ld), target / mask (B, L, 22, 3) "
                         "and mean / std (D,)")
    grad = torch.empty_like(x0) if out is None else out
    with torch.cuda.device(dev):
        capi.check(lib.cmdi_joint_guidance_seed(_ptr(x0), B, D, L, int(ld), _ptr(target), _ptr(mask), _ptr(mean), _ptr(std),
                                                int(abs_3d), grad.data_ptr(), _stream_ptr(dev)), "cmdi_joint_guidance_seed")
    return grad


def foot_contact_seed(x0: torch.Tensor, mean: torch.Tensor, std: torch.Tensor, abs_3d: bool, valid: Optional[torch.Tensor] = None,
                      c_c: float = 1.0, target: Optional[torch.Tensor] = None, mask: Optional[torch.Tensor] = None,
                      c_j: float = 0.0, ld: int = 0, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """cmdi_foot_contact_seed: c_j dL_j/dx0 + c_c dL_c/dx0 on a CUDA device, L_c the foot-contact loss
    (cmdi_sample_args.foot_contact) with valid (B, L) the valid frames (None: all) and L_j joint_guidance_seed's loss
    (target / mask None: no joint term).  Layouts as joint_guidance_seed."""
    lib = capi.load()
    dev = x0.device
    if dev.type != "cuda":
        raise RuntimeError("foot_contact_seed runs on CUDA devices only (no CPU fallback)")
    f = lambda t, dt=torch.float32: None if t is None else t.to(dev, dt).contiguous()  # noqa: E731
    x0, mean, std, valid, target, mask = f(x0), f(mean), f(std), f(valid, torch.uint8), f(target), f(mask, torch.uint8)
    B, D = x0.shape[0], mean.shape[0]
    L = x0.shape[1] if ld else x0.shape[-1]
    want = (B, L, ld) if ld else (B, D, 1, L)
    if (tuple(x0.shape) != want or std.shape != (D,) or (valid is not None and valid.numel() != B * L) or
            (target is None) != (mask is None) or
            (target is not None and (target.shape != (B, L, 22, 3) or mask.shape != (B, L, 22, 3)))):
        raise ValueError("foot_contact_seed: x0 must be (B, D, 1, L) (ld = 0) or (B, L, ld), mean / std (D,), valid B * L "
                         "frames, and target / mask (B, L, 22, 3) both or neither")
    grad = torch.empty_like(x0) if out is None else out
    with torch.cuda.device(dev):
        capi.check(lib.cmdi_foot_contact_seed(_ptr(x0), B, D, L, int(ld), _ptr(valid), _ptr(target), _ptr(mask), _ptr(mean),
                                              _ptr(std), int(abs_3d), float(c_j), float(c_c), grad.data_ptr(), _stream_ptr(dev)),
                   "cmdi_foot_contact_seed")
    return grad


def obstacle_seed(x0: torch.Tensor, mean: torch.Tensor, std: torch.Tensor, abs_3d: bool, obstacles: torch.Tensor,
                  obstacle_joints: int = 1, c_o: float = 1.0, valid: Optional[torch.Tensor] = None, foot_contact: bool = False,
                  c_c: float = 0.0, target: Optional[torch.Tensor] = None, mask: Optional[torch.Tensor] = None,
                  c_j: float = 0.0, ld: int = 0, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """cmdi_obstacle_seed: c_j dL_j/dx0 + c_c dL_c/dx0 + c_o dL_o/dx0 on a CUDA device, L_o the obstacle loss
    (cmdi_sample_args.obstacle_guidance) of obstacles (B, K, 3) (c_x, c_z, r) over the joints of the bit mask
    obstacle_joints, with valid (B, L) the valid frames (None: all); L_c foot_contact_seed's loss when foot_contact (same
    valid); L_j joint_guidance_seed's loss (target / mask None: no joint term).  Layouts as joint_guidance_seed."""
    lib = capi.load()
    dev = x0.device
    if dev.type != "cuda":
        raise RuntimeError("obstacle_seed runs on CUDA devices only (no CPU fallback)")
    f = lambda t, dt=torch.float32: None if t is None else t.to(dev, dt).contiguous()  # noqa: E731
    x0, mean, std, valid, target, mask = f(x0), f(mean), f(std), f(valid, torch.uint8), f(target), f(mask, torch.uint8)
    obstacles = f(obstacles)
    B, D = x0.shape[0], mean.shape[0]
    L = x0.shape[1] if ld else x0.shape[-1]
    want = (B, L, ld) if ld else (B, D, 1, L)
    if (tuple(x0.shape) != want or std.shape != (D,) or (valid is not None and valid.numel() != B * L) or
            obstacles.dim() != 3 or obstacles.shape[0] != B or obstacles.shape[2] != 3 or
            (target is None) != (mask is None) or
            (target is not None and (target.shape != (B, L, 22, 3) or mask.shape != (B, L, 22, 3)))):
        raise ValueError("obstacle_seed: x0 must be (B, D, 1, L) (ld = 0) or (B, L, ld), mean / std (D,), obstacles "
                         "(B, K, 3), valid B * L frames, and target / mask (B, L, 22, 3) both or neither")
    K = int(obstacles.shape[1])
    grad = torch.empty_like(x0) if out is None else out
    with torch.cuda.device(dev):
        capi.check(lib.cmdi_obstacle_seed(_ptr(x0), B, D, L, int(ld), _ptr(valid), _ptr(target), _ptr(mask), _ptr(mean),
                                          _ptr(std), int(abs_3d), float(c_j), int(bool(foot_contact)), float(c_c),
                                          _ptr(obstacles) if K else None, K, int(obstacle_joints), float(c_o),
                                          grad.data_ptr(), _stream_ptr(dev)), "cmdi_obstacle_seed")
    return grad

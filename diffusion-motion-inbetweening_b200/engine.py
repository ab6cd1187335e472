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
                obs_mask: Optional[torch.Tensor] = None) -> torch.Tensor:
        """MDM.forward / ClassifierFreeSampleModel.forward for a batch sharing one (original) timestep."""
        host = not x.is_cuda
        x = x.to(torch.float32).contiguous()
        B = x.shape[0]
        out = torch.empty_like(x)

        def prep(t):
            if t is None:
                return None
            t = t.to(torch.float32).contiguous()
            return t.cpu() if host else t.to(self.device)

        cond_emb, text_scale, obs_x0 = prep(cond_emb), prep(text_scale), prep(obs_x0)
        if obs_mask is not None:
            obs_mask = obs_mask.to(torch.uint8).contiguous()
            obs_mask = obs_mask.cpu() if host else obs_mask.to(self.device)
        a = capi.ForwardArgs(B, _ptr(x), int(timestep), _ptr(cond_emb), int(uncond), int(cfg), _ptr(text_scale), int(host),
                             _ptr(obs_x0), _ptr(obs_mask))
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
               window_frames0: Optional[Sequence[int]] = None, global_frames: int = 0, want_window_out: bool = False):
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
        n_iter = self.num_timesteps - int(skip_timesteps)
        if num_steps:
            n_iter = min(n_iter, int(num_steps))
        plms_steps = n_iter + (self._plms_steps if resume else 0)  # iterations of the PLMS history after this call
        old_eps, n_old = None, 0
        if want_old_eps and sampler == capi.SAMPLER_PLMS:
            n_old = min(plms_steps, int(plms_order) - 1)  # the length of the reference's list after that many steps
            old_eps = torch.empty((max(n_old, 1),) + shape, dtype=torch.float32, device=dev, pin_memory=host_buffers)
        unipc = sampler == capi.SAMPLER_UNIPC
        dpm = sampler in (capi.SAMPLER_DPM_SOLVER, capi.SAMPLER_DPM_SOLVER_SDE)
        repaint = sampler == capi.SAMPLER_REPAINT
        a = capi.SampleArgs(batch, sampler, float(eta), int(skip_timesteps), int(num_steps), int(resume), _ptr(init_image), _ptr(x_T), _ptr(noise_tape),
                            int(seed) & (2 ** 64 - 1), int(sample_offset), int(rng_mode), int(aten_offset), int(aten_increment),
                            int(aten_threads), _ptr(cond_emb), int(uncond), int(cfg), _ptr(text_scale),
                            _ptr(y_mask), int(imputate), int(stop_imputation_at), _ptr(inpainted_motion),
                            _ptr(inpainting_mask), int(recon_guidance), int(stop_recguidance_at), coef_arr, _ptr(pred), _ptr(dump),
                            dump_arr, n_dump, int(host_buffers),
                            int(use_graph), _ptr(obs_x0), _ptr(obs_mask),
                            0 if sampler in (capi.SAMPLER_DDIM_REVERSE, capi.SAMPLER_UNIPC) or dpm or repaint
                            else int(plms_order),
                            _ptr(old_eps), int(dpm_order) if dpm else 0,
                            int(unipc_order) if unipc else 0, int(unipc_variant) if unipc else 0,
                            int(unipc_corrector) if unipc else 0,
                            int(repaint_jump_length) if repaint else 0, int(repaint_jump_n_sample) if repaint else 0,
                            K, f0_arr if K else None, int(global_frames), _ptr(windows))
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
                       text_scale=None, obs_x0=None, obs_mask=None) -> torch.Tensor:
        """One guided evaluation and its input-VJP (cmdi_test_input_vjp): (cfg ? 2 : 1, B, njoints, 1, nframes), the
        gradient of sum((inpainted_motion - x0_hat)^2 * inpainting_mask) w.r.t. x through each pass, cond pass first."""
        dev = lambda t, dt=torch.float32: None if t is None else t.to(self.device, dt).contiguous()  # noqa: E731
        x = dev(x)
        B = x.shape[0]
        cond_emb, text_scale, obs_x0, inpainted_motion = dev(cond_emb), dev(text_scale), dev(obs_x0), dev(inpainted_motion)
        obs_mask, inpainting_mask = dev(obs_mask, torch.uint8), dev(inpainting_mask, torch.uint8)
        grad = torch.empty((2 if cfg else 1,) + tuple(x.shape), dtype=torch.float32, device=self.device)
        a = capi.ForwardArgs(B, _ptr(x), int(timestep), _ptr(cond_emb), int(uncond), int(cfg), _ptr(text_scale), 0,
                             _ptr(obs_x0), _ptr(obs_mask))
        with torch.cuda.device(self.device):
            capi.check(self.lib.cmdi_test_input_vjp(self._h, ctypes.byref(a), _ptr(inpainted_motion), _ptr(inpainting_mask),
                                                    grad.data_ptr(), _stream_ptr(self.device)), "cmdi_test_input_vjp")
        return grad

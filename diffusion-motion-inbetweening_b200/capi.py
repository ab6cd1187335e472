"""ctypes binding of libcondmdi_b200.so (the C ABI declared in include/condmdi_b200.h).

There is no CPU fallback: if the shared library cannot be loaded every entry point raises.
"""
from __future__ import annotations

import ctypes
import os
from ctypes import POINTER, Structure, c_char_p, c_double, c_float, c_int, c_int32, c_int64, c_uint8, c_uint64, c_void_p

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("CONDMDI_B200_LIB") or os.path.join(HERE, "libcondmdi_b200.so")  # override: A/B builds

PRECISION_BF16X3 = 3
PRECISION_BF16 = 1
PRECISION_FP16 = 2  # "autocast", MDM_UNET only: the arithmetic of torch.autocast("cuda", float16) (use_fp16 checkpoints)
RNG_ENGINE, RNG_TORCH = 0, 1
SAMPLER_DDPM = 0
SAMPLER_DDIM = 1
SAMPLER_PLMS = 2
SAMPLER_DDIM_REVERSE = 3  # DDIM inversion x_t -> x_{t+1} (ddim_reverse_sample); the loop ascends from skip_timesteps
SAMPLER_DPM_SOLVER = 4  # DPM-Solver++ multistep, orders 1-3 (dpm_order)
SAMPLER_UNIPC = 5  # UniPC predictor-corrector, orders 1-3 (unipc_order, unipc_variant, unipc_corrector)
SAMPLER_DPM_SOLVER_SDE = 6  # SDE-DPM-Solver++ multistep, orders 1-2 (dpm_order); DDPM's per-step draws
SAMPLER_REPAINT = 7  # RePaint resampling around DDPM (repaint_jump_length, repaint_jump_n_sample); one draw per walk op
UNIPC_BH1, UNIPC_BH2 = 1, 2  # unipc_variant
ARCH_TRANS_ENC, ARCH_UNET = 0, 1
MOTION_ABS3D_TO_REL, MOTION_REL_TO_ABS3D, MOTION_REL_TO_JOINTS, MOTION_ABS3D_TO_JOINTS = 0, 1, 2, 3

EXPORTS = [
    "cmdi_engine_create", "cmdi_engine_destroy", "cmdi_load_weights", "cmdi_set_schedule", "cmdi_model_forward",
    "cmdi_sample", "cmdi_launch_count", "cmdi_last_error", "cmdi_version", "cmdi_test_linear", "cmdi_test_attention",
    "cmdi_test_layernorm", "cmdi_test_step", "cmdi_test_normal", "cmdi_profile_pass", "cmdi_test_layernorm_bwd", "cmdi_test_attention_bwd",
    "cmdi_test_normal_aten", "cmdi_recover_from_ric", "cmdi_test_input_vjp", "cmdi_joints_to_features", "cmdi_convert_motion",
    "cmdi_test_chain_layer", "cmdi_test_attention_hi", "cmdi_test_attention_bwd_at",
]


class ModelCfg(Structure):
    _fields_ = [("njoints", c_int32), ("nframes", c_int32), ("latent_dim", c_int32), ("ff_size", c_int32),
                ("num_layers", c_int32), ("num_heads", c_int32), ("max_batch", c_int32), ("has_text", c_int32),
                ("precision", c_int32), ("arch", c_int32), ("unet_levels", c_int32), ("unet_dim_mults", c_int32 * 4),
                ("keyframe_conditioned", c_int32)]


class TensorDesc(Structure):
    _fields_ = [("name", c_char_p), ("data", c_void_p), ("numel", c_int64), ("on_host", c_int32)]


class ForwardArgs(Structure):
    _fields_ = [("batch", c_int32), ("x", c_void_p), ("timestep", c_int32), ("cond_emb", c_void_p), ("uncond", c_int32),
                ("cfg", c_int32), ("text_scale", c_void_p), ("host_buffers", c_int32), ("obs_x0", c_void_p), ("obs_mask", c_void_p)]


class SampleArgs(Structure):
    _fields_ = [("batch", c_int32), ("sampler", c_int32), ("eta", c_float), ("skip_timesteps", c_int32), ("num_steps", c_int32), ("resume", c_int32),
                ("init_image", c_void_p), ("x_T", c_void_p), ("noise_tape", c_void_p), ("seed", c_uint64),
                ("sample_offset", c_uint64), ("rng_mode", c_int32), ("aten_offset", c_uint64), ("aten_increment", c_uint64),
                ("aten_threads", ctypes.c_uint32), ("cond_emb", c_void_p), ("uncond", c_int32), ("cfg", c_int32), ("text_scale", c_void_p),
                ("y_mask", c_void_p), ("imputate", c_int32), ("stop_imputation_at", c_int32),
                ("inpainted_motion", c_void_p), ("inpainting_mask", c_void_p), ("recon_guidance", c_int32),
                ("stop_recguidance_at", c_int32), ("recon_coef", POINTER(c_float)), ("pred_xstart_out", c_void_p),
                ("dump_xstart", c_void_p), ("dump_steps", POINTER(c_int32)), ("n_dump", c_int32),
                ("host_buffers", c_int32), ("use_graph", c_int32), ("obs_x0", c_void_p), ("obs_mask", c_void_p),
                ("plms_order", c_int32), ("plms_old_eps_out", c_void_p), ("dpm_order", c_int32),
                ("unipc_order", c_int32), ("unipc_variant", c_int32), ("unipc_corrector", c_int32),
                ("repaint_jump_length", c_int32), ("repaint_jump_n_sample", c_int32),
                ("window_count", c_int32), ("window_frames0", POINTER(c_int32)), ("global_frames", c_int32),
                ("window_out", c_void_p)]


class LibraryMissing(RuntimeError):
    pass


_lib = None


def load(build_if_missing: bool = True) -> ctypes.CDLL:
    """Load the shared library (building it with nvcc first if it is absent and a compiler is available)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH) and build_if_missing:
        try:
            from . import build as _build
            _build.build()
        except Exception as ex:  # noqa: BLE001
            raise LibraryMissing(f"libcondmdi_b200.so is missing and could not be built: {ex}") from ex
    if not os.path.exists(LIB_PATH):
        raise LibraryMissing(f"{LIB_PATH} not found: build it with `python -m condmdi_b200.build` (no CPU fallback exists)")
    lib = ctypes.CDLL(LIB_PATH)
    lib.cmdi_last_error.restype = c_char_p
    lib.cmdi_version.restype = c_char_p
    lib.cmdi_launch_count.restype = c_int64
    lib.cmdi_launch_count.argtypes = [c_void_p]
    lib.cmdi_engine_create.argtypes = [POINTER(ModelCfg), c_int, POINTER(c_void_p)]
    lib.cmdi_engine_destroy.argtypes = [c_void_p]
    lib.cmdi_load_weights.argtypes = [c_void_p, POINTER(TensorDesc), c_int]
    lib.cmdi_set_schedule.argtypes = [c_void_p, POINTER(c_double), c_int, POINTER(c_int64)]
    lib.cmdi_model_forward.argtypes = [c_void_p, POINTER(ForwardArgs), c_void_p, c_void_p]
    lib.cmdi_sample.argtypes = [c_void_p, POINTER(SampleArgs), c_void_p, c_void_p]
    lib.cmdi_test_linear.argtypes = [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int,
                                     c_int, c_void_p]
    lib.cmdi_test_attention.argtypes = [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p]
    lib.cmdi_test_attention_hi.argtypes = lib.cmdi_test_attention.argtypes
    lib.cmdi_test_layernorm.argtypes = [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_void_p]
    lib.cmdi_test_step.argtypes = [c_void_p, c_int, c_float, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                                   c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]
    lib.cmdi_test_normal.argtypes = [c_void_p, c_int, ctypes.c_longlong, c_uint64, c_uint64, c_uint64, c_void_p]
    lib.cmdi_test_normal_aten.argtypes = [c_void_p, ctypes.c_longlong, c_uint64, c_uint64, ctypes.c_uint32, c_void_p]
    ll = ctypes.c_longlong
    lib.cmdi_recover_from_ric.argtypes = [c_void_p, ll, ll, ll, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p,
                                          ll, ll, ll, ll, c_void_p]
    lib.cmdi_joints_to_features.argtypes = [c_void_p, ll, ll, c_int, c_int, c_int, c_double, c_void_p, ll, ll, ll, c_void_p]
    lib.cmdi_convert_motion.argtypes = [c_int, c_void_p, ll, ll, ll, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p, c_int,
                                        c_void_p, c_void_p, c_int, c_double, c_void_p, ll, ll, ll, c_void_p]
    lib.cmdi_profile_pass.argtypes = [c_void_p, c_int, c_int, c_int, POINTER(c_float), c_int, POINTER(c_int), c_void_p]
    lib.cmdi_test_layernorm_bwd.argtypes = [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_void_p]
    lib.cmdi_test_attention_bwd.argtypes = [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_void_p]
    lib.cmdi_test_attention_bwd_at.argtypes = [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p]
    lib.cmdi_test_chain_layer.argtypes = [POINTER(c_void_p), POINTER(c_void_p), c_int, c_int, c_float, c_void_p]
    lib.cmdi_test_input_vjp.argtypes = [c_void_p, POINTER(ForwardArgs), c_void_p, c_void_p, c_void_p, c_void_p]
    _lib = lib
    return lib


def check(rc: int, what: str = "condmdi_b200") -> None:
    if rc != 0:
        msg = load().cmdi_last_error().decode(errors="replace")
        raise RuntimeError(f"{what} failed: {msg}")

"""GPU: every refusal cmdi_sample can return on an engine with weights and a schedule loaded, one case per refusal.

Each case asserts the refusal's full text and that the refused call left the engine as it found it: a DPM-Solver++ loop
runs two steps, the refused call comes (with resume = 0 unless the refusal is about a resume), and the loop's resume call
finishes it bit for bit like the same loop without the refused call.  The refused calls go through the raw C ABI, since
Engine.sample refuses some of these inputs before the library sees them.
"""
import ctypes
from ctypes import byref

import pytest
import torch

import condmdi_b200 as C
from oracle import condmdi_oracle as O

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
B, D, L = 2, 263, 196
SHAPE = (B, D, 1, L)
K = C.capi
DPM, SDE, PLMS, UNIPC, REPAINT, REV = (K.SAMPLER_DPM_SOLVER, K.SAMPLER_DPM_SOLVER_SDE, K.SAMPLER_PLMS, K.SAMPLER_UNIPC,
                                       K.SAMPLER_REPAINT, K.SAMPLER_DDIM_REVERSE)
SKIP = 6  # ddim10: steps 3, 2, 1, 0
UNET_PRECISION = ("reconstruction guidance (the denoiser's input-VJP) is implemented for the transformer denoiser and, at "
                  "CMDI_PRECISION_FP16 (condmdi_b200.PRECISION_FP16), for MDM_UNET")


def _frames(*f):
    return (ctypes.c_int32 * len(f))(*f)


def _floats(n):
    return (ctypes.c_float * n)(*([0.5] * n))


# (case id, fields of the refused call over a valid DPM-Solver++ call of order 2, its refusal)
WIN = dict(window_count=2, window_frames0=_frames(0, 98), global_frames=294)  # a valid placement of two windows
JOINT = dict(joint_guidance=1, joint_coef=_floats(10), joint_target="x", joint_mask="x", joint_mean="x", joint_std="x")
TRANSFORMER = [
    ("null_out", dict(out=None), "null argument"),
    ("batch", dict(batch=3), "batch 3 outside [1, max_batch=2]"),
    ("unknown_sampler", dict(sampler=8), "unknown sampler 8"),
    ("negative_sampler", dict(sampler=-1), "unknown sampler -1"),
    ("dpm_order_elsewhere", dict(sampler=PLMS, plms_order=2),
     "dpm_order is a CMDI_SAMPLER_DPM_SOLVER / CMDI_SAMPLER_DPM_SOLVER_SDE field: it must be 0 for sampler 2"),
    ("unipc_field_elsewhere", dict(unipc_variant=1), "unipc_variant is a CMDI_SAMPLER_UNIPC field: it must be 0 for sampler 4"),
    ("repaint_field_elsewhere", dict(repaint_jump_n_sample=2),
     "repaint_jump_n_sample is a CMDI_SAMPLER_REPAINT field: it must be 0 for sampler 4"),
    ("dpm_eta", dict(eta=0.5), "CMDI_SAMPLER_DPM_SOLVER: eta (DPM-Solver++ is deterministic after x_T: eta must be 0) must be unset"),
    ("unipc_eta", dict(sampler=UNIPC, dpm_order=0, unipc_order=2, unipc_variant=2, eta=0.5),
     "CMDI_SAMPLER_UNIPC: eta (UniPC is deterministic after x_T: eta must be 0) must be unset"),
    ("sde_eta", dict(sampler=SDE, eta=0.5),
     "CMDI_SAMPLER_DPM_SOLVER_SDE: eta (the SDE solver's noise is fixed by the schedule: eta must be 0) must be unset"),
    ("repaint_eta", dict(sampler=REPAINT, dpm_order=0, repaint_jump_length=1, repaint_jump_n_sample=2, eta=0.5),
     "CMDI_SAMPLER_REPAINT: eta (RePaint denoises with p_sample: eta must be 0) must be unset"),
    ("reverse_eta", dict(sampler=REV, dpm_order=0, eta=0.5),
     "CMDI_SAMPLER_DDIM_REVERSE: eta (the reverse ODE is deterministic: eta must be 0) must be unset"),
    ("dpm_noise_tape", dict(noise_tape="tape"), "CMDI_SAMPLER_DPM_SOLVER: noise_tape (no noise is drawn after x_T) must be unset"),
    ("reverse_noise_tape", dict(sampler=REV, dpm_order=0, noise_tape="tape"), "CMDI_SAMPLER_DDIM_REVERSE: noise_tape must be unset"),
    ("reverse_init_image", dict(sampler=REV, dpm_order=0, init_image="x"), "CMDI_SAMPLER_DDIM_REVERSE: init_image must be unset"),
    ("dump_xstart", dict(dump_xstart="x"), "CMDI_SAMPLER_DPM_SOLVER: dump_xstart must be unset"),
    ("plms_order", dict(plms_order=2), "CMDI_SAMPLER_DPM_SOLVER: plms_order must be unset"),
    ("plms_old_eps_out", dict(plms_old_eps_out="x"), "CMDI_SAMPLER_DPM_SOLVER: plms_old_eps_out must be unset"),
    ("resume_init_image", dict(resume=1, init_image="x"),
     "CMDI_SAMPLER_DPM_SOLVER: init_image (a resume call continues the running state) must be unset"),
    ("dpm_order", dict(dpm_order=4), "dpm_order 4 outside [1, 3]"),
    ("sde_order", dict(sampler=SDE, dpm_order=3), "dpm_order 3 outside [1, 2] (CMDI_SAMPLER_DPM_SOLVER_SDE)"),
    ("unipc_order", dict(sampler=UNIPC, dpm_order=0, unipc_order=4, unipc_variant=2), "unipc_order 4 outside [1, 3]"),
    ("plms_order_bounds", dict(sampler=PLMS, dpm_order=0, plms_order=5), "plms_order 5 outside [2, 4]"),
    ("repaint_jump_length", dict(sampler=REPAINT, dpm_order=0, repaint_jump_n_sample=2), "repaint_jump_length 0 must be >= 1"),
    ("repaint_jump_n_sample", dict(sampler=REPAINT, dpm_order=0, repaint_jump_length=1), "repaint_jump_n_sample 0 must be >= 1"),
    ("unipc_variant", dict(sampler=UNIPC, dpm_order=0, unipc_order=2, unipc_variant=3),
     "unipc_variant 3 is neither CMDI_UNIPC_BH1 (1) nor CMDI_UNIPC_BH2 (2)"),
    ("unipc_corrector", dict(sampler=UNIPC, dpm_order=0, unipc_order=2, unipc_variant=2, unipc_corrector=2),
     "unipc_corrector 2 is neither 0 nor 1"),
    ("reverse_x_T", dict(sampler=REV, dpm_order=0, x_T=None), "CMDI_SAMPLER_DDIM_REVERSE needs x_T, the state to invert"),
    ("window_field", dict(global_frames=294), "global_frames is a window field: it must be unset when window_count is 0"),
    ("window_count", dict(window_count=-1), "window_count -1 must be >= 0"),
    ("window_sampler", dict(WIN, sampler=REPAINT, dpm_order=0, repaint_jump_length=1, repaint_jump_n_sample=2),
     "window_count: sampler 7 (DDIM inversion / RePaint) does not run on overlapping windows"),
    ("window_batch", dict(WIN, window_count=3, window_frames0=_frames(0, 49, 98)),
     "window_count 3 does not divide batch 2 (row s * K + k is window k of global sample s)"),
    ("window_frames0", dict(WIN, window_frames0=None), "window_frames0 is required when window_count is set"),
    ("global_frames", dict(WIN, global_frames=100), "global_frames 100 is shorter than a window (196 frames)"),
    ("window_placement", dict(WIN, window_frames0=_frames(0, 97)),
     "window_frames0[1] = 97: the first frames must start at 0, ascend strictly with no gap between windows of 196 "
     "frames, and end at global_frames - 196 = 98"),
    ("window_old_eps", dict(WIN, sampler=PLMS, dpm_order=0, plms_order=2, plms_old_eps_out="x"),
     "plms_old_eps_out must be NULL on overlapping windows"),
    ("plms_tape", dict(sampler=PLMS, dpm_order=0, plms_order=2, noise_tape="tape"),
     "PLMS draws no per-step noise and has no dump_steps: noise_tape and dump_xstart must be NULL"),
    ("cfg", dict(cfg=1, text_scale="scale"), "cfg sampling needs cond_emb and text_scale (cfg_sampler.py:26, :35)"),
    ("keyframe_cfg_model", dict(keyframe_scale="scale"), "keyframe_scale (keyframe CFG) needs a keyframe-conditioned MDM_UNET"),
    ("imputate", dict(imputate=1, inpainted_motion="x"),
     "imputate / reconstruction_guidance need inpainted_motion and inpainting_mask (editing_util.py:330, :343)"),
    ("recon_coef", dict(recon_guidance=1, inpainted_motion="x", inpainting_mask="mask"), "reconstruction_guidance needs recon_coef"),
    ("joint_fields", dict(JOINT, joint_std=None), "joint_guidance needs joint_coef, joint_target, joint_mask, joint_mean and joint_std"),
    ("foot_contact_fields", dict(foot_contact=1, joint_mean="x", joint_std="x"),
     "foot_contact needs foot_contact_coef, joint_mean and joint_std"),
    ("joint_windows", dict(JOINT, **WIN),
     "joint-position guidance does not run on overlapping windows (each window's root starts at its own origin)"),
    ("skip_timesteps", dict(skip_timesteps=10), "skip_timesteps 10 outside [0, 10)"),
    ("resume", dict(resume=1), "DPM-Solver++ resume at step 3 does not continue the running history"),
    ("repaint_walk", dict(sampler=REPAINT, dpm_order=0, repaint_jump_length=1, repaint_jump_n_sample=50_000_000),
     "repaint_jump_length 1 and repaint_jump_n_sample 50000000 give a walk of 299999998 ops (at most 2^28)"),
    ("rng_torch", dict(rng_mode=K.RNG_TORCH), "rng_mode=CMDI_RNG_TORCH needs aten_threads > 0 and aten_offset / aten_increment "
     "multiples of 4"),
    ("rng_mode", dict(rng_mode=2), "unknown rng_mode 2"),
    ("has_text", dict(cond_emb="cond"), "cond_emb given but the engine was created with has_text = 0"),
    ("host_noise_tape", dict(sampler=SDE, host_buffers=1, x_T=None, noise_tape="tape"),
     "noise_tape must be a device pointer (it is a test aid; stage it once outside the call)"),
]
# a keyframe-conditioned MDM_UNET at bf16x3 without text; its valid call carries obs_x0 / obs_mask
UNET = [
    ("keyframe_cfg_keyframes", dict(keyframe_scale="scale", obs_x0=None, obs_mask=None),
     "keyframe_scale (keyframe CFG) needs obs_x0 and obs_mask"),
    ("keyframe_cfg_passes", dict(keyframe_scale="scale", cfg=1, cond_emb="cond", text_scale="scale"),
     "keyframe CFG runs 3 passes of batch 2: 6 sequences, more than the 2 * max_batch = 4 the engine holds"),
    ("recon_precision", dict(recon_guidance=1, recon_coef=_floats(10), inpainted_motion="x", inpainting_mask="mask"),
     UNET_PRECISION),
    ("joint_precision", dict(JOINT), UNET_PRECISION),
    ("obs_pair", dict(obs_mask=None), "with spatial conditioning, both obs_x0 and obs_mask must be provided (mdm_unet.py:775)"),
    ("obs_needed", dict(obs_x0=None, obs_mask=None), "a keyframe-conditioned UNet needs obs_x0 and obs_mask"),
]


@pytest.fixture(scope="module")
def data():
    g = torch.Generator().manual_seed(0)
    t = dict(x=torch.randn(SHAPE, generator=g), tape=torch.randn((4,) + SHAPE, generator=g), scale=torch.full((B,), 2.5),
             cond=torch.randn(B, 512, generator=g), mask=(torch.rand(SHAPE, generator=g) < 0.3).to(torch.uint8))
    return {k: v.to(DEV).contiguous() for k, v in t.items()}


def _engine(m, sd):
    assert not any(m.load_state_dict(sd, strict=False))
    eng = m.to(DEV).engine_for(torch.device(DEV), max_batch=B)
    d = C.create_gaussian_diffusion(timestep_respacing="ddim10")
    eng.set_schedule(d.betas, d.timestep_map)
    return eng


@pytest.fixture(scope="module")
def transformer():
    return _engine(C.MDM(num_layers=2), O.random_state_dict(seed=3, layers=2)), {}


@pytest.fixture(scope="module")
def unet(data):
    return _engine(C.MDM_UNET(keyframe_conditioned=True), O.random_unet_state_dict(seed=11)), \
        dict(obs_x0=data["x"], obs_mask=data["mask"])


def _loop(eng, data, kw, between=None):
    """A four-step DPM-Solver++ loop in two calls of two steps; `between()` runs between them."""
    first = eng.sample(B, sampler=DPM, skip_timesteps=SKIP, num_steps=2, x_T=data["x"], dpm_order=2, **kw)["sample"]
    if between:
        between()
    return eng.sample(B, sampler=DPM, skip_timesteps=SKIP + 2, resume=True, x_T=first, dpm_order=2, **kw)["sample"]


def _refuse(eng, data, kw, fields, msg):
    want = _loop(eng, data, kw)
    args = dict(batch=B, sampler=DPM, skip_timesteps=SKIP, x_T="x", dpm_order=2, **kw)
    args.update(fields)
    out = args.pop("out", "x")
    # strings name the test tensors; any other value is the field's own
    args = {k: (data[v].data_ptr() if isinstance(v, str) else v.data_ptr() if isinstance(v, torch.Tensor) else v)
            for k, v in args.items()}
    a = K.SampleArgs(**args)
    res = torch.empty(SHAPE, device=DEV)

    def refused_call():
        rc = eng.lib.cmdi_sample(eng._h, byref(a), res.data_ptr() if out else None, None)
        assert rc != 0
        assert eng.lib.cmdi_last_error().decode() == msg

    torch.cuda.synchronize()
    got = _loop(eng, data, kw, refused_call)
    assert torch.equal(got, want)


@pytest.mark.parametrize("fields,msg", [c[1:] for c in TRANSFORMER], ids=[c[0] for c in TRANSFORMER])
def test_transformer_refusal_leaves_engine_untouched(transformer, data, fields, msg):
    eng, kw = transformer
    _refuse(eng, data, kw, fields, msg)


@pytest.mark.parametrize("fields,msg", [c[1:] for c in UNET], ids=[c[0] for c in UNET])
def test_unet_refusal_leaves_engine_untouched(unet, data, fields, msg):
    eng, kw = unet
    _refuse(eng, data, kw, fields, msg)


def test_valid_call_is_accepted(transformer, unet, data):
    """The call every case starts from is accepted, so each case's refusal is its own field's."""
    for eng, kw in (transformer, unet):
        a = K.SampleArgs(batch=B, sampler=DPM, skip_timesteps=SKIP, x_T=data["x"].data_ptr(), dpm_order=2,
                         **{k: v.data_ptr() for k, v in kw.items()})
        res = torch.empty(SHAPE, device=DEV)
        assert eng.lib.cmdi_sample(eng._h, byref(a), res.data_ptr(), None) == 0, eng.lib.cmdi_last_error()
        torch.cuda.synchronize()

"""TEST INFRASTRUCTURE -- shows that the restatement's p_mean_variance with reconstruction guidance on the keyframe-conditioned
MDM_UNET equals the UNMODIFIED reference's, in fp32 and under autocast, and writes tests/golden/unet_guidance.* from the
reference's outputs.

Run in the build container (needs the reference tree):   python -m oracle.make_golden_unet_guidance

The reference computes the guidance gradient of a use_fp16 checkpoint as `torch.autograd.grad` after a forward inside
`amp.autocast(enabled=conf.fp16)` (gaussian_diffusion.py:388-425).  Here the module-level `amp` of gaussian_diffusion is
replaced by a shim mapping `autocast(enabled)` to `torch.autocast("cpu", float16, enabled=...)` (a harness shim, no source
edit), conf.fp16 is set, and the restatement's p_mean_variance runs with its model call (condmdi_oracle._model) wrapped
in the same context (`model_calls_under`, the same kind of shim) -- around the model call only, the guidance gradient
outside it.  The two must agree bit for bit, which pins where autocast's casts fall in the forward AND which
dtypes autograd's backward sees (DESIGN.md section 2); what CUDA computes comes from the GPU tests
(tests/test_gpu_unet_guidance.py).  Cases, on the xl geometry (configs/model.py `motion_unet_adagn_xl`, keyframe input
conditioning, text):
  cfg.t500 / cfg.t30   ClassifierFreeSampleModel (scale 2.5), imputation, w = 20, default schedule
  plain.t500           the model without the CFG wrapper, no imputation, exponential schedule
"""
from __future__ import annotations

import contextlib
import os
import sys
import types

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import condmdi_oracle as O  # noqa: E402
from oracle import reference_harness as RH  # noqa: E402
from oracle.golden_io import save_golden  # noqa: E402
from oracle.make_golden import GOLDEN  # noqa: E402


def cpu_autocast():
    return torch.autocast("cpu", dtype=torch.float16)


def cases():
    """(name, cfg, t, imputate, schedule) of every checked evaluation."""
    return [("cfg.t500", True, 500, True, None), ("cfg.t30", True, 30, True, None), ("plain.t500", False, 500, False, "exponential")]


def inputs():
    gi = O.golden_inputs()
    return {k: gi[k] for k in ("x", "cond", "x_obs", "text_scale", "y_mask", "lengths", "kf_mask")}


def conditioning(gi, cfg, imputate, schedule):
    return O.Conditioning(cond_emb=gi["cond"], cfg=cfg, text_scale=gi["text_scale"], y_mask=gi["y_mask"], imputate=imputate,
                          stop_imputation_at=0, inpainted_motion=gi["x_obs"], inpainting_mask=gi["kf_mask"],
                          reconstruction_guidance=True, reconstruction_weight=20.0, gradient_schedule=schedule,
                          stop_recguidance_at=0, obs_x0=gi["x_obs"], obs_mask=gi["kf_mask"])


@contextlib.contextmanager
def model_calls_under(context):
    """Run every model call of condmdi_oracle.p_mean_variance (its module-level `_model`) inside `context()`, as the
    reference wraps `model(...)` in `amp.autocast` (gaussian_diffusion.py:388-389); context None: unchanged."""
    plain = O._model
    if context is not None:
        def wrapped(*args):
            with context():
                return plain(*args)
        O._model = wrapped
    try:
        yield
    finally:
        O._model = plain


def run_oracle(sd, gi, cfg, t, imputate, schedule, autocast):
    c = conditioning(gi, cfg, imputate, schedule)
    with model_calls_under(cpu_autocast if autocast else None):
        out = O.p_mean_variance(sd, O.make_tables(""), gi["x"], torch.tensor([t, t]), c)
    return out["pred_xstart"].detach(), out["mean"].detach()


def run_reference(ref, diff, m, gi, cfg, t, imputate, schedule, autocast):
    y = {"text": ["a", "b"], "mask": gi["y_mask"], "lengths": gi["lengths"], "inpainted_motion": gi["x_obs"],
         "inpainting_mask": gi["kf_mask"], "reconstruction_guidance": True, "reconstruction_weight": 20.0,
         "gradient_schedule": schedule, "diffusion_steps": 1000, "stop_recguidance_at": 0}
    if cfg:
        y["text_scale"] = gi["text_scale"]
    if imputate:
        y.update(imputate=1, stop_imputation_at=0, replacement_distribution="conditional")
    model = ref.cfg_sampler.ClassifierFreeSampleModel(m) if cfg else m
    diff.conf.fp16 = autocast
    out = diff.p_mean_variance(model, gi["x"], torch.tensor([t, t]), clip_denoised=False,
                               model_kwargs={"y": y, "obs_x0": gi["x_obs"], "obs_mask": gi["kf_mask"]})
    return out["pred_xstart"].detach(), out["mean"].detach()


def golden_unet_guidance():
    ref = RH.import_reference()
    gd = ref.gd
    saved_amp = gd.amp
    gd.amp = types.SimpleNamespace(autocast=lambda enabled=True: torch.autocast("cpu", dtype=torch.float16, enabled=enabled))
    gi = inputs()
    sd = O.random_unet_state_dict(seed=11, text=True)
    m = RH.build_reference_unet(text=True)
    missing, unexpected = m.load_state_dict(sd, strict=False)
    assert not missing and not unexpected, (missing, unexpected)
    m._synthetic_text_emb = gi["cond"]
    diff = RH.build_reference_diffusion("")
    out = {}
    try:
        for name, cfg, t, imputate, schedule in cases():
            f32 = None
            for mode in ("fp32", "fp16"):
                ac = mode == "fp16"
                r = run_reference(ref, diff, m, gi, cfg, t, imputate, schedule, ac)
                o = run_oracle(sd, gi, cfg, t, imputate, schedule, ac)
                exact = all(torch.equal(a, b) for a, b in zip(r, o))
                err = max((a - b).abs().max().item() for a, b in zip(r, o))
                if f32 is None:
                    f32 = r
                gap = (r[0] - f32[0]).abs().max().item()
                print(f"  {mode} {name:10s} reference == restatement: {exact} (max diff {err:.3e})   "
                      f"max |pred_xstart - fp32's| = {gap:.3e}")
                assert exact, f"{mode} {name}: the restatement differs from the reference by {err:.3e}"
                out[f"{mode}.{name}.pred_xstart"] = r[0].numpy()
                out[f"{mode}.{name}.mean"] = r[1].numpy()
    finally:
        gd.amp = saved_amp
    save_golden(GOLDEN, "unet_guidance", **out)


def main():
    if not RH.available():
        raise SystemExit("the reference tree is required to (re)generate golden vectors")
    os.makedirs(GOLDEN, exist_ok=True)
    torch.set_num_threads(os.cpu_count() or 1)
    golden_unet_guidance()
    for f in sorted(os.listdir(GOLDEN)):
        if f.startswith("unet_guidance."):
            print(f, os.path.getsize(os.path.join(GOLDEN, f)) // 1024, "KiB")


if __name__ == "__main__":
    main()

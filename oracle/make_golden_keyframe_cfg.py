"""TEST INFRASTRUCTURE -- shows that oracle/keyframe_cfg_oracle.py equals keyframe classifier-free guidance composed
around the UNMODIFIED reference's MDM_UNET and sampling loops, and writes tests/golden/keyframe_cfg.* from the
reference's outputs.

Run in the build container (needs the reference tree):   python -m oracle.make_golden_keyframe_cfg

The reference has no keyframe CFG (its scripts raise NotImplementedError or ignore y['keyframe_scale']), so the guided
model is composed here by `KeyframeCFG`, a small nn.Module that calls the reference's MDM_UNET three times (two for a
no_cond model) with the reference's own conditioning conventions (y['uncond'], obs_x0 / obs_mask) and combines the
outputs in the documented order.  The reference's p_sample_loop / ddim_sample_loop / plms_sample_loop drive it.  Cases,
on the xl geometry (configs/model.py `motion_unet_adagn_xl`, keyframe input conditioning, text), per-sample w_k != w_t:
  fwd.t500 / fwd.t30       one forward
  ddpm / ddim / plms       the last two steps of a ddim50 loop with imputation
  guided.fp32 / .fp16      p_mean_variance with reconstruction guidance (w = 20) at t = 500, in fp32 and under CPU fp16
                           autocast (the shim of make_golden_unet_guidance)
  nocond.t500              the two-pass form of a no_cond keyframe model
"""
from __future__ import annotations

import os
import sys
import types

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import condmdi_oracle as O  # noqa: E402
from oracle import keyframe_cfg_oracle as K  # noqa: E402
from oracle import plms_oracle as P  # noqa: E402
from oracle.golden_io import save_golden  # noqa: E402
from oracle.make_golden import GOLDEN  # noqa: E402
from oracle.make_golden_unet_guidance import cpu_autocast, model_calls_under  # noqa: E402

SKIP = 48  # the last two steps of ddim50


class KeyframeCFG(torch.nn.Module):
    """Keyframe classifier-free guidance around a reference MDM_UNET (no reference source copied)."""

    def __init__(self, model):
        super().__init__()
        self.model = model

    def forward(self, x, timesteps, y=None, obs_x0=None, obs_mask=None, **kwargs):
        y_uncond = dict(y)
        y_uncond["uncond"] = True
        wk = y["keyframe_scale"].view(-1, 1, 1, 1)
        c = self.model(x, timesteps, y, obs_x0, obs_mask, **kwargs)
        n = self.model(x, timesteps, y_uncond, obs_x0, torch.zeros_like(obs_mask), **kwargs)
        if "text" not in self.model.cond_mode:
            return n + wk * (c - n)
        u = self.model(x, timesteps, y_uncond, obs_x0, obs_mask, **kwargs)
        a = n + wk * (u - n)
        return a + y["text_scale"].view(-1, 1, 1, 1) * (c - u)


def inputs():
    gi = O.golden_inputs()
    gi["keyframe_scale"] = torch.tensor([1.75, 0.6])  # != text_scale
    return gi


def y_of(gi, text=True, imputate=False, guided=False):
    y = {"mask": gi["y_mask"], "lengths": gi["lengths"], "keyframe_scale": gi["keyframe_scale"]}
    if text:
        y.update(text=["a", "b"], text_scale=gi["text_scale"])
    if imputate:
        y.update(imputate=1, stop_imputation_at=0, replacement_distribution="conditional", inpainted_motion=gi["x_obs"],
                 inpainting_mask=gi["kf_mask"])
    if guided:
        y.update(reconstruction_guidance=True, reconstruction_weight=20.0, gradient_schedule=None, diffusion_steps=1000,
                 stop_recguidance_at=0, inpainted_motion=gi["x_obs"], inpainting_mask=gi["kf_mask"])
    return y


def cond_of(gi, text=True, imputate=False, guided=False):
    kw = dict(cond_emb=gi["cond"] if text else None, cfg=text, text_scale=gi["text_scale"], y_mask=gi["y_mask"],
              obs_x0=gi["x_obs"], obs_mask=gi["kf_mask"], inpainted_motion=gi["x_obs"], inpainting_mask=gi["kf_mask"])
    if imputate:
        kw.update(imputate=True, stop_imputation_at=0)
    if guided:
        kw.update(reconstruction_guidance=True, reconstruction_weight=20.0, stop_recguidance_at=0)
    return O.Conditioning(**kw)


CASES = ["fwd.t500", "fwd.t30", "ddpm", "ddim", "plms", "guided.fp32", "nocond.t500"]


def weights():
    return O.random_unet_state_dict(seed=11, text=True), O.random_unet_state_dict(seed=12)


def restated_outputs(names=CASES):
    """The restatement's output of every case in `names` (fp32, CPU)."""
    gi = inputs()
    sd, sdn = weights()
    tab = O.make_tables("ddim50")
    shape = tuple(gi["x"].shape)
    out = {}
    with K.keyframe_cfg(gi["keyframe_scale"]):
        for name in names:
            if name.startswith("fwd."):
                t = int(name[5:])
                with torch.no_grad():
                    out[name] = O._model(sd, gi["x"], torch.tensor([t, t]), cond_of(gi))
            elif name == "nocond.t500":
                with torch.no_grad():
                    out[name] = O._model(sdn, gi["x"], torch.tensor([500, 500]), cond_of(gi, text=False))
            elif name in ("ddpm", "ddim"):
                out[name] = O.sample_loop(sd, tab, shape, cond_of(gi, imputate=True), gi["tape"][:3], sampler=name,
                                          skip_timesteps=SKIP, init_image=gi["x_obs"])
            elif name == "plms":
                out[name] = P.plms_sample_loop(sd, tab, shape, cond_of(gi, imputate=True), gi["tape"][:1],
                                               skip_timesteps=SKIP, init_image=gi["x_obs"])
            elif name.startswith("guided."):
                with model_calls_under(cpu_autocast if name.endswith("fp16") else None):
                    out[name] = O.p_mean_variance(sd, O.make_tables(""), gi["x"], torch.tensor([500, 500]),
                                                  cond_of(gi, guided=True))["pred_xstart"].detach()
    return out


def reference_outputs(ref, RH):
    gi = inputs()
    shape = tuple(gi["x"].shape)
    m = RH.build_reference_unet(text=True)
    mn = RH.build_reference_unet()
    sd, sdn = weights()
    for mod, w in ((m, sd), (mn, sdn)):
        missing, unexpected = mod.load_state_dict(w, strict=False)
        assert not missing and not unexpected, (missing, unexpected)
    m._synthetic_text_emb = gi["cond"]
    kw = {"obs_x0": gi["x_obs"], "obs_mask": gi["kf_mask"]}
    d50 = RH.build_reference_diffusion("ddim50")
    out = {}
    with torch.no_grad():
        for t in (500, 30):
            out[f"fwd.t{t}"] = KeyframeCFG(m)(gi["x"], torch.tensor([t, t]), y_of(gi), **kw)
        out["nocond.t500"] = KeyframeCFG(mn)(gi["x"], torch.tensor([500, 500]), y_of(gi, text=False), **kw)
    for name, loop in (("ddpm", d50.p_sample_loop), ("ddim", d50.ddim_sample_loop), ("plms", d50.plms_sample_loop)):
        n_draws = 1 if name == "plms" else 3
        with RH.noise_tape(gi["tape"][:n_draws]):
            out[name] = loop(KeyframeCFG(m), shape, clip_denoised=False, model_kwargs={"y": y_of(gi, imputate=True), **kw},
                             skip_timesteps=SKIP, init_image=gi["x_obs"], device="cpu", progress=False)
    gd = ref.gd
    saved_amp = gd.amp
    gd.amp = types.SimpleNamespace(autocast=lambda enabled=True: torch.autocast("cpu", dtype=torch.float16, enabled=enabled))
    d = RH.build_reference_diffusion("")
    try:
        for mode in ("fp32", "fp16"):
            d.conf.fp16 = mode == "fp16"
            out[f"guided.{mode}"] = d.p_mean_variance(KeyframeCFG(m), gi["x"], torch.tensor([500, 500]), clip_denoised=False,
                                                      model_kwargs={"y": y_of(gi, guided=True), **kw})["pred_xstart"].detach()
    finally:
        gd.amp = saved_amp
    return out


def main():
    from oracle import reference_harness as RH
    if not RH.available():
        raise SystemExit("the reference tree is required to (re)generate golden vectors")
    os.makedirs(GOLDEN, exist_ok=True)
    torch.set_num_threads(os.cpu_count() or 1)
    ref = RH.import_reference()
    want = reference_outputs(ref, RH)
    got = restated_outputs(CASES + ["guided.fp16"])
    arrays = {}
    for name, r in want.items():
        exact = torch.equal(r, got[name])
        print(f"  {name:12s} reference == restatement: {exact} (max diff {(r - got[name]).abs().max().item():.3e})")
        assert exact, name
        arrays[f"{name}.ref"] = r.numpy()
    save_golden(GOLDEN, "keyframe_cfg", **arrays)


if __name__ == "__main__":
    main()

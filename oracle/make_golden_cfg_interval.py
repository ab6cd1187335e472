"""TEST INFRASTRUCTURE -- shows that oracle/cfg_interval_oracle.py equals classifier-free guidance limited to an interval
of steps composed around the UNMODIFIED reference's models and sampling loops, and writes tests/golden/cfg_interval.*
from the reference's outputs.

Run in the build container (needs the reference tree):   python -m oracle.make_golden_cfg_interval

The reference has no CFG interval, so it is composed here by `IntervalCFG`, a small nn.Module that calls the reference's
own ClassifierFreeSampleModel (or the keyframe-CFG composition of make_golden_keyframe_cfg) at the steps inside the
interval and the inner MDM / MDM_UNET alone at the others.  It receives the original timestep from the reference's
_WrappedModel and maps it back to the step index through the diffusion's timestep_map.  The reference's p_sample_loop /
ddim_sample_loop / plms_sample_loop drive it over the last STEPS steps of ddim50 (t = 5 .. 0), with per-sample text
scales:
  tf.ddpm / tf.ddim / tf.plms   transformer, text CFG, interval [2, 4] (PLMS's first step evaluates t = 5 outside it
                                and t = 4 inside it)
  unet.ddim                     MDM_UNET xl with keyframe input, text CFG and imputation, interval [2, 4]
  kfcfg.plms                    MDM_UNET xl, keyframe CFG with text CFG and imputation, interval [2, 4]
  tf.guided.ddpm                transformer, text CFG, imputation and reconstruction guidance (w = 20) stopping at
                                t = 3, interval [1, 4]: the guidance and interval boundaries differ
"""
from __future__ import annotations

import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import cfg_interval_oracle as CI  # noqa: E402
from oracle import condmdi_oracle as O  # noqa: E402
from oracle import keyframe_cfg_oracle as K  # noqa: E402
from oracle import plms_oracle as P  # noqa: E402
from oracle.golden_io import save_golden  # noqa: E402
from oracle.make_golden import GOLDEN  # noqa: E402

STEPS = 6
SKIP = 50 - STEPS  # the last STEPS steps of ddim50
# case -> (model, sampler, interval (stop_cfg_at, start_cfg_at), imputation, stop_recguidance_at or None)
CASES = {
    "tf.ddpm": ("tf", "ddpm", (2, 4), False, None),
    "tf.ddim": ("tf", "ddim", (2, 4), False, None),
    "tf.plms": ("tf", "plms", (2, 4), False, None),
    "unet.ddim": ("unet", "ddim", (2, 4), True, None),
    "kfcfg.plms": ("kfcfg", "plms", (2, 4), True, None),
    "tf.guided.ddpm": ("tf", "ddpm", (1, 4), True, 3),
}


class IntervalCFG(torch.nn.Module):
    """`guided` at the steps stop <= t <= start, `inner` at the others (no reference source copied)."""

    def __init__(self, guided, inner, timestep_map, stop, start):
        super().__init__()
        self.guided, self.inner = guided, inner
        self.step_of = {int(m): i for i, m in enumerate(timestep_map)}
        self.stop, self.start = stop, start

    def forward(self, x, timesteps, y=None, **kwargs):
        steps = {self.step_of[int(v)] for v in timesteps.reshape(-1).tolist()}
        assert len(steps) == 1
        m = self.guided if CI.active(steps.pop(), self.stop, self.start) else self.inner
        return m(x, timesteps, y=y, **kwargs)


def inputs():
    gi = O.golden_inputs()
    gi["keyframe_scale"] = torch.tensor([1.75, 0.6])
    return gi


def weights():
    return O.random_state_dict(seed=7, text=True), O.random_unet_state_dict(seed=11, text=True)


def y_of(gi, kf, imputate, stop_rg):
    y = {"mask": gi["y_mask"], "lengths": gi["lengths"], "text": ["a", "b"], "text_scale": gi["text_scale"]}
    if kf:
        y["keyframe_scale"] = gi["keyframe_scale"]
    if imputate:
        y.update(imputate=1, stop_imputation_at=0, replacement_distribution="conditional", inpainted_motion=gi["x_obs"],
                 inpainting_mask=gi["kf_mask"])
    if stop_rg is not None:
        y.update(reconstruction_guidance=True, reconstruction_weight=20.0, gradient_schedule=None, diffusion_steps=1000,
                 stop_recguidance_at=stop_rg, inpainted_motion=gi["x_obs"], inpainting_mask=gi["kf_mask"])
    return y


def cond_of(gi, unet, imputate, stop_rg):
    kw = dict(cond_emb=gi["cond"], cfg=True, text_scale=gi["text_scale"], y_mask=gi["y_mask"], inpainted_motion=gi["x_obs"],
              inpainting_mask=gi["kf_mask"])
    if unet:
        kw.update(obs_x0=gi["x_obs"], obs_mask=gi["kf_mask"])
    if imputate:
        kw.update(imputate=True, stop_imputation_at=0)
    if stop_rg is not None:
        kw.update(reconstruction_guidance=True, reconstruction_weight=20.0, stop_recguidance_at=stop_rg)
    return O.Conditioning(**kw)


def n_draws(sampler):
    return 1 if sampler == "plms" else STEPS + 1


def restated_outputs(names=tuple(CASES)):
    """The restatement's final sample of every case in `names` (fp32, CPU)."""
    gi = inputs()
    sdt, sdu = weights()
    tab = O.make_tables("ddim50")
    shape = tuple(gi["x"].shape)
    out = {}
    for name in names:
        arch, sampler, (stop, start), imputate, stop_rg = CASES[name]
        sd = sdt if arch == "tf" else sdu
        c = cond_of(gi, arch != "tf", imputate, stop_rg)
        init = gi["x_obs"] if imputate else None
        tape = gi["tape"][:n_draws(sampler)]
        kf = K.keyframe_cfg(gi["keyframe_scale"]) if arch == "kfcfg" else torch.no_grad()
        with kf, CI.cfg_interval(tab, stop, start):
            if sampler == "plms":
                out[name] = P.plms_sample_loop(sd, tab, shape, c, tape, skip_timesteps=SKIP, init_image=init)
            else:
                out[name] = O.sample_loop(sd, tab, shape, c, tape, sampler=sampler, skip_timesteps=SKIP, init_image=init)
    return out


def reference_outputs(ref, RH):
    from oracle.make_golden import ref_model_with
    from oracle.make_golden_keyframe_cfg import KeyframeCFG
    gi = inputs()
    shape = tuple(gi["x"].shape)
    sdt, sdu = weights()
    mt = ref_model_with(sdt, text=True)
    mt._synthetic_text_emb = gi["cond"]
    mu = RH.build_reference_unet(text=True)
    missing, unexpected = mu.load_state_dict(sdu, strict=False)
    assert not missing and not unexpected, (missing, unexpected)
    mu._synthetic_text_emb = gi["cond"]
    d50 = RH.build_reference_diffusion("ddim50")
    loops = {"ddpm": d50.p_sample_loop, "ddim": d50.ddim_sample_loop, "plms": d50.plms_sample_loop}
    out = {}
    for name, (arch, sampler, (stop, start), imputate, stop_rg) in CASES.items():
        inner = mt if arch == "tf" else mu
        guided = KeyframeCFG(mu) if arch == "kfcfg" else ref.cfg_sampler.ClassifierFreeSampleModel(inner)
        model = IntervalCFG(guided, inner, d50.timestep_map, stop, start)
        kw = {"y": y_of(gi, arch == "kfcfg", imputate, stop_rg)}
        if arch != "tf":
            kw.update(obs_x0=gi["x_obs"], obs_mask=gi["kf_mask"])
        with RH.noise_tape(gi["tape"][:n_draws(sampler)]):
            out[name] = loops[sampler](model, shape, clip_denoised=False, model_kwargs=kw, skip_timesteps=SKIP,
                                       init_image=gi["x_obs"] if imputate else None, device="cpu", progress=False)
    return out


def main():
    from oracle import reference_harness as RH
    if not RH.available():
        raise SystemExit("the reference tree is required to (re)generate golden vectors")
    os.makedirs(GOLDEN, exist_ok=True)
    torch.set_num_threads(os.cpu_count() or 1)
    ref = RH.import_reference()
    want = reference_outputs(ref, RH)
    got = restated_outputs()
    arrays = {}
    for name, r in want.items():
        r = r.detach()
        err = (r - got[name]).abs().max().item() / r.abs().max().item()
        print(f"  {name:15s} reference == restatement: {torch.equal(r, got[name])} (max diff / max |ref| {err:.3e})")
        arrays[f"{name}.ref"] = r.numpy()
    save_golden(GOLDEN, "cfg_interval", **arrays)


if __name__ == "__main__":
    main()

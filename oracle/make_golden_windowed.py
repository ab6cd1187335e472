"""TEST INFRASTRUCTURE -- anchors the overlapping-window restatement (oracle/windowed_oracle.py) to the UNMODIFIED reference
and writes tests/golden/windowed.*.

Run in the build container (needs the reference tree):   python -m oracle.make_golden_windowed

The reference samples one window per sequence.  For each configuration of windowed_oracle.FIXTURES this drives the
reference's own SpacedDiffusion.p_sample / ddim_sample (its model, ClassifierFreeSampleModel, imputation, keyframe input
and reconstruction guidance, read from model_kwargs) on the batch of B * K window rows, with the windows' crops of the
global inputs and of the global noise tape.  The blend is inserted by a harness shim, no source edit: the diffusion
object's p_mean_variance is wrapped so that the pred_xstart the reference computed is replaced by the window blend, and
the posterior mean is recomputed from it through the reference's q_posterior_mean_variance.  The result is gathered to
the global layout.  It asserts that the restatement agrees and stores the REFERENCE-driven output:
  - text_k2    transformer, per-window prompts, CFG 2.5 + imputation, 300 frames in 2 windows of 196, DDPM, last 5 steps;
  - guided_k3  the same with reconstruction guidance w = 20 (stop_recguidance_at = 2), 200 frames in 3 windows of 120
               (frames 80..119 covered three times, by the end-aligned window too), DDIM, last 4 steps;
  - unet_k3    keyframe-conditioned MDM_UNET xl, CFG 2.5 + keyframe input, the K = 3 placement, DDPM, last 4 steps.
Each starts from q_sample(x_obs) at its first step (init_image).
"""
from __future__ import annotations

import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import condmdi_oracle as O  # noqa: E402
from oracle import reference_harness as RH  # noqa: E402
from oracle import windowed_oracle as W  # noqa: E402
from oracle.golden_io import save_golden  # noqa: E402
from oracle.make_golden import GOLDEN, close, ref_model_with  # noqa: E402

# |reference-driven loop - restatement| in fp32: the two p_mean_variance implementations agree to the last bits of the
# denoiser's own summation order
ANCHOR_TOL = 2e-5


def blend_shim(diffusion, f0, n):
    """Wrap diffusion.p_mean_variance (an instance attribute shadows the method p_sample / ddim_sample call): the
    reference's pred_xstart replaced by the window blend, the mean recomputed by its q_posterior_mean_variance."""
    plain = diffusion.p_mean_variance

    def shim(model, x, t, **kw):
        out = dict(plain(model, x, t, **kw))
        pred = W.blend(out["pred_xstart"], f0, n)
        mean, _, _ = diffusion.q_posterior_mean_variance(x_start=pred, x_t=x, t=t)
        out["pred_xstart"], out["mean"] = pred, mean
        return out
    diffusion.p_mean_variance = shim
    return plain


def run_reference(name, model):
    N, F, O_, sampler, respacing, skip, guided, unet = W.FIXTURES[name]
    f0 = W.placement(N, F, O_)
    K, Bw = len(f0), W.B_FIX * len(f0)
    x_obs, kf, cond_w, scale, tape = W.fixture_inputs(name)
    crop = lambda t: W.crop(t, f0, F).contiguous()  # noqa: E731
    model_core = model.model if hasattr(model, "model") else model
    model_core._synthetic_text_emb = cond_w
    y = {"text": [str(i) for i in range(Bw)], "text_scale": scale.repeat_interleave(K),
         "mask": torch.ones(Bw, 1, 1, F, dtype=torch.bool), "lengths": torch.full((Bw,), F)}
    kwargs = {"y": y}
    if unet:
        kwargs.update(obs_x0=crop(x_obs), obs_mask=crop(kf))
    else:
        y.update(imputate=1, stop_imputation_at=1, replacement_distribution="conditional", inpainted_motion=crop(x_obs),
                 inpainting_mask=crop(kf))
    if guided:
        y.update(reconstruction_guidance=True, reconstruction_weight=20.0, gradient_schedule=None, diffusion_steps=1000,
                 stop_recguidance_at=2)
    d = RH.build_reference_diffusion(respacing)
    blend_shim(d, f0, N)
    t0 = d.num_timesteps - 1 - skip
    img = d.q_sample(crop(x_obs), torch.full((Bw,), t0, dtype=torch.long), crop(tape[0]))
    for k, i in enumerate(range(t0, -1, -1)):
        t = torch.tensor([i] * Bw)
        noise = crop(tape[1 + k])
        with RH.noise_tape(noise[None]) as st:
            if sampler == "ddpm":
                out = d.p_sample(model, img, t, clip_denoised=False, model_kwargs=kwargs)
            else:
                out = d.ddim_sample(model, img, t, clip_denoised=False, model_kwargs=kwargs, eta=0.0)
        assert st["k"] == 1, st["k"]
        img = out["sample"].detach()
    return W.gather(img, f0, N)


def golden_windowed():
    ref = RH.import_reference()
    out = {}
    sdt = O.random_state_dict(seed=7, text=True)
    mt = ref_model_with(sdt, text=True)
    sdu = O.random_unet_state_dict(seed=11, text=True)
    mu = RH.build_reference_unet(text=True)
    missing, unexpected = mu.load_state_dict(sdu, strict=False)
    assert not missing and not unexpected, (missing, unexpected)
    for name in sorted(W.FIXTURES):
        unet = W.FIXTURES[name][-1]
        sd, core = (sdu, mu) if unet else (sdt, mt)
        print(name)
        got_ref = run_reference(name, ref.cfg_sampler.ClassifierFreeSampleModel(core))
        got = W.fixture_restatement(name, sd)
        err = (got_ref.double() - got.double()).abs().max().item()
        close(got_ref, got, ANCHOR_TOL, f"{name}: reference-driven windows vs restatement")
        x_obs, _, cond_w, _, tape = W.fixture_inputs(name)
        out[f"{name}.ref"] = got_ref.numpy()
        out[f"{name}.err"] = np.array([err])
        out[f"{name}.checksum"] = np.array([float(x_obs.double().sum()), float(tape.double().sum()), float(cond_w.double().sum())])
    save_golden(GOLDEN, "windowed", **out)


def main():
    if not RH.available():
        raise SystemExit("the reference tree is required to (re)generate golden vectors")
    os.makedirs(GOLDEN, exist_ok=True)
    torch.set_num_threads(os.cpu_count() or 1)
    golden_windowed()
    for f in sorted(os.listdir(GOLDEN)):
        if f.startswith("windowed."):
            print(f, os.path.getsize(os.path.join(GOLDEN, f)) // 1024, "KiB")


if __name__ == "__main__":
    main()

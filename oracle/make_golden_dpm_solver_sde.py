"""TEST INFRASTRUCTURE -- anchors the SDE-DPM-Solver++ restatement (oracle/dpm_solver_sde_oracle.py) to the UNMODIFIED
reference and writes tests/golden/dpm_solver_sde.*.

Run in the build container (needs the reference tree):   python -m oracle.make_golden_dpm_solver_sde

The reference has no SDE-DPM-Solver++; its order 1 is the DDPM posterior step.  For every configuration below this runs
the reference's own p_sample_loop and the restated order 1 on the same noise tape (x_T, then one draw per step, the
last included), asserts that they agree, and stores the REFERENCE's output (the order-1 anchor) with the restatement's
order-2 output (regression values):
  - B = 2, ddim50, transformer no_cond, the whole loop;
  - CFG 2.5 + imputation, the last 5 steps;
  - CFG + imputation + reconstruction guidance (w = 20, stop_recguidance_at = 2 inside the loop), the last 4 steps;
  - the keyframe-conditioned MDM_UNET xl with CFG, the last 5 steps.
The tape is golden_inputs()'s 8 draws cycled to the 51 a whole ddim50 loop takes (as tests/golden/sampler.npz's ddim50
loop does).
"""
from __future__ import annotations

import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import condmdi_oracle as O  # noqa: E402
from oracle import dpm_solver_sde_oracle as S  # noqa: E402
from oracle import reference_harness as RH  # noqa: E402
from oracle.golden_io import save_golden  # noqa: E402
from oracle.make_golden import GOLDEN, close, ref_model_with  # noqa: E402

B, D, L = 2, 263, 196
# |reference DDPM - restated order 1| in fp32: the folded coefficients round differently from the reference's posterior
# tables and exp(0.5 log variance) (measured: 1.7e-6 no_cond whole loop, 4.7e-6 CFG + imputation, 5.1e-6 guided
# w = 20, 8.5e-6 UNet xl)
ANCHOR_TOL = 2e-5


def tape51(tape: torch.Tensor) -> torch.Tensor:
    """golden_inputs()'s 8 draws cycled to x_T + 50 per-step draws"""
    return tape[torch.arange(51) % 8]


def golden_dpm_solver_sde():
    ref = RH.import_reference()
    out = {}
    gi = O.golden_inputs()
    x, cond, x_obs, tape, scale, lengths, y_mask, kf_mask = (gi[k] for k in (
        "x", "cond", "x_obs", "tape", "text_scale", "lengths", "y_mask", "kf_mask"))
    out["inputs.checksum"] = np.array([float(x.double().sum()), float(tape.double().sum()), float(cond.double().sum())])
    tape = tape51(tape)
    sd = O.random_state_dict(seed=7, text=False)
    m = ref_model_with(sd, text=False)
    sdt = O.random_state_dict(seed=7, text=True)
    mt = ref_model_with(sdt, text=True)
    mt._synthetic_text_emb = cond
    cfgm = ref.cfg_sampler.ClassifierFreeSampleModel(mt)
    d50 = RH.build_reference_diffusion("ddim50")
    tab50 = O.make_tables("ddim50")
    shape = (B, D, 1, L)

    def run_ref(model, kwargs, skip=0, init_image=None):
        n = 50 - skip
        with RH.noise_tape(tape[:n + 1]) as st:
            r = d50.p_sample_loop(model, shape, model_kwargs=kwargs, device="cpu", clip_denoised=False,
                                  skip_timesteps=skip, init_image=init_image)
        assert st["k"] == n + 1, st["k"]  # x_T, then one randn_like per step, the last included
        return r

    def case(name, model, kwargs, sdx, c, skip=0, init_image=None):
        print(name)
        r = run_ref(model, kwargs, skip, init_image)
        o = {order: S.dpm_solver_sde_sample_loop(sdx, tab50, shape, c, tape, order, skip_timesteps=skip, init_image=init_image)
             for order in (1, 2)}
        err = (r.double() - o[1].double()).abs().max().item()
        print(f"  order 1: max|order 1 - reference p_sample_loop| = {err:.3e}")
        close(r, o[1], ANCHOR_TOL, f"{name}: reference p_sample_loop vs order 1")
        print(f"  order 2: max|order 2 - reference p_sample_loop| = {(o[2] - r).abs().max().item():.3e}")
        out[f"{name}.ddpm_ref"] = r.numpy()
        out[f"{name}.o1_err"] = np.array([err])
        out[f"{name}.o2"] = o[2].numpy()

    case("no_cond", m, {"y": {}}, sd, O.Conditioning())

    ykw = {"text": ["a", "b"], "text_scale": scale, "mask": y_mask, "lengths": lengths, "imputate": 1,
           "stop_imputation_at": 1, "replacement_distribution": "conditional", "inpainted_motion": x_obs,
           "inpainting_mask": kf_mask}
    c = O.Conditioning(cond_emb=cond, cfg=True, text_scale=scale, y_mask=y_mask, imputate=True, stop_imputation_at=1,
                       inpainted_motion=x_obs, inpainting_mask=kf_mask)
    case("cfg_impute", cfgm, {"y": ykw}, sdt, c, skip=45, init_image=x_obs)

    ykw2 = dict(ykw)
    ykw2.update(reconstruction_guidance=True, reconstruction_weight=20.0, gradient_schedule=None, diffusion_steps=1000,
                stop_recguidance_at=2)
    c2 = O.Conditioning(cond_emb=cond, cfg=True, text_scale=scale, y_mask=y_mask, imputate=True, stop_imputation_at=1,
                        inpainted_motion=x_obs, inpainting_mask=kf_mask, reconstruction_guidance=True,
                        reconstruction_weight=20.0, stop_recguidance_at=2)
    case("guided", cfgm, {"y": ykw2}, sdt, c2, skip=46, init_image=x_obs)

    sdu = O.random_unet_state_dict(seed=11, text=True)
    mu = RH.build_reference_unet(text=True)
    missing, unexpected = mu.load_state_dict(sdu, strict=False)
    assert not missing and not unexpected, (missing, unexpected)
    mu._synthetic_text_emb = cond
    cfgu = ref.cfg_sampler.ClassifierFreeSampleModel(mu)
    kw = {"y": {"text": ["a", "b"], "text_scale": scale, "mask": y_mask, "lengths": lengths}, "obs_x0": x_obs, "obs_mask": kf_mask}
    cu = O.Conditioning(cond_emb=cond, cfg=True, text_scale=scale, obs_x0=x_obs, obs_mask=kf_mask)
    case("unet", cfgu, kw, sdu, cu, skip=45, init_image=x_obs)
    save_golden(GOLDEN, "dpm_solver_sde", **out)


def main():
    if not RH.available():
        raise SystemExit("the reference tree is required to (re)generate golden vectors")
    os.makedirs(GOLDEN, exist_ok=True)
    torch.set_num_threads(os.cpu_count() or 1)
    golden_dpm_solver_sde()
    for f in sorted(os.listdir(GOLDEN)):
        if f.startswith("dpm_solver_sde."):
            print(f, os.path.getsize(os.path.join(GOLDEN, f)) // 1024, "KiB")


if __name__ == "__main__":
    main()

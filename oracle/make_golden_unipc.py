"""TEST INFRASTRUCTURE -- anchors the UniPC restatement (oracle/unipc_oracle.py) to the UNMODIFIED reference and writes
tests/golden/unipc.*.

Run in the build container (needs the reference tree):   python -m oracle.make_golden_unipc

The reference has no UniPC; its order 1 without the corrector is DDIM at eta = 0.  For every configuration below this
runs the reference's own ddim_sample_loop (eta = 0; the per-step draws are zeros, which sigma = 0 multiplies anyway) and
the restated order 1 without the corrector on the same inputs, asserts that they agree, and stores the REFERENCE's output
(the anchor) with the restatement's outputs at orders 1-3, with and without the corrector, under bh1 and bh2 (regression
values; order 1 without the corrector does not depend on the variant and is stored once, as "p1").  The configurations
are those of tests/golden/dpm_solver.*:
  - B = 2, ddim50, transformer no_cond, the whole loop;
  - CFG 2.5 + imputation, the last 5 steps;
  - CFG + imputation + reconstruction guidance (w = 20, stop_recguidance_at = 2 inside the loop), the last 4 steps;
  - the keyframe-conditioned MDM_UNET xl with CFG, the last 5 steps.
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
from oracle import unipc_oracle as U  # noqa: E402
from oracle.golden_io import save_golden  # noqa: E402
from oracle.make_golden import GOLDEN, close, ref_model_with  # noqa: E402

B, D, L = 2, 263, 196
# |reference DDIM - restated order 1| in fp32: the folded update rounds differently from the reference's eps form (the
# same bound, and the same folded row, as make_golden_dpm_solver's order 1)
ANCHOR_TOL = 1e-4


def variants():
    """(key, order, variant, corrector) of every stored run"""
    out = [("p1", 1, "bh2", False)]
    for variant in U.VARIANTS:
        out += [(f"p{o}_{variant}", o, variant, False) for o in (2, 3)]
        out += [(f"c{o}_{variant}", o, variant, True) for o in (1, 2, 3)]
    return out


def golden_unipc():
    ref = RH.import_reference()
    out = {}
    gi = O.golden_inputs()
    x, cond, x_obs, tape, scale, lengths, y_mask, kf_mask = (gi[k] for k in (
        "x", "cond", "x_obs", "tape", "text_scale", "lengths", "y_mask", "kf_mask"))
    out["inputs.checksum"] = np.array([float(x.double().sum()), float(tape.double().sum()), float(cond.double().sum())])
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
        draws = torch.cat([tape[:1], torch.zeros((n,) + shape)])  # x_T, then one (unused) randn_like per step
        with RH.noise_tape(draws) as st:
            r = d50.ddim_sample_loop(model, shape, model_kwargs=kwargs, device="cpu", clip_denoised=False, eta=0.0,
                                     skip_timesteps=skip, init_image=init_image)
        assert st["k"] == n + 1, st["k"]
        return r

    def case(name, model, kwargs, sdx, c, skip=0, init_image=None):
        print(name)
        r = run_ref(model, kwargs, skip, init_image)
        out[f"{name}.ddim_ref"] = r.numpy()
        for key, order, variant, corrector in variants():
            o = U.unipc_sample_loop(sdx, tab50, shape, c, tape, order, variant, corrector, skip_timesteps=skip,
                                    init_image=init_image)
            if key == "p1":
                err = (r.double() - o.double()).abs().max().item()
                close(r, o, ANCHOR_TOL, f"{name}: reference ddim_sample_loop vs UniP order 1")
                out[f"{name}.p1_err"] = np.array([err])
            else:
                print(f"  {key}: max|{key} - reference DDIM| = {(o - r).abs().max().item():.3e}")
            out[f"{name}.{key}"] = o.numpy()

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
    save_golden(GOLDEN, "unipc", **out)


def main():
    if not RH.available():
        raise SystemExit("the reference tree is required to (re)generate golden vectors")
    os.makedirs(GOLDEN, exist_ok=True)
    torch.set_num_threads(os.cpu_count() or 1)
    golden_unipc()
    for f in sorted(os.listdir(GOLDEN)):
        if f.startswith("unipc."):
            print(f, os.path.getsize(os.path.join(GOLDEN, f)) // 1024, "KiB")


if __name__ == "__main__":
    main()

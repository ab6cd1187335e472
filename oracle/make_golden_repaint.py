"""TEST INFRASTRUCTURE -- anchors the RePaint restatement (oracle/repaint_oracle.py) to the UNMODIFIED reference and writes
tests/golden/repaint.*.

Run in the build container (needs the reference tree):   python -m oracle.make_golden_repaint

The reference has no RePaint loop, but every denoise op of the walk is its p_sample.  For every configuration below this
drives the reference's own SpacedDiffusion.p_sample (its model, ClassifierFreeSampleModel, imputation and reconstruction
guidance, read from model_kwargs as in its p_sample_loop) along the walk, with the undo op x <- a_p x + b_p z restated,
on one noise tape (x_T, then one draw per op).  It asserts that the restatement agrees, and stores the REFERENCE-driven
output:
  - B = 2, ddim50, transformer no_cond, the whole loop, jump_length 5, jump_n_sample 3;
  - CFG 2.5 + imputation, the last 10 steps, jump_length 4, jump_n_sample 3 (jump points 4 and 0);
  - CFG + imputation + reconstruction guidance (w = 20), the last 6 steps, jump_length 3, jump_n_sample 2, with
    stop_recguidance_at = 2: the jumped stretch 3..1 is revisited guided at 3 and 2 and unguided at 1;
  - the keyframe-conditioned MDM_UNET xl with CFG, the last 5 steps, jump_length 2, jump_n_sample 2.
The tape is golden_inputs()'s 8 draws cycled to the walk's length.
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
from oracle import repaint_oracle as R  # noqa: E402
from oracle.golden_io import save_golden  # noqa: E402
from oracle.make_golden import GOLDEN, close, ref_model_with  # noqa: E402

B, D, L = 2, 263, 196
# |reference-driven walk - restatement| in fp32: the two p_sample implementations agree to the last bits of the
# denoiser's own summation order
ANCHOR_TOL = 2e-5
# (name, skip_timesteps, jump_length, jump_n_sample)
CASES = [("no_cond", 0, 5, 3), ("cfg_impute", 40, 4, 3), ("guided", 44, 3, 2), ("unet", 45, 2, 2)]


def cycled(tape: torch.Tensor, n: int) -> torch.Tensor:
    """golden_inputs()'s 8 draws cycled to x_T + n per-op draws"""
    return tape[torch.arange(n + 1) % 8]


def golden_repaint():
    ref = RH.import_reference()
    out = {}
    gi = O.golden_inputs()
    x, cond, x_obs, tape8, scale, lengths, y_mask, kf_mask = (gi[k] for k in (
        "x", "cond", "x_obs", "tape", "text_scale", "lengths", "y_mask", "kf_mask"))
    out["inputs.checksum"] = np.array([float(x.double().sum()), float(tape8.double().sum()), float(cond.double().sum())])
    sd = O.random_state_dict(seed=7, text=False)
    m = ref_model_with(sd, text=False)
    sdt = O.random_state_dict(seed=7, text=True)
    mt = ref_model_with(sdt, text=True)
    mt._synthetic_text_emb = cond
    cfgm = ref.cfg_sampler.ClassifierFreeSampleModel(mt)
    d50 = RH.build_reference_diffusion("ddim50")
    tab50 = O.make_tables("ddim50")
    a, b = R.undo_coefficients(tab50)
    shape = (B, D, 1, L)

    def run_ref(model, kwargs, skip, j, r, tape, init_image):
        """the reference's p_sample along the walk; the undo op restated"""
        t0 = 49 - skip
        walk = R.build_walk(t0, j, r)
        img = tape[0].clone()
        if init_image is not None:
            img = d50.q_sample(init_image, torch.full((B,), t0, dtype=torch.long), img)
        with RH.noise_tape(tape[1:len(walk) + 1]) as st:
            for kind, p in walk:
                if kind == R.UNDO:
                    img = R.undo(img, a[p], b[p], torch.randn_like(img))
                    continue
                with torch.no_grad():
                    img = d50.p_sample(model, img, torch.tensor([p] * B), clip_denoised=False, model_kwargs=kwargs)["sample"]
        assert st["k"] == len(walk), st["k"]  # one draw per op, step 0's included
        return img

    def case(name, model, kwargs, sdx, c):
        _, skip, j, r = next(cs for cs in CASES if cs[0] == name)
        print(name)
        walk = R.build_walk(49 - skip, j, r)
        nd, nu = R.op_counts(49 - skip, j, r)
        assert (sum(k == R.DENOISE for k, _ in walk), sum(k == R.UNDO for k, _ in walk)) == (nd, nu)
        tape = cycled(tape8, len(walk))
        init = x_obs if skip else None
        got_ref = run_ref(model, kwargs, skip, j, r, tape, init)
        got = R.repaint_sample_loop(sdx, tab50, shape, c, tape, j, r, skip_timesteps=skip, init_image=init)
        err = (got_ref.double() - got.double()).abs().max().item()
        print(f"  {nd} denoise + {nu} undo ops: max|restatement - reference p_sample walk| = {err:.3e}")
        close(got_ref, got, ANCHOR_TOL, f"{name}: reference p_sample walk vs restatement")
        out[f"{name}.ref"] = got_ref.numpy()
        out[f"{name}.err"] = np.array([err])
        out[f"{name}.config"] = np.array([skip, j, r])

    case("no_cond", m, {"y": {}}, sd, O.Conditioning())

    ykw = {"text": ["a", "b"], "text_scale": scale, "mask": y_mask, "lengths": lengths, "imputate": 1,
           "stop_imputation_at": 1, "replacement_distribution": "conditional", "inpainted_motion": x_obs,
           "inpainting_mask": kf_mask}
    c = O.Conditioning(cond_emb=cond, cfg=True, text_scale=scale, y_mask=y_mask, imputate=True, stop_imputation_at=1,
                       inpainted_motion=x_obs, inpainting_mask=kf_mask)
    case("cfg_impute", cfgm, {"y": ykw}, sdt, c)

    ykw2 = dict(ykw)
    ykw2.update(reconstruction_guidance=True, reconstruction_weight=20.0, gradient_schedule=None, diffusion_steps=1000,
                stop_recguidance_at=2)
    c2 = O.Conditioning(cond_emb=cond, cfg=True, text_scale=scale, y_mask=y_mask, imputate=True, stop_imputation_at=1,
                        inpainted_motion=x_obs, inpainting_mask=kf_mask, reconstruction_guidance=True,
                        reconstruction_weight=20.0, stop_recguidance_at=2)
    case("guided", cfgm, {"y": ykw2}, sdt, c2)

    sdu = O.random_unet_state_dict(seed=11, text=True)
    mu = RH.build_reference_unet(text=True)
    missing, unexpected = mu.load_state_dict(sdu, strict=False)
    assert not missing and not unexpected, (missing, unexpected)
    mu._synthetic_text_emb = cond
    cfgu = ref.cfg_sampler.ClassifierFreeSampleModel(mu)
    kw = {"y": {"text": ["a", "b"], "text_scale": scale, "mask": y_mask, "lengths": lengths}, "obs_x0": x_obs, "obs_mask": kf_mask}
    cu = O.Conditioning(cond_emb=cond, cfg=True, text_scale=scale, obs_x0=x_obs, obs_mask=kf_mask)
    case("unet", cfgu, kw, sdu, cu)
    save_golden(GOLDEN, "repaint", **out)


def main():
    if not RH.available():
        raise SystemExit("the reference tree is required to (re)generate golden vectors")
    os.makedirs(GOLDEN, exist_ok=True)
    torch.set_num_threads(os.cpu_count() or 1)
    golden_repaint()
    for f in sorted(os.listdir(GOLDEN)):
        if f.startswith("repaint."):
            print(f, os.path.getsize(os.path.join(GOLDEN, f)) // 1024, "KiB")


if __name__ == "__main__":
    main()

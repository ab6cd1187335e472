"""TEST INFRASTRUCTURE -- anchors the joint-guidance restatement (oracle/joint_guidance_oracle.py) to the UNMODIFIED
reference and writes tests/golden/joint_guidance.*.

Run in the build container (needs the reference tree):   python -m oracle.make_golden_joint_guidance

The reference has no joint guidance, so the fixtures come from its own pieces: its model call (MDM / MDM_UNET wrapped in
its ClassifierFreeSampleModel), its recover_from_ric (data_loaders/humanml/scripts/motion_process.py:402-489) on the
de-normalised x0_hat, both losses differentiated with torch.autograd.grad, driven by the restated update
x0_tilde = x0_hat - ~M (c_r dL_r/dz + c_j dL_j/dz) and imputation.  One guided evaluation (p_mean_variance's pred_xstart
and mean) per case, on golden_inputs() and joint_guidance_oracle.inputs(seed=5):
  - the transformer, CFG 2.5, imputation, reconstruction (w = 20) + joint guidance (weight 0.1), t = 500 and 30, in the
    abs_3d and the relative representation;
  - the transformer, CFG 2.5, joint guidance alone (no feature keyframes), abs_3d, t = 500;
  - the keyframe-conditioned MDM_UNET xl with CFG 2.5, imputation, reconstruction + joint guidance, abs_3d, t = 500, in
    fp32 and under CPU fp16 autocast (the model call inside torch.autocast("cpu", float16), the losses outside it).
It asserts that the restatement agrees and stores the REFERENCE-driven outputs with the measured gaps.
"""
from __future__ import annotations

import contextlib
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import condmdi_oracle as O  # noqa: E402
from oracle import joint_guidance_oracle as J  # noqa: E402
from oracle import reference_harness as RH  # noqa: E402
from oracle.golden_io import save_golden  # noqa: E402
from oracle.make_golden import GOLDEN, ref_model_with  # noqa: E402
from oracle.make_golden_unet_guidance import cpu_autocast, model_calls_under  # noqa: E402

B, D, L = 2, 263, 196
WEIGHT = 0.1
# (name, model, t, abs_3d, feature keyframes, autocast)
CASES = [("trans.rel.t500", "trans", 500, False, True, False), ("trans.rel.t30", "trans", 30, False, True, False),
         ("trans.abs.t500", "trans", 500, True, True, False), ("trans.abs.t30", "trans", 30, True, True, False),
         ("trans.joint_only.t500", "trans", 500, True, False, False),
         ("unet.fp32.t500", "unet", 500, True, True, False), ("unet.fp16.t500", "unet", 500, True, True, True)]


def conditioning(gi, keyframes, unet):
    kf = dict(imputate=True, stop_imputation_at=0, inpainted_motion=gi["x_obs"], inpainting_mask=gi["kf_mask"],
              reconstruction_guidance=True, reconstruction_weight=20.0, stop_recguidance_at=0) if keyframes else {}
    obs = dict(obs_x0=gi["x_obs"], obs_mask=gi["kf_mask"]) if unet else {}
    return O.Conditioning(cond_emb=gi["cond"], cfg=True, text_scale=gi["text_scale"], y_mask=gi["y_mask"], **kf, **obs)


def term(abs_3d):
    mean, std, jt, jm, _ = J.inputs(B, L, seed=5)
    return J.JointTerm(jt, jm, mean, std, abs_3d, WEIGHT)


def run_reference(ref_fk, model, gi, t, j: J.JointTerm, keyframes, unet, autocast):
    """the reference's model call and recover_from_ric under autograd, the restated update"""
    tab = O.make_tables("")
    tt = torch.tensor([t, t])
    y = {"text": ["a", "b"], "text_scale": gi["text_scale"], "mask": gi["y_mask"], "lengths": gi["lengths"]}
    extra = {"obs_x0": gi["x_obs"], "obs_mask": gi["kf_mask"]} if unet else {}
    ym = gi["y_mask"]
    M = gi["kf_mask"] & ym if keyframes else torch.zeros(B, D, 1, L, dtype=torch.bool)
    Mj = j.mask & ym.reshape(B, L)[:, :, None, None]
    z = gi["x"].detach().clone().requires_grad_(True)
    with torch.enable_grad():
        with cpu_autocast() if autocast else contextlib.nullcontext():
            hat = model(z, tt, y=y, **extra)
        hat = hat.float()
        data = hat.permute(0, 2, 3, 1) * j.std + j.mean                      # inv_transform of (B, 1, L, 263)
        pos = ref_fk(data, 22, abs_3d=j.abs_3d)[:, 0]                        # (B, L, 22, 3)
        cj = J._coef(None, 1000, j.weight, tab, tt, z.shape, z.device)
        grad = cj * torch.autograd.grad(((pos - j.target).square() * Mj).sum(), z, retain_graph=keyframes)[0]
        if keyframes:
            cr = J._coef(None, 1000, 20.0, tab, tt, z.shape, z.device)
            grad = cr * torch.autograd.grad(((gi["x_obs"] - hat).square() * M).sum(), z)[0] + grad
    hat = hat.detach()
    tilde = hat - grad * (~M).float()
    pred = (tilde * ~M) + (gi["x_obs"] * M)
    mean = O.extract(tab.posterior_mean_coef1, tt, z.shape) * pred + O.extract(tab.posterior_mean_coef2, tt, z.shape) * gi["x"]
    return pred, mean


def run_oracle(sd, gi, t, j, keyframes, unet, autocast):
    with model_calls_under(cpu_autocast if autocast else None):
        out = J.p_mean_variance(sd, O.make_tables(""), gi["x"], torch.tensor([t, t]), conditioning(gi, keyframes, unet), j)
    return out["pred_xstart"].detach(), out["mean"].detach()


def golden_joint_guidance():
    ref = RH.import_reference()
    from data_loaders.humanml.scripts.motion_process import recover_from_ric as ref_fk  # noqa: E402
    gi = O.golden_inputs()
    sdt = O.random_state_dict(seed=7, text=True)
    mt = ref_model_with(sdt, text=True)
    mt._synthetic_text_emb = gi["cond"]
    sdu = O.random_unet_state_dict(seed=11, text=True)
    mu = RH.build_reference_unet(text=True)
    missing, unexpected = mu.load_state_dict(sdu, strict=False)
    assert not missing and not unexpected, (missing, unexpected)
    mu._synthetic_text_emb = gi["cond"]
    models = {"trans": (ref.cfg_sampler.ClassifierFreeSampleModel(mt), sdt),
              "unet": (ref.cfg_sampler.ClassifierFreeSampleModel(mu), sdu)}
    out = {"inputs.checksum": np.array([float(gi["x"].double().sum()), float(term(True).target.double().sum())])}
    for name, which, t, abs_3d, keyframes, autocast in CASES:
        model, sd = models[which]
        j = term(abs_3d)
        r = run_reference(ref_fk, model, gi, t, j, keyframes, which == "unet", autocast)
        o = run_oracle(sd, gi, t, j, keyframes, which == "unet", autocast)
        err = max((a - b).abs().max().item() for a, b in zip(r, o))
        scale = r[0].abs().max().item()
        print(f"  {name:22s} reference == restatement: {all(torch.equal(a, b) for a, b in zip(r, o))}  "
              f"max diff {err:.3e} (max |pred_xstart| {scale:.3e})")
        assert err <= 1e-4 * max(1.0, scale), f"{name}: the restatement differs from the reference by {err:.3e}"
        out[f"{name}.pred_xstart"] = r[0].numpy()
        out[f"{name}.mean"] = r[1].numpy()
        out[f"{name}.err"] = np.array([err])
    save_golden(GOLDEN, "joint_guidance", **out)


def main():
    if not RH.available():
        raise SystemExit("the reference tree is required to (re)generate golden vectors")
    os.makedirs(GOLDEN, exist_ok=True)
    torch.set_num_threads(os.cpu_count() or 1)
    golden_joint_guidance()
    for f in sorted(os.listdir(GOLDEN)):
        if f.startswith("joint_guidance."):
            print(f, os.path.getsize(os.path.join(GOLDEN, f)) // 1024, "KiB")


if __name__ == "__main__":
    main()

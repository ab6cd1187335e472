"""TEST INFRASTRUCTURE -- anchors the foot-contact restatement (oracle/foot_contact_oracle.py) to the UNMODIFIED reference
and writes tests/golden/foot_contact.*.

Run in the build container (needs the reference tree):   python -m oracle.make_golden_foot_contact

The reference has no sampling-time foot-contact guidance, so the fixtures come from its own pieces: its model call (MDM /
MDM_UNET wrapped in its ClassifierFreeSampleModel), its recover_from_ric (data_loaders/humanml/scripts/motion_process.py)
on the de-normalised x0_hat, the losses differentiated with torch.autograd.grad, driven by the restated update
x0_tilde = x0_hat - ~M (c_r dL_r/dz + c_j dL_j/dz + c_c dL_c/dz) and imputation.  One guided evaluation (p_mean_variance's
pred_xstart and mean) per case, on golden_inputs() (ragged lengths 196 and 150) with the contact channels' statistics of
foot_contact_oracle.inputs(seed=5):
  - the transformer, CFG 2.5, imputation, reconstruction (w = 20) + foot-contact guidance (weight 0.1), t = 500, in the
    abs_3d and the relative representation; the same with joint guidance too (weight 0.1), abs_3d, t = 30; foot-contact
    guidance alone (no feature keyframes), abs_3d, t = 500;
  - the keyframe-conditioned MDM_UNET xl with CFG 2.5, imputation, reconstruction + foot-contact guidance, abs_3d,
    t = 500, in fp32 and under CPU fp16 autocast (the model call inside torch.autocast("cpu", float16), the losses
    outside it).
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
from oracle import foot_contact_oracle as FC  # noqa: E402
from oracle import joint_guidance_oracle as J  # noqa: E402
from oracle import reference_harness as RH  # noqa: E402
from oracle.golden_io import save_golden  # noqa: E402
from oracle.make_golden import GOLDEN, ref_model_with  # noqa: E402
from oracle.make_golden_unet_guidance import cpu_autocast, model_calls_under  # noqa: E402

B, D, L = 2, 263, 196
WEIGHT = 0.1
# (name, model, t, abs_3d, feature keyframes, joint term, autocast)
CASES = [("trans.abs.t500", "trans", 500, True, True, False, False),
         ("trans.rel.t500", "trans", 500, False, True, False, False),
         ("trans.abs.joint.t30", "trans", 30, True, True, True, False),
         ("trans.fc_only.t500", "trans", 500, True, False, False, False),
         ("unet.fp32.t500", "unet", 500, True, True, False, False),
         ("unet.fp16.t500", "unet", 500, True, True, False, True)]


def conditioning(gi, keyframes, unet):
    kf = dict(imputate=True, stop_imputation_at=0, inpainted_motion=gi["x_obs"], inpainting_mask=gi["kf_mask"],
              reconstruction_guidance=True, reconstruction_weight=20.0, stop_recguidance_at=0) if keyframes else {}
    obs = dict(obs_x0=gi["x_obs"], obs_mask=gi["kf_mask"]) if unet else {}
    return O.Conditioning(cond_emb=gi["cond"], cfg=True, text_scale=gi["text_scale"], y_mask=gi["y_mask"], **kf, **obs)


def terms(abs_3d, joint):
    mean, std, _, _ = FC.inputs(B, L, seed=5)
    fc = FC.FootContactTerm(mean, std, abs_3d, WEIGHT)
    if not joint:
        return fc, None
    _, _, jt, jm, _ = J.inputs(B, L, seed=5)
    return fc, J.JointTerm(jt, jm, mean, std, abs_3d, WEIGHT)


def run_reference(ref_fk, model, gi, t, fc: FC.FootContactTerm, j, keyframes, unet, autocast):
    """the reference's model call and recover_from_ric under autograd, the restated losses and update"""
    tab = O.make_tables("")
    tt = torch.tensor([t, t])
    y = {"text": ["a", "b"], "text_scale": gi["text_scale"], "mask": gi["y_mask"], "lengths": gi["lengths"]}
    extra = {"obs_x0": gi["x_obs"], "obs_mask": gi["kf_mask"]} if unet else {}
    ym = gi["y_mask"]
    M = gi["kf_mask"] & ym if keyframes else torch.zeros(B, D, 1, L, dtype=torch.bool)
    m = ym.reshape(B, L)
    z = gi["x"].detach().clone().requires_grad_(True)
    with torch.enable_grad():
        with cpu_autocast() if autocast else contextlib.nullcontext():
            hat = model(z, tt, y=y, **extra)
        hat = hat.float()
        data = hat.permute(0, 2, 3, 1) * fc.std + fc.mean                    # inv_transform of (B, 1, L, 263)
        pos = ref_fk(data, 22, abs_3d=fc.abs_3d)[:, 0]                       # (B, L, 22, 3)
        kappa = data[:, 0, :, 259:263].detach() > 0.5                        # (B, L, 4): feet_l (7, 10), feet_r (8, 11)
        w = (kappa[:, :-1] & m[:, :-1, None] & m[:, 1:, None]).float()
        feet = pos[:, :, [7, 10, 8, 11]]
        loss_c = ((feet[:, 1:] - feet[:, :-1]).square().sum(-1) * w).sum()
        cc = J._coef(None, 1000, fc.weight, tab, tt, z.shape, z.device)
        grad = cc * torch.autograd.grad(loss_c, z, retain_graph=True)[0]
        if j is not None:
            Mj = j.mask & m[:, :, None, None]
            cj = J._coef(None, 1000, j.weight, tab, tt, z.shape, z.device)
            grad = cj * torch.autograd.grad(((pos - j.target).square() * Mj).sum(), z, retain_graph=keyframes)[0] + grad
        if keyframes:
            cr = J._coef(None, 1000, 20.0, tab, tt, z.shape, z.device)
            grad = cr * torch.autograd.grad(((gi["x_obs"] - hat).square() * M).sum(), z)[0] + grad
    hat = hat.detach()
    tilde = hat - grad * (~M).float()
    pred = (tilde * ~M) + (gi["x_obs"] * M)
    mean = O.extract(tab.posterior_mean_coef1, tt, z.shape) * pred + O.extract(tab.posterior_mean_coef2, tt, z.shape) * gi["x"]
    return pred, mean, int(w.sum().item())


def run_oracle(sd, gi, t, fc, j, keyframes, unet, autocast):
    with model_calls_under(cpu_autocast if autocast else None):
        out = FC.p_mean_variance(sd, O.make_tables(""), gi["x"], torch.tensor([t, t]), conditioning(gi, keyframes, unet), fc, j)
    return out["pred_xstart"].detach(), out["mean"].detach()


def golden_foot_contact():
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
    out = {"inputs.checksum": np.array([float(gi["x"].double().sum()), float(terms(True, False)[0].mean.double().sum())])}
    for name, which, t, abs_3d, keyframes, joint, autocast in CASES:
        model, sd = models[which]
        fc, j = terms(abs_3d, joint)
        pred, mean, n_contacts = run_reference(ref_fk, model, gi, t, fc, j, keyframes, which == "unet", autocast)
        r = (pred, mean)
        o = run_oracle(sd, gi, t, fc, j, keyframes, which == "unet", autocast)
        err = max((a - b).abs().max().item() for a, b in zip(r, o))
        scale = r[0].abs().max().item()
        print(f"  {name:22s} contact pairs {n_contacts:4d}  reference == restatement: "
              f"{all(torch.equal(a, b) for a, b in zip(r, o))}  max diff {err:.3e} (max |pred_xstart| {scale:.3e})")
        assert n_contacts > 0, f"{name}: no contact label exceeds 0.5"
        assert err <= 1e-4 * max(1.0, scale), f"{name}: the restatement differs from the reference by {err:.3e}"
        out[f"{name}.pred_xstart"] = r[0].numpy()
        out[f"{name}.mean"] = r[1].numpy()
        out[f"{name}.err"] = np.array([err])
    save_golden(GOLDEN, "foot_contact", **out)


def main():
    if not RH.available():
        raise SystemExit("the reference tree is required to (re)generate golden vectors")
    os.makedirs(GOLDEN, exist_ok=True)
    torch.set_num_threads(os.cpu_count() or 1)
    golden_foot_contact()
    for f in sorted(os.listdir(GOLDEN)):
        if f.startswith("foot_contact."):
            print(f, os.path.getsize(os.path.join(GOLDEN, f)) // 1024, "KiB")


if __name__ == "__main__":
    main()

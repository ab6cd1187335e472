"""TEST INFRASTRUCTURE -- pins the PLMS restatement (oracle/plms_oracle.py) against the UNMODIFIED reference's
plms_sample_loop_progressive and writes tests/golden/plms.*.

Run in the build container (needs the reference tree):   python -m oracle.make_golden_plms

Same procedure as oracle/make_golden.py: run the reference's own code on CPU on the seeded inputs of
`condmdi_oracle.golden_inputs`, run the restatement on the same inputs, assert they agree, store the REFERENCE's
outputs.  It also runs the whole order-2 / order-4 loops as a float64 chain of the restatement and prints how far the
fp32 runs are from it (DESIGN.md section 2).
"""
from __future__ import annotations

import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import condmdi_oracle as O  # noqa: E402
from oracle import plms_oracle as P  # noqa: E402
from oracle import reference_harness as RH  # noqa: E402
from oracle.golden_io import save_golden  # noqa: E402
from oracle.make_golden import GOLDEN, close, ref_model_with  # noqa: E402

B, D, L = 2, 263, 196


def golden_plms():
    """plms_sample_loop_progressive (gaussian_diffusion.py:1589-1804): the pseudo improved Euler first step (two
    evaluations, the second at t - 1), the Adams-Bashforth ramp through orders 2 -> 3 -> 4, CFG, imputation,
    reconstruction guidance, the keyframe-conditioned MDM_UNET and a one-step call at t = 0."""
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

    def run_ref(model, kwargs, order, steps=None, **kw):
        """(sample, pred_xstart, old_eps snapshot) of every yield: the reference yields the same history list every step
        and mutates it afterwards, so its values are copied at the yield"""
        outs = []
        with RH.noise_tape(tape[:1]):
            for k, o_ in enumerate(d50.plms_sample_loop_progressive(model, shape, model_kwargs=kwargs, device="cpu",
                                                                    clip_denoised=False, order=order, **kw)):
                outs.append({"sample": o_["sample"].clone(), "pred_xstart": o_["pred_xstart"].clone(),
                             "old_eps": [e.clone() for e in o_["old_eps"]]})
                if steps is not None and k + 1 == steps:
                    break
        return outs

    def check_all(r, o, tol, what):
        assert len(r) == len(o), (len(r), len(o))
        for k in range(len(r)):
            close(r[k]["sample"], o[k]["sample"], tol, f"{what} k={k} sample")
            close(r[k]["pred_xstart"], o[k]["pred_xstart"], tol, f"{what} k={k} pred_xstart")
            assert len(r[k]["old_eps"]) == len(o[k]["old_eps"])
            for a, b in zip(r[k]["old_eps"], o[k]["old_eps"]):
                # eps = (r1 x - x0) / r2 amplifies by 1 / r2[t] (up to ~60 at the last steps of ddim50)
                close(a, b, tol * 100, f"{what} k={k} old_eps")

    for order in (2, 4):
        print(f"plms_sample_loop ddim50, order {order}, all 50 steps")
        r = run_ref(m, {"y": {}}, order)
        o = P.plms_sample_loop(sd, tab50, shape, O.Conditioning(), tape, order, return_all=True)
        sd64 = {k: v.double() for k, v in sd.items()}
        o64 = P.plms_sample_loop(sd64, tab50, shape, O.Conditioning(), tape.double(), order, return_all=True)
        for k in (0, 1, 2, 3, 10, 20, 30, 40, 45, 48, 49):
            e_ro = (r[k]["sample"] - o[k]["sample"]).abs().max().item()
            e_r64 = (r[k]["sample"].double() - o64[k]["sample"]).abs().max().item()
            e_o64 = (o[k]["sample"].double() - o64[k]["sample"]).abs().max().item()
            print(f"  k={k:2d} (t={49 - k:2d}): |ref32 - oracle32| = {e_ro:.3e}  |ref32 - f64| = {e_r64:.3e}  "
                  f"|oracle32 - f64| = {e_o64:.3e}  max|x| = {r[k]['sample'].abs().max().item():.3f}")
        check_all(r[:4], o[:4], 5e-5, f"plms order {order}")
        close(r[-1]["sample"], o[-1]["sample"], 2e-4, f"plms order {order} final sample")
        keep = (0, 1, 2) if order == 2 else (3,)
        for k in keep:
            out[f"o{order}.sample_k{k}"] = r[k]["sample"].numpy()
        out[f"o{order}.final"] = r[-1]["sample"].numpy()
        out[f"o{order}.ref_err_vs_f64"] = np.array([(r[-1]["sample"].double() - o64[-1]["sample"]).abs().max().item(),
                                                    (r[-1]["sample"].double() - o64[-1]["sample"]).abs().mean().item()])

    ykw = {"text": ["a", "b"], "text_scale": scale, "mask": y_mask, "lengths": lengths, "imputate": 1,
           "stop_imputation_at": 1, "replacement_distribution": "conditional", "inpainted_motion": x_obs,
           "inpainting_mask": kf_mask}
    c = O.Conditioning(cond_emb=cond, cfg=True, text_scale=scale, y_mask=y_mask, imputate=True, stop_imputation_at=1,
                       inpainted_motion=x_obs, inpainting_mask=kf_mask)
    print("plms order 2, CFG 2.5 + imputation (stop_imputation_at=1), last 5 steps")
    r = run_ref(cfgm, {"y": ykw}, 2, skip_timesteps=45, init_image=x_obs)
    o = P.plms_sample_loop(sdt, tab50, shape, c, tape, 2, skip_timesteps=45, init_image=x_obs, return_all=True)
    check_all(r, o, 1e-4, "cfg+impute")
    out["cfg_impute.final"] = r[-1]["sample"].numpy()

    print("plms order 2, CFG + imputation + reconstruction guidance (w=20), first 2 steps")
    ykw2 = dict(ykw)
    ykw2.update(reconstruction_guidance=True, reconstruction_weight=20.0, gradient_schedule=None, diffusion_steps=1000,
                stop_recguidance_at=0)
    c2 = O.Conditioning(cond_emb=cond, cfg=True, text_scale=scale, y_mask=y_mask, imputate=True, stop_imputation_at=1,
                        inpainted_motion=x_obs, inpainting_mask=kf_mask, reconstruction_guidance=True, reconstruction_weight=20.0)
    r = run_ref(cfgm, {"y": ykw2}, 2, steps=2)
    o = P.plms_sample_loop(sdt, tab50, shape, c2, tape, 2, max_steps=2, return_all=True)
    check_all(r, o, 1e-4, "recon guidance")
    out["recon.sample_k1"] = r[-1]["sample"].numpy()

    print("plms order 2, one-step call at t = 0 (skip_timesteps = 49)")
    r = run_ref(m, {"y": {}}, 2, skip_timesteps=49, init_image=x_obs)
    o = P.plms_sample_loop(sd, tab50, shape, O.Conditioning(), tape, 2, skip_timesteps=49, init_image=x_obs, return_all=True)
    check_all(r, o, 5e-5, "t=0 one step")
    out["t0.sample"] = r[-1]["sample"].numpy()

    print("plms order 3, CFG + keyframe-conditioned MDM_UNET xl, last 5 steps")
    sdu = O.random_unet_state_dict(seed=11, text=True)
    mu = RH.build_reference_unet(text=True)
    missing, unexpected = mu.load_state_dict(sdu, strict=False)
    assert not missing and not unexpected, (missing, unexpected)
    mu._synthetic_text_emb = cond
    cfgu = ref.cfg_sampler.ClassifierFreeSampleModel(mu)
    kw = {"y": {"text": ["a", "b"], "text_scale": scale, "mask": y_mask, "lengths": lengths}, "obs_x0": x_obs, "obs_mask": kf_mask}
    r = run_ref(cfgu, kw, 3, skip_timesteps=45, init_image=x_obs)
    cu = O.Conditioning(cond_emb=cond, cfg=True, text_scale=scale, obs_x0=x_obs, obs_mask=kf_mask)
    o = P.plms_sample_loop(sdu, tab50, shape, cu, tape, 3, skip_timesteps=45, init_image=x_obs, return_all=True)
    check_all(r, o, 5e-5, "unet order 3")
    out["unet.final"] = r[-1]["sample"].numpy()
    save_golden(GOLDEN, "plms", **out)


def main():
    if not RH.available():
        raise SystemExit("the reference tree is required to (re)generate golden vectors")
    os.makedirs(GOLDEN, exist_ok=True)
    torch.set_num_threads(os.cpu_count() or 1)
    golden_plms()
    for f in sorted(os.listdir(GOLDEN)):
        if f.startswith("plms."):
            print(f, os.path.getsize(os.path.join(GOLDEN, f)) // 1024, "KiB")


if __name__ == "__main__":
    main()

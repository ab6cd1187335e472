"""TEST INFRASTRUCTURE -- pins the DDIM inversion restatement (oracle/ddim_reverse_oracle.py) against the UNMODIFIED
reference's ddim_reverse_sample and writes tests/golden/ddim_reverse.*.

Run in the build container (needs the reference tree):   python -m oracle.make_golden_ddim_reverse

Same procedure as oracle/make_golden.py: run the reference's own code on CPU on the seeded inputs of
`condmdi_oracle.golden_inputs`, run the restatement on the same inputs, assert they agree, store the REFERENCE's
outputs.  Two checks per step:
  - the reverse update (:1442-1450) restated on the reference's own x and pred_xstart equals the reference's sample bit
    for bit;
  - the whole restated step (p_mean_variance included) equals the reference's bit for bit where the restated denoiser
    does (MDM_UNET), and otherwise agrees within the tolerance oracle/make_golden.py uses for the transformer forward.
The whole 50-step inversion is also run as a float64 chain of the restatement; how far the fp32 reference ends from it
is stored (DESIGN.md section 2).  All cases on ddim50, B = 2.
"""
from __future__ import annotations

import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import condmdi_oracle as O  # noqa: E402
from oracle import ddim_reverse_oracle as R  # noqa: E402
from oracle import reference_harness as RH  # noqa: E402
from oracle.golden_io import save_golden  # noqa: E402
from oracle.make_golden import GOLDEN, close, ref_model_with  # noqa: E402

B, D, L = 2, 263, 196
SINGLE_T = (0, 1, 10, 48, 49)  # t = 49: alphas_cumprod_next = 0
# fixtures kept (each B = 2 tensor is 0.4 MB): single steps per model, and iterations of the whole inversion
KEEP_T = {"nocond": SINGLE_T, "text": (0, 49), "cfg": (0, 10, 49)}
WHOLE_KEEP = (0, 1, 25, 49)  # states after these iterations (49 = the end); pred_xstart at the first and the last


def golden_ddim_reverse():
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
    tab = O.make_tables("ddim50")
    assert np.array_equal(d50.alphas_cumprod_next, R.alphas_cumprod_next(tab))

    def ref_step(model, kwargs, x_, t):
        with torch.no_grad():
            r = d50.ddim_reverse_sample(model, x_, torch.tensor([t] * B), clip_denoised=False, model_kwargs=kwargs)
        return {"sample": r["sample"].detach(), "pred_xstart": r["pred_xstart"].detach()}

    def check(r, x_, t, o, tol, what):
        """r: the reference's step from x_ at t; o: the restatement's"""
        upd = R.reverse_update(tab, x_, torch.tensor([t] * B), r["pred_xstart"])
        assert torch.equal(upd, r["sample"]), f"{what}: the restated update differs from the reference's"
        exact = torch.equal(o["sample"], r["sample"]) and torch.equal(o["pred_xstart"], r["pred_xstart"])
        print(f"  {what}: restated step == reference bit for bit: {exact}")
        if tol == 0:
            assert exact, what
        close(r["pred_xstart"], o["pred_xstart"], tol, f"{what} pred_xstart")
        close(r["sample"], o["sample"], tol * 10 if t == 0 else tol, f"{what} sample")  # t = 0 amplifies ~6x

    ytext = {"text": ["a", "b"]}
    ycfg = {"text": ["a", "b"], "text_scale": scale}
    cases = [("nocond", m, {"y": {}}, sd, O.Conditioning()),
             ("text", mt, {"y": ytext}, sdt, O.Conditioning(cond_emb=cond)),
             ("cfg", cfgm, {"y": ycfg}, sdt, O.Conditioning(cond_emb=cond, cfg=True, text_scale=scale))]
    for name, model, kw, sd_, c in cases:
        print(f"ddim_reverse_sample, transformer {name}, single steps at t = {SINGLE_T}")
        for t in SINGLE_T:
            r = ref_step(model, kw, x, t)
            o = R.ddim_reverse_sample(sd_, tab, x, torch.tensor([t] * B), c)
            check(r, x, t, o, 5e-5, f"{name} t={t}")
            if t in KEEP_T[name]:
                out[f"{name}.t{t}.sample"] = r["sample"].numpy()
                out[f"{name}.t{t}.pred_xstart"] = r["pred_xstart"].numpy()

    print("whole ddim50 inversion, transformer no_cond, teacher-forced per step")
    states = [x]
    for t in range(50):
        r = ref_step(m, {"y": {}}, states[-1], t)
        o = R.ddim_reverse_sample(sd, tab, states[-1], torch.tensor([t] * B), O.Conditioning())
        check(r, states[-1], t, o, 2e-4, f"whole t={t}")  # the states grow: the gate of the ddim50 loop above
        states.append(r["sample"])
        if t in WHOLE_KEEP:
            out[f"whole.k{t}.sample"] = r["sample"].numpy()
        if t in (0, 49):
            out[f"whole.k{t}.pred_xstart"] = r["pred_xstart"].numpy()
    o32 = R.ddim_reverse_sample_loop(sd, tab, x, O.Conditioning())
    sd64 = {k: v.double() for k, v in sd.items()}
    o64 = R.ddim_reverse_sample_loop(sd64, tab, x.double(), O.Conditioning())
    end = states[-1]
    e_ro, e_r64 = (end - o32).abs().max().item(), (end.double() - o64).abs().max().item()
    print(f"  end: |ref32 - oracle32| = {e_ro:.3e}  |ref32 - f64| = {e_r64:.3e}  max|x_T| = {end.abs().max().item():.3f}")
    out["whole.ref_err_vs_f64"] = np.array([e_r64, (end.double() - o64).abs().mean().item()])
    out["whole.oracle32_vs_ref32"] = np.array([e_ro])

    print("CFG 2.5 + imputation (stop_imputation_at = 1), t = 0, 1, 2")
    ykw = {"text": ["a", "b"], "text_scale": scale, "mask": y_mask, "lengths": lengths, "imputate": 1,
           "stop_imputation_at": 1, "replacement_distribution": "conditional", "inpainted_motion": x_obs,
           "inpainting_mask": kf_mask}
    c = O.Conditioning(cond_emb=cond, cfg=True, text_scale=scale, y_mask=y_mask, imputate=True, stop_imputation_at=1,
                       inpainted_motion=x_obs, inpainting_mask=kf_mask)
    xs = x
    for t in range(3):
        r = ref_step(cfgm, {"y": ykw}, xs, t)
        o = R.ddim_reverse_sample(sdt, tab, xs, torch.tensor([t] * B), c)
        check(r, xs, t, o, 1e-4, f"cfg+impute t={t}")
        out[f"cfg_impute.t{t}.sample"] = r["sample"].numpy()
        if t >= 1:  # imputing
            out[f"cfg_impute.t{t}.pred_xstart"] = r["pred_xstart"].numpy()
        xs = r["sample"]

    print("CFG + imputation + reconstruction guidance (w = 20), t = 10, 11")
    ykw2 = dict(ykw)
    ykw2.update(reconstruction_guidance=True, reconstruction_weight=20.0, gradient_schedule=None, diffusion_steps=1000,
                stop_recguidance_at=0)
    c2 = O.Conditioning(cond_emb=cond, cfg=True, text_scale=scale, y_mask=y_mask, imputate=True, stop_imputation_at=1,
                        inpainted_motion=x_obs, inpainting_mask=kf_mask, reconstruction_guidance=True,
                        reconstruction_weight=20.0)
    xs = x
    for t in (10, 11):
        r = ref_step(cfgm, {"y": ykw2}, xs, t)
        o = R.ddim_reverse_sample(sdt, tab, xs, torch.tensor([t] * B), c2)
        check(r, xs, t, o, 2e-4, f"guided t={t}")
        out[f"guided.t{t}.sample"] = r["sample"].numpy()
        out[f"guided.t{t}.pred_xstart"] = r["pred_xstart"].numpy()
        xs = r["sample"]

    print("keyframe-conditioned MDM_UNET xl, CFG: single steps at t = 0, 49 and a 4-step segment t = 20..23")
    sdu = O.random_unet_state_dict(seed=11, text=True)
    mu = RH.build_reference_unet(text=True)
    missing, unexpected = mu.load_state_dict(sdu, strict=False)
    assert not missing and not unexpected, (missing, unexpected)
    mu._synthetic_text_emb = cond
    cfgu = ref.cfg_sampler.ClassifierFreeSampleModel(mu)
    kw = {"y": {"text": ["a", "b"], "text_scale": scale, "mask": y_mask, "lengths": lengths}, "obs_x0": x_obs, "obs_mask": kf_mask}
    cu = O.Conditioning(cond_emb=cond, cfg=True, text_scale=scale, obs_x0=x_obs, obs_mask=kf_mask)
    for t in (0, 49):
        r = ref_step(cfgu, kw, x, t)
        o = R.ddim_reverse_sample(sdu, tab, x, torch.tensor([t] * B), cu)
        check(r, x, t, o, 0, f"unet t={t}")
        out[f"unet.t{t}.sample"] = r["sample"].numpy()
        out[f"unet.t{t}.pred_xstart"] = r["pred_xstart"].numpy()
    xs = x
    for t in range(20, 24):
        r = ref_step(cfgu, kw, xs, t)
        o = R.ddim_reverse_sample(sdu, tab, xs, torch.tensor([t] * B), cu)
        check(r, xs, t, o, 0, f"unet segment t={t}")
        xs = r["sample"]
    out["unet.seg20_24.sample"] = xs.numpy()
    save_golden(GOLDEN, "ddim_reverse", **out)


def main():
    if not RH.available():
        raise SystemExit("the reference tree is required to (re)generate golden vectors")
    os.makedirs(GOLDEN, exist_ok=True)
    torch.set_num_threads(os.cpu_count() or 1)
    golden_ddim_reverse()
    for f in sorted(os.listdir(GOLDEN)):
        if f.startswith("ddim_reverse."):
            print(f, os.path.getsize(os.path.join(GOLDEN, f)) // 1024, "KiB")


if __name__ == "__main__":
    main()

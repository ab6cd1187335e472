"""GPU: the MDM_UNET denoiser (the architecture of the published CondMDI checkpoints; SURVEY.md 8f-4) and the keyframe
INPUT conditioning it consumes (8f-1), behind the same engine / sampler / C ABI as the transformer.

  * tests/golden/unet.npz: outputs of the UNMODIFIED reference `MDM_UNET` (configs/model.py `motion_unet_adagn_xl`: dim 512,
    dim_mults (2,2,2,2), AdaGN, keyframe-conditioned, text) -- one evaluation, the CFG-wrapped evaluation, p_sample_loop steps
  * the CPU oracle (bit-identical to the reference on those fixtures, oracle/make_golden.py::golden_unet) at other shapes

Gate: rtol 1e-3 / atol 1e-4.
"""
import os

import numpy as np
import pytest
import torch

import condmdi_b200 as C
from oracle import condmdi_oracle as O
from oracle.golden_io import load_golden

pytestmark = pytest.mark.gpu
GATE = dict(rtol=1e-3, atol=1e-4)
B, D, L = 2, 263, 196
DEV = "cuda:0"


@pytest.fixture(scope="module")
def gold(golden_dir):
    return load_golden(golden_dir, "unet")


@pytest.fixture(scope="module")
def gi():
    return O.golden_inputs()


@pytest.fixture(scope="module")
def xl(gi):
    sd = O.random_unet_state_dict(seed=11, text=True)
    m = C.MDM_UNET(keyframe_conditioned=True, cond_mode="text", cond_mask_prob=0.1)
    missing, unexpected = m.load_state_dict(sd, strict=False)
    assert not missing and not unexpected
    m = m.to(DEV)
    table = {"a": gi["cond"][0].to(DEV), "b": gi["cond"][1].to(DEV)}
    m.encode_text = lambda texts: torch.stack([table[t] for t in texts])
    return m, sd


def close(a, b, what=""):
    a, b = torch.as_tensor(a).cpu().float(), torch.as_tensor(b).cpu().float()
    err = (a - b).abs()
    print(f"[{what}] max_abs={err.max():.3e} mean_abs={err.mean():.3e}")
    return torch.allclose(a, b, **GATE)


def test_unet_forward_vs_reference_golden(xl, gi, gold):
    m, sd = xl
    x, xo, kf = gi["x"].to(DEV), gi["x_obs"].to(DEV), gi["kf_mask"].to(DEV)
    t = torch.tensor(gold["fwd.t"]).to(DEV)        # per-sample timesteps [999, 37]
    got = m(x, t, y={"text": ["a", "b"]}, obs_x0=xo, obs_mask=kf)
    assert got.shape == (B, D, 1, L) and got.dtype == torch.float32 and got.is_cuda
    assert close(got, gold["fwd.out"], "unet forward (text, keyframes) vs reference")
    assert close(m(x, t, y={"text": ["a", "b"], "uncond": True}, obs_x0=xo, obs_mask=kf), gold["fwd_uncond.out"], "unet uncond")
    w = C.ClassifierFreeSampleModel(m)
    y = {"text": ["a", "b"], "text_scale": gi["text_scale"].to(DEV)}
    got = w(x, torch.tensor([500, 500]).to(DEV), y=y, obs_x0=xo, obs_mask=kf)
    assert close(got, gold["fwd_cfg.out"], "unet cfg forward vs reference")
    with pytest.raises(AssertionError):           # mdm_unet.py:775
        m(x, t, y={"text": ["a", "b"]}, obs_x0=xo)


def test_unet_sampling_loops_vs_reference_golden(xl, gi, gold):
    """p_sample_loop with the keyframes as top-level obs_x0 / obs_mask model_kwargs (sample/conditional_synthesis.py:159-162)."""
    m, sd = xl
    w = C.ClassifierFreeSampleModel(m)
    d = C.create_gaussian_diffusion()
    d.noise_tape = gi["tape"].to(DEV)
    xo, kf = gi["x_obs"].to(DEV), gi["kf_mask"].to(DEV)
    kw = {"y": {"text": ["a", "b"], "text_scale": gi["text_scale"].to(DEV), "mask": gi["y_mask"].to(DEV), "lengths": gi["lengths"]},
          "obs_x0": xo, "obs_mask": kf}
    outs = []
    for k, o in enumerate(d.p_sample_loop_progressive(w, (B, D, 1, L), model_kwargs=kw)):
        outs.append(o)
        if k == 2:
            break
    assert close(outs[-1]["sample"], gold["ddpm3.sample"], "unet 3 steps from t=999: sample")
    assert close(outs[-1]["pred_xstart"], gold["ddpm3.pred_xstart"], "unet 3 steps: pred_xstart")
    got = d.p_sample_loop(w, (B, D, 1, L), model_kwargs=kw, skip_timesteps=996, init_image=xo)
    assert close(got, gold["tail4.sample"], "unet 4-step tail vs reference")
    # reconstruction guidance needs the denoiser's input-VJP, which exists for the transformer only: a clear error
    kw2 = {"y": dict(kw["y"], reconstruction_guidance=True, reconstruction_weight=20.0, gradient_schedule=None, diffusion_steps=1000,
                     stop_recguidance_at=0, inpainted_motion=xo, inpainting_mask=kf), "obs_x0": xo, "obs_mask": kf}
    with pytest.raises(RuntimeError, match="transformer"):
        d.p_sample_loop(w, (B, D, 1, L), model_kwargs=kw2, skip_timesteps=998)


@pytest.mark.parametrize("mults,kf_cond", [((1, 1), True), ((1, 1, 1), False), ((2, 2), True)])
def test_unet_other_geometries_vs_oracle(gi, mults, kf_cond):
    """2- and 3-level UNets, 512 / 1024 channels, with and without keyframe input conditioning; unconditional model."""
    sd = O.random_unet_state_dict(seed=3, mults=mults, keyframe_conditioned=kf_cond)
    m = C.MDM_UNET(dim_mults=mults, keyframe_conditioned=kf_cond)
    assert not any(m.load_state_dict(sd, strict=False))
    m = m.to(DEV)
    t = torch.tensor([41, 41])
    xo, kf = (gi["x_obs"], gi["kf_mask"]) if kf_cond else (None, None)
    got = m(gi["x"].to(DEV), t.to(DEV), y={}, obs_x0=None if xo is None else xo.to(DEV), obs_mask=None if kf is None else kf.to(DEV))
    assert close(got, O.unet_forward(sd, gi["x"], t, None, False, xo, kf), f"unet {mults} kf={kf_cond} vs oracle")


def test_unet_b64_loop_with_imputation_vs_oracle():
    """B = 64 (the BASELINE batch): DDIM tail with keyframe input conditioning AND imputation, 2-level UNet, vs the oracle."""
    Bf = 64
    g = torch.Generator().manual_seed(12)
    sd = O.random_unet_state_dict(seed=5, mults=(1, 1))
    m = C.MDM_UNET(dim_mults=(1, 1), keyframe_conditioned=True)
    m.load_state_dict(sd, strict=False)
    m = m.to(DEV)
    x_obs = torch.randn(Bf, D, 1, L, generator=g)
    lengths = torch.randint(20, 197, (Bf,), generator=g)
    kf = C.get_keyframes_mask(x_obs, lengths, "benchmark_sparse", trans_length=5)
    y_mask = (torch.arange(L)[None] < lengths[:, None]).view(Bf, 1, 1, L)
    tape = torch.randn(5, Bf, D, 1, L, generator=g)
    d = C.create_gaussian_diffusion(timestep_respacing="ddim50")
    d.noise_tape = tape.to(DEV)
    y = {"mask": y_mask.to(DEV), "imputate": 1, "stop_imputation_at": 1, "replacement_distribution": "conditional",
         "inpainted_motion": x_obs.to(DEV), "inpainting_mask": kf.to(DEV)}
    got = d.ddim_sample_loop(m, (Bf, D, 1, L), model_kwargs={"y": y, "obs_x0": x_obs.to(DEV), "obs_mask": kf.to(DEV)},
                             skip_timesteps=46, init_image=x_obs.to(DEV))
    c = O.Conditioning(y_mask=y_mask, imputate=True, stop_imputation_at=1, inpainted_motion=x_obs, inpainting_mask=kf, obs_x0=x_obs,
                       obs_mask=kf)
    want = O.sample_loop(sd, O.make_tables("ddim50"), (Bf, D, 1, L), c, tape, "ddim", skip_timesteps=46, init_image=x_obs)
    assert close(got, want, "unet B=64 ddim tail + imputation vs oracle")


def test_unet_drop_in_for_a_foreign_module(gi):
    """`resolve_model` recognises an MDM_UNET by its state-dict keys: a module this package has never seen (plain nested
    nn.Module containers under the reference's keys, reference attribute names) goes through `accelerate()`-style sampling."""
    sd = O.random_unet_state_dict(seed=9, mults=(1, 1))
    foreign = torch.nn.Module()
    for key, t in sd.items():
        mod, parts = foreign, key.split(".")
        for part in parts[:-1]:
            if part not in mod._modules:
                mod.add_module(part, torch.nn.Module())
            mod = mod._modules[part]
        if parts[-1] == "pe":
            if "pe" not in mod._buffers:
                mod.register_buffer("pe", t.clone())
        else:
            mod.register_parameter(parts[-1], torch.nn.Parameter(t.clone(), requires_grad=False))
    foreign.arch, foreign.cond_mode, foreign.cond_mask_prob, foreign.keyframe_conditioned = "unet", "no_cond", 0.0, True
    foreign.njoints, foreign.nfeats = D, 1
    foreign = foreign.to(DEV)
    inner, is_cfg = C.resolve_model(foreign)
    assert inner is foreign and not is_cfg and hasattr(foreign, "engine_for")
    d = C.create_gaussian_diffusion()
    d.noise_tape = gi["tape"].to(DEV)
    xo, kf = gi["x_obs"].to(DEV), gi["kf_mask"].to(DEV)
    got = d.p_sample_loop(foreign, (B, D, 1, L), model_kwargs={"y": {}, "obs_x0": xo, "obs_mask": kf}, skip_timesteps=996)
    c = O.Conditioning(obs_x0=gi["x_obs"], obs_mask=gi["kf_mask"])
    want = O.sample_loop(sd, O.make_tables(""), (B, D, 1, L), c, gi["tape"], "ddpm", skip_timesteps=996)
    assert close(got, want, "foreign UNet module through the sampler vs oracle")

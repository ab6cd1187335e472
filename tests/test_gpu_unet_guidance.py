"""GPU: reconstruction guidance on MDM_UNET at CMDI_PRECISION_FP16 -- the UNet's input-VJP in the arithmetic autograd uses
after the reference's autocast forward (DESIGN.md section 6).

  A = the oracle's unet_forward on CUDA tensors inside torch.autocast("cuda", torch.float16), its gradient taken by
      torch.autograd.grad outside the autocast region, as gaussian_diffusion.py:388-425 does
  F = the same in exact fp32

Gates as test_gpu_unet_fp16.py, in max and mean of the absolute difference: |engine - A| <= track |A - F| and
|engine - F| <= 2 |A - F|; every ratio is printed.  A CFG evaluation is checked as its two pass gradients (each seeded
with the fp32 combine's s G and G - s G), which the step kernel adds.
"""
import contextlib

import pytest
import torch

import condmdi_b200 as C
from oracle import condmdi_oracle as O
from oracle import plms_oracle as P

pytestmark = pytest.mark.gpu
D, L = 263, 196
DEV = "cuda:0"
FP16 = C.PRECISION_FP16
UNET_FORWARD = O.unet_forward


@contextlib.contextmanager
def exact_fp32():
    saved = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    try:
        yield
    finally:
        torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = saved


def ctx_of(autocast):
    return torch.autocast("cuda", dtype=torch.float16) if autocast else exact_fp32()


def gate(got, a, f, what, track=1.0):
    got, a, f = got.double().cpu(), a.double().cpu(), f.double().cpu()
    e_a, a_f, e_f = (got - a).abs(), (a - f).abs(), (got - f).abs()
    r = {"max|E-A|/max|A-F|": (e_a.max() / a_f.max()).item(), "mean|E-A|/mean|A-F|": (e_a.mean() / a_f.mean()).item(),
         "max|E-F|/max|A-F|": (e_f.max() / a_f.max()).item(), "mean|E-F|/mean|A-F|": (e_f.mean() / a_f.mean()).item()}
    print(f"[{what}] |A-F| max={a_f.max():.3e} mean={a_f.mean():.3e} |A| max={a.abs().max():.3e}  "
          + "  ".join(f"{k}={v:.3f}" for k, v in r.items()))
    assert a_f.max() > 0
    assert r["max|E-A|/max|A-F|"] <= track and r["mean|E-A|/mean|A-F|"] <= track, what
    assert r["max|E-F|/max|A-F|"] <= 2.0 and r["mean|E-F|/mean|A-F|"] <= 2.0, what


def module(mults=(2, 2, 2, 2), kf_cond=True, text=True, seed=11):
    sd = O.random_unet_state_dict(seed=seed, mults=mults, keyframe_conditioned=kf_cond, text=text)
    kw = {"cond_mode": "text", "cond_mask_prob": 0.1} if text else {}
    m = C.MDM_UNET(dim_mults=mults, keyframe_conditioned=kf_cond, **kw)
    assert not any(m.load_state_dict(sd, strict=False))
    return m.to(DEV), sd


def inputs(B, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, D, 1, L, generator=g)
    xo = torch.randn(B, D, 1, L, generator=g)
    lengths = torch.randint(40, L + 1, (B,), generator=g)
    kf = C.get_keyframes_mask(xo, lengths, "benchmark_sparse", trans_length=5)
    cond = torch.randn(B, 512, generator=g)
    scale = torch.full((B,), 2.5)
    return x, xo, kf, cond, scale


def oracle_vjp(sdd, x, t, xo, M, cond=None, uncond=False, obs=None, kf=None, scale=None, autocast=True):
    """The pass gradients of sum((xo - x0_hat)^2 * M) w.r.t. x, autograd after a forward under autocast (or fp32)."""
    dev = lambda v: None if v is None else v.to(DEV)  # noqa: E731
    x, xo, M, cond, obs, kf = dev(x), dev(xo), dev(M), dev(cond), dev(obs), dev(kf)
    tt = torch.full((x.shape[0],), int(t), device=DEV)
    z = x.detach().requires_grad_(True)
    with ctx_of(autocast):
        outs = [UNET_FORWARD(sdd, z, tt, cond, uncond, obs, kf)]
        if scale is not None:
            outs.append(UNET_FORWARD(sdd, z, tt, cond, True, obs, kf))
    with ctx_of(False):
        hat = outs[0] if scale is None else outs[1] + (scale.to(DEV).view(-1, 1, 1, 1) * (outs[0] - outs[1]))
        loss = ((xo - hat).square() * M).sum()
        seeds = torch.autograd.grad(loss, outs, retain_graph=True)
        return torch.stack([torch.autograd.grad(o, z, s_, retain_graph=True)[0] for o, s_ in zip(outs, seeds)])


VJP_CASES = [
    # (name, B, mults, kf_cond, text, mode)
    ("xl-text", 2, (2, 2, 2, 2), True, True, "text"),
    ("xl-uncond", 2, (2, 2, 2, 2), True, True, "uncond"),
    ("xl-cfg", 2, (2, 2, 2, 2), True, True, "cfg"),
    ("xl-cfg-B64", 64, (2, 2, 2, 2), True, True, "cfg"),
    ("xl-nokf-cfg", 2, (2, 2, 2, 2), False, True, "cfg"),
    ("11-kf", 2, (1, 1), True, False, "plain"),
    ("11-nokf", 2, (1, 1), False, False, "plain"),
    ("111-kf", 2, (1, 1, 1), True, False, "plain"),
    ("111-nokf", 2, (1, 1, 1), False, False, "plain"),
]


@pytest.mark.parametrize("name,B,mults,kf_cond,text,mode", VJP_CASES, ids=[c[0] for c in VJP_CASES])
def test_input_vjp(name, B, mults, kf_cond, text, mode):
    m, sd = module(mults, kf_cond, text)
    sdd = {k: v.to(DEV) for k, v in sd.items()}
    x, xo, kf, cond, scale = inputs(B, seed=B + len(mults))
    obs, okf = (xo, kf) if kf_cond else (None, None)
    kw = {}
    if text:
        kw["cond"] = cond
    if mode == "uncond":
        kw["uncond"] = True
    cfg = mode == "cfg"
    eng = m.engine_for(DEV, max_batch=B, precision=FP16, nframes=L)
    for t in (500, 30):
        got = eng.test_input_vjp(x, t, xo, kf, cond_emb=kw.get("cond"), uncond=kw.get("uncond", False), cfg=cfg,
                                 text_scale=scale if cfg else None, obs_x0=obs, obs_mask=okf)
        a = oracle_vjp(sdd, x, t, xo, kf, obs=obs, kf=okf, scale=scale if cfg else None, **kw)
        f = oracle_vjp(sdd, x, t, xo, kf, obs=obs, kf=okf, scale=scale if cfg else None, autocast=False, **kw)
        assert got.shape == a.shape
        for k, what in enumerate(["cond", "uncond"][: got.shape[0]]):
            gate(got[k], a[k], f[k], f"vjp {name} t={t} {what} pass")


def test_bf16x3_unet_still_refuses_guidance():
    m, _ = module((1, 1), True, False, seed=3)
    x, xo, kf, _, _ = inputs(2, seed=1)
    eng = m.engine_for(DEV, max_batch=2, nframes=L)
    with pytest.raises(RuntimeError, match="transformer"):
        eng.test_input_vjp(x, 500, xo, kf, obs_x0=xo, obs_mask=kf)


# ---------------------------------------------------------------------------------------------------------------------
# loops against the oracle sampled with its model calls on the GPU under autocast (A) / in fp32 (F)
# ---------------------------------------------------------------------------------------------------------------------
def oracle_loop(sd, run):
    sdd = {k: v.to(DEV) for k, v in sd.items()}
    want = {}
    try:
        for name, ac in (("A", True), ("F", False)):
            def gpu_forward(sd_, x, t, cond_emb=None, uncond=False, obs_x0=None, obs_mask=None, _ac=ac):
                dev = lambda v: None if v is None else v.to(DEV)  # noqa: E731
                with ctx_of(_ac):
                    out = UNET_FORWARD(sdd, dev(x), dev(t), dev(cond_emb), uncond, dev(obs_x0), dev(obs_mask))
                return out.float().cpu()
            O.unet_forward = gpu_forward
            want[name] = run()
    finally:
        O.unet_forward = UNET_FORWARD
    return want["A"], want["F"]


def setup(B, seed, text=True):
    m, sd = module(text=text)
    w = C.ClassifierFreeSampleModel(m)
    x_obs, _, kf, cond, scale = inputs(B, seed)
    g = torch.Generator().manual_seed(seed + 1)
    lengths = torch.randint(40, L + 1, (B,), generator=g)
    y_mask = (torch.arange(L)[None] < lengths[:, None]).view(B, 1, 1, L)
    table = {str(i): cond[i].to(DEV) for i in range(B)}
    m.encode_text = lambda texts: torch.stack([table[s] for s in texts])
    y = {"text": [str(i) for i in range(B)], "text_scale": scale.to(DEV), "mask": y_mask.to(DEV),
         "inpainted_motion": x_obs.to(DEV), "inpainting_mask": kf.to(DEV), "reconstruction_guidance": True,
         "reconstruction_weight": 20.0, "gradient_schedule": None, "diffusion_steps": 1000, "stop_recguidance_at": 0}
    c = O.Conditioning(cond_emb=cond, cfg=True, text_scale=scale, y_mask=y_mask, inpainted_motion=x_obs, inpainting_mask=kf,
                       obs_x0=x_obs, obs_mask=kf, reconstruction_guidance=True, reconstruction_weight=20.0)
    return m, w, sd, x_obs, kf, y, c, g


def test_ddpm_tail_cfg_imputation_guidance_b2():
    B = 2
    m, w, sd, x_obs, kf, y, c, g = setup(B, seed=21)
    y.update(imputate=1, stop_imputation_at=1, replacement_distribution="conditional")
    c.imputate, c.stop_imputation_at = True, 1
    tape = torch.randn(5, B, D, 1, L, generator=g)
    d = C.create_gaussian_diffusion()
    d.precision = FP16
    d.noise_tape = tape.to(DEV)
    kw = {"y": y, "obs_x0": x_obs.to(DEV), "obs_mask": kf.to(DEV)}
    got = d.p_sample_loop(w, (B, D, 1, L), model_kwargs=kw, skip_timesteps=996, init_image=x_obs.to(DEV))
    a, f = oracle_loop(sd, lambda: O.sample_loop(sd, O.make_tables(""), (B, D, 1, L), c, tape, "ddpm", skip_timesteps=996,
                                                init_image=x_obs))
    gate(got, a, f, "B=2 ddpm 4-step tail, cfg + imputation + guidance w=20", track=1.5)


def test_ddim50_tail_b64_stop_recguidance_inside():
    B = 64
    m, w, sd, x_obs, kf, y, c, g = setup(B, seed=22)
    y.update(stop_recguidance_at=3, gradient_schedule="exponential")
    c.stop_recguidance_at, c.gradient_schedule = 3, "exponential"
    tape = torch.randn(7, B, D, 1, L, generator=g)
    d = C.create_gaussian_diffusion(timestep_respacing="ddim50")
    d.precision = FP16
    d.noise_tape = tape.to(DEV)
    kw = {"y": y, "obs_x0": x_obs.to(DEV), "obs_mask": kf.to(DEV)}
    got = d.ddim_sample_loop(w, (B, D, 1, L), model_kwargs=kw, skip_timesteps=44, init_image=x_obs.to(DEV))
    a, f = oracle_loop(sd, lambda: O.sample_loop(sd, O.make_tables("ddim50"), (B, D, 1, L), c, tape, "ddim", skip_timesteps=44,
                                                init_image=x_obs))
    gate(got, a, f, "B=64 ddim50 6-step tail, cfg + guidance (stop_recguidance_at=3, exponential)", track=1.5)


def test_plms_order2_guided_first_step():
    B = 2
    m, w, sd, x_obs, kf, y, c, g = setup(B, seed=23)
    y.update(stop_recguidance_at=46)
    c.stop_recguidance_at = 46
    tape = torch.randn(1, B, D, 1, L, generator=g)
    d = C.create_gaussian_diffusion(timestep_respacing="ddim50")
    d.precision = FP16
    d.noise_tape = tape.to(DEV)
    kw = {"y": y, "obs_x0": x_obs.to(DEV), "obs_mask": kf.to(DEV)}
    res = []
    for k, o in enumerate(d.plms_sample_loop_progressive(w, (B, D, 1, L), model_kwargs=kw, skip_timesteps=2, order=2,
                                                          init_image=x_obs.to(DEV))):
        res.append(o["sample"])
        if k == 3:
            break
    # the first step evaluates at t = 47 and t = 46, both guided; the later steps at 46 (guided), 45 and 44
    a, f = oracle_loop(sd, lambda: P.plms_sample_loop(sd, O.make_tables("ddim50"), (B, D, 1, L), c, tape, 2, skip_timesteps=2,
                                                     init_image=x_obs, max_steps=4))
    gate(res[-1], a, f, "B=2 plms order 2, 4 steps, guided first step (cfg + guidance)", track=1.5)


# ---------------------------------------------------------------------------------------------------------------------
# bit-for-bit properties
# ---------------------------------------------------------------------------------------------------------------------
def engine_args(B, seed):
    m, w, sd, x_obs, kf, y, c, g = setup(B, seed)
    eng = m.engine_for(DEV, max_batch=B, precision=FP16, nframes=L)
    d = C.create_gaussian_diffusion(timestep_respacing="ddim50")
    eng.set_schedule(d.betas, d.timestep_map)
    coef = [1.0] * d.num_timesteps
    kw = dict(batch=B, sampler=C.capi.SAMPLER_DDIM, skip_timesteps=40, seed=5, cond_emb=torch.randn(B, 512, generator=g).to(DEV),
              cfg=True, text_scale=torch.full((B,), 2.5, device=DEV), inpainted_motion=x_obs.to(DEV), inpainting_mask=kf.to(DEV),
              recon_guidance=True, stop_recguidance_at=4, recon_coef=coef, obs_x0=x_obs.to(DEV), obs_mask=kf.to(DEV))
    return m, eng, kw


def test_graph_replay_equals_direct_launches_and_guiding_leaves_unguided_loops_alone():
    B = 2
    m, eng, kw = engine_args(B, seed=31)
    direct = eng.sample(use_graph=False, **kw)["sample"]
    graph = eng.sample(use_graph=True, **kw)["sample"]
    assert torch.equal(direct, graph)
    plain = {k: v for k, v in kw.items() if k not in ("recon_guidance", "stop_recguidance_at", "recon_coef")}
    before = eng.launch_count
    after_guided = eng.sample(**plain)["sample"]
    per_loop = eng.launch_count - before
    fresh_m, fresh, _ = engine_args(B, seed=31)
    assert fresh is not eng
    alone = fresh.sample(**plain)["sample"]  # (its first call also builds the timestep-embedding table: 5 launches)
    assert torch.equal(after_guided, alone)
    f0 = fresh.launch_count
    assert torch.equal(fresh.sample(**plain)["sample"], alone)
    assert fresh.launch_count - f0 == per_loop
    # one more step costs one unguided pass and the step kernel, as before guidance existed: for xl, 82 launches (input and
    # embedding builders, 3 time-MLP GEMMs, 16 blocks of 4 launches + 4 residual convolutions, 3 + 3 resampling convolutions,
    # final_conv's 3)
    b1 = fresh.launch_count
    fresh.sample(**dict(plain, skip_timesteps=39))
    assert fresh.launch_count - b1 - per_loop == 82 + 1


def test_progressive_generator_equals_fused_loop():
    B = 2
    m, w, sd, x_obs, kf, y, c, g = setup(B, seed=41)
    y.update(imputate=1, stop_imputation_at=0, replacement_distribution="conditional", stop_recguidance_at=2)
    tape = torch.randn(5, B, D, 1, L, generator=g)
    d = C.create_gaussian_diffusion(timestep_respacing="ddim50")
    d.precision = FP16
    d.noise_tape = tape.to(DEV)
    kw = {"y": y, "obs_x0": x_obs.to(DEV), "obs_mask": kf.to(DEV)}
    fused = d.ddim_sample_loop(w, (B, D, 1, L), model_kwargs=kw, skip_timesteps=46, init_image=x_obs.to(DEV))
    last = None
    for o in d.ddim_sample_loop_progressive(w, (B, D, 1, L), model_kwargs=kw, skip_timesteps=46, init_image=x_obs.to(DEV)):
        last = o["sample"]
    assert torch.equal(fused, last)

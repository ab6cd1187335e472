"""GPU: DDIM inversion (ddim_reverse_sample, gaussian_diffusion.py:1418-1452, and the loops around it) behind the public API,
against
  (1) tests/golden/ddim_reverse.* -- outputs of the UNMODIFIED reference (oracle/make_golden_ddim_reverse.py), and
  (2) the CPU oracle at B = 2 and B = 64, teacher-forced on the engine's own states at every step,
at rtol 1e-3 / atol 1e-4 per step; the fp16 UNet against the autocast / fp32 oracle runs with the gates of
test_gpu_unet_fp16.py; bit-for-bit identities between the entry points; errors; launch accounting.

Numerics: the reverse ODE amplifies.  Along the state path one step multiplies a perturbation of x_t by
J_t = sqrt(1 - abar_{t+1}) sqrt(1/abar_t) / sqrt(1/abar_t - 1), and a perturbation of x0 by
|sqrt(abar_{t+1}) - sqrt(1 - abar_{t+1}) / sqrt(1/abar_t - 1)|.  The product of the J_t over a whole loop telescopes to
1 / sqrt(1 - abar_0) ~ 1 / sqrt(1/abar_0 - 1) ~ 156 for the cosine schedule.  At t = 0 the x0 factor is ~5.8 on ddim50, so
the t = 0 gate is the per-step gate times that factor (`amp_x0`, computed below from the tables).

The inverted state grows (|x_T| ~ 760 from |x_0| ~ 4.5 with these random weights), and the transformer's bf16x3 operands
carry 16 significant bits of it: the denoiser input and the weights it meets are each represented to 2^-16 relative.  So
x0 predicted from a large state is within atol + rtol |x0| + 2^-15 max|x_t| of the fp32 oracle (`x0_gate`); at
max|x_t| <= 3 that is the plain per-step gate to within 1e-4.  Given x_t, the update is the same fp32 arithmetic in both,
so x_{t+1} carries that x0 term times amp_x0(t), plus a few fp32 roundings of the eps path at J_t max|x_t| (`sample_gate`).
"""
import ctypes

import numpy as np
import pytest
import torch

import condmdi_b200 as C
from oracle import condmdi_oracle as O
from oracle import ddim_reverse_oracle as R
from oracle.golden_io import load_golden
from test_gpu_unet_fp16 import gate as fp16_gate, oracle as fp16_oracle, to_dev, xl_inputs, xl_module
from test_gpu_unet_guidance import gate as guided_gate, oracle_loop, setup as guided_setup

pytestmark = pytest.mark.gpu
RTOL, ATOL = 1e-3, 1e-4
B, D, L = 2, 263, 196
SHAPE = (B, D, 1, L)
DEV = "cuda:0"
TAB = O.make_tables("ddim50")


@pytest.fixture(scope="module")
def gold(golden_dir):
    return load_golden(golden_dir, "ddim_reverse")


@pytest.fixture(scope="module")
def gi():
    return O.golden_inputs()


def _model(text, gi=None):
    sd = O.random_state_dict(seed=7, text=text)
    m = C.MDM(cond_mode="text" if text else "no_cond", cond_mask_prob=0.1)
    missing, unexpected = m.load_state_dict(sd, strict=False)
    assert not missing and not unexpected
    m = m.to(DEV)
    if text:
        m.encode_text = lambda texts: gi["cond"].to(DEV)
    return m, sd


@pytest.fixture(scope="module")
def plain():
    return _model(False)


@pytest.fixture(scope="module")
def texty(gi):
    return _model(True, gi)


def amp_x0(t):
    """|d x_{t+1} / d x0| of one reverse step (float64 tables): sqrt(abar_next) - sqrt(1 - abar_next) / sqrt(1/abar_t - 1)"""
    an = R.alphas_cumprod_next(TAB)[t]
    return abs(np.sqrt(an) - np.sqrt(1 - an) / TAB.sqrt_recipm1_alphas_cumprod[t])


def j_state(t):
    """|d x_{t+1} / d x_t| along the state path: sqrt(1 - abar_next) sqrt(1/abar_t) / sqrt(1/abar_t - 1)"""
    an = R.alphas_cumprod_next(TAB)[t]
    return np.sqrt(1 - an) * TAB.sqrt_recip_alphas_cumprod[t] / TAB.sqrt_recipm1_alphas_cumprod[t]


def step_gate(got, want, t, what, is_sample):
    """rtol 1e-3 / atol 1e-4; a sample at t = 0 is allowed amp_x0(0) times that (the x0 error it carries is scaled)"""
    got, want = torch.as_tensor(got).cpu().double(), torch.as_tensor(want).cpu().double()
    k = amp_x0(t) if (is_sample and t == 0) else 1.0
    err = (got - want).abs()
    ok = bool((err <= ATOL * k + RTOL * k * want.abs()).all())
    print(f"[{what}] t={t} max_abs={err.max():.3e} max_rel={(err / want.abs().clamp_min(1e-6)).max():.3e} factor={k:.2f}")
    return ok


def x0_gate(got, want, x_t, t, what):
    """the per-step gate for x0 plus the bf16x3 representation of the state the denoiser reads: 2^-15 max|x_t|"""
    got, want = torch.as_tensor(got).cpu().double(), torch.as_tensor(want).cpu().double()
    extra = 2.0 ** -15 * float(x_t.abs().max())
    err = (got - want).abs()
    ok = bool((err <= ATOL + extra + RTOL * want.abs()).all())
    print(f"[{what}] t={t} max|x_t|={float(x_t.abs().max()):.1f} max_abs={err.max():.3e} "
          f"max_abs / (atol + 2^-15 max|x_t|) = {err.max() / (ATOL + extra):.3f}")
    return ok


def sample_gate(got, want, x_t, t, what):
    """step_gate's x_{t+1} gate plus what x0_gate's extra term becomes through the update, amp_x0(t) 2^-15 max|x_t|, and
    four fp32 roundings (2^-21 relative) of the eps path's terms, J_t max|x_t|"""
    got, want = torch.as_tensor(got).cpu().double(), torch.as_tensor(want).cpu().double()
    xm = float(x_t.abs().max())
    k = amp_x0(0) if t == 0 else 1.0
    extra = amp_x0(t) * 2.0 ** -15 * xm + 2.0 ** -21 * j_state(t) * xm
    err = (got - want).abs()
    ok = bool((err <= k * (ATOL + RTOL * want.abs()) + extra).all())
    print(f"[{what}] t={t} max|x_t|={xm:.1f} max_abs={err.max():.3e} max_abs / (atol + extra) = {err.max() / (k * ATOL + extra):.3f}")
    return ok


def test_schedule_amplification_figures():
    assert 5.7 < amp_x0(0) < 5.9
    total = np.prod([j_state(t) for t in range(50)])
    a0 = TAB.alphas_cumprod[0]
    assert abs(total - 1 / np.sqrt(1 - a0)) < 1e-9 * total  # sqrt(1 - abar_50) / sqrt(1 - abar_0), abar_50 = 0
    assert abs(total * TAB.sqrt_recipm1_alphas_cumprod[0] - 1) < 1e-4 and 150 < total < 160


# ------------------------------------------------------------------------------------------------
# the reference's own outputs
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name,ts", [("nocond", (0, 1, 10, 48, 49)), ("text", (0, 49)), ("cfg", (0, 10, 49))])
def test_single_steps_vs_reference_golden(plain, texty, gi, gold, name, ts):
    m = plain[0] if name == "nocond" else texty[0]
    model = C.ClassifierFreeSampleModel(m) if name == "cfg" else m
    y = {"text": ["a", "b"], "text_scale": gi["text_scale"].to(DEV)} if name == "cfg" else ({"text": ["a", "b"]} if name == "text" else {})
    d = C.create_gaussian_diffusion(timestep_respacing="ddim50")
    x = gi["x"].to(DEV)
    for t in ts:
        out = d.ddim_reverse_sample(model, x, torch.tensor([t, t]), model_kwargs={"y": y})
        assert step_gate(out["pred_xstart"], gold[f"{name}.t{t}.pred_xstart"], t, f"{name} pred_xstart", False)
        assert step_gate(out["sample"], gold[f"{name}.t{t}.sample"], t, f"{name} sample", True)


def test_whole_inversion_vs_reference_golden(plain, gi, gold):
    """teacher-forced steps from the reference's states, then the whole loop end to end"""
    m, sd = plain
    d = C.create_gaussian_diffusion(timestep_respacing="ddim50")
    kw = {"y": {}}
    o = d.ddim_reverse_sample(m, gi["x"].to(DEV), [0, 0], model_kwargs=kw)
    assert step_gate(o["pred_xstart"], gold["whole.k0.pred_xstart"], 0, "whole k=0 pred_xstart", False)
    assert step_gate(o["sample"], gold["whole.k0.sample"], 0, "whole k=0 sample", True)
    o = d.ddim_reverse_sample(m, torch.from_numpy(gold["whole.k0.sample"]).to(DEV), [1, 1], model_kwargs=kw)
    assert step_gate(o["sample"], gold["whole.k1.sample"], 1, "whole k=1 sample (from the reference's x_1)", True)
    # end to end.  Bound: each step may add the per-step gate, e_t = atol + rtol |x_{t+1}|, and the later steps scale it
    # by the product of their state factors J_s (the whole product telescopes to ~156); the model path is inside e_t,
    # which is measured teacher-forced.  bound = sum_t e_t prod_{s>t} J_s, |x_{t+1}| taken from the restated loop.
    got = d.ddim_reverse_sample_loop(m, gi["x"].to(DEV), model_kwargs=kw).cpu().double()
    want = torch.from_numpy(gold["whole.k49.sample"]).double()
    mags = [o_["sample"].abs().max().item() for o_ in R.ddim_reverse_sample_loop(sd, TAB, gi["x"], O.Conditioning(), return_all=True)]
    J = [j_state(t) for t in range(50)]
    bound = sum((ATOL + RTOL * mags[t]) * np.prod(J[t + 1:]) for t in range(50))
    err = (got - want).abs().max().item()
    print(f"[whole ddim50 inversion, B=2] max|engine - reference| = {err:.3e} (max|x_T| = {want.abs().max():.1f}), "
          f"bound from the per-step gate = {bound:.3e}, ratio {err / bound:.3f}")
    assert err <= bound


def test_cfg_imputation_and_guidance_vs_reference_golden(texty, gi, gold):
    m, _ = texty
    w = C.ClassifierFreeSampleModel(m)
    d = C.create_gaussian_diffusion(timestep_respacing="ddim50")
    y = {"text": ["a", "b"], "text_scale": gi["text_scale"].to(DEV), "mask": gi["y_mask"].to(DEV), "lengths": gi["lengths"],
         "imputate": 1, "stop_imputation_at": 1, "replacement_distribution": "conditional",
         "inpainted_motion": gi["x_obs"].to(DEV), "inpainting_mask": gi["kf_mask"].to(DEV)}
    x = gi["x"].to(DEV)
    for t in range(3):  # teacher-forced from the reference's states
        o = d.ddim_reverse_sample(w, x, [t, t], model_kwargs={"y": y})
        if t >= 1:
            assert step_gate(o["pred_xstart"], gold[f"cfg_impute.t{t}.pred_xstart"], t, "cfg+impute pred_xstart", False)
        assert step_gate(o["sample"], gold[f"cfg_impute.t{t}.sample"], t, "cfg+impute sample", True)
        x = torch.from_numpy(gold[f"cfg_impute.t{t}.sample"]).to(DEV)
    y.update(reconstruction_guidance=True, reconstruction_weight=20.0, gradient_schedule=None, diffusion_steps=1000,
             stop_recguidance_at=0)
    x = gi["x"].to(DEV)
    for t in (10, 11):
        o = d.ddim_reverse_sample(w, x, [t, t], model_kwargs={"y": y})
        assert step_gate(o["pred_xstart"], gold[f"guided.t{t}.pred_xstart"], t, "guided w=20 pred_xstart", False)
        assert step_gate(o["sample"], gold[f"guided.t{t}.sample"], t, "guided w=20 sample", True)
        x = torch.from_numpy(gold[f"guided.t{t}.sample"]).to(DEV)


def _unet_xl(gi):
    sd = O.random_unet_state_dict(seed=11, text=True)
    m = C.MDM_UNET(keyframe_conditioned=True, cond_mode="text", cond_mask_prob=0.1)
    assert not any(m.load_state_dict(sd, strict=False))
    m = m.to(DEV)
    table = {"a": gi["cond"][0].to(DEV), "b": gi["cond"][1].to(DEV)}
    m.encode_text = lambda texts: torch.stack([table[t] for t in texts])
    xo, kf = gi["x_obs"].to(DEV), gi["kf_mask"].to(DEV)
    kw = {"y": {"text": ["a", "b"], "text_scale": gi["text_scale"].to(DEV), "mask": gi["y_mask"].to(DEV), "lengths": gi["lengths"]},
          "obs_x0": xo, "obs_mask": kf}
    return C.ClassifierFreeSampleModel(m), kw, xo, kf


def test_unet_xl_cfg_keyframes_vs_reference_golden(gi, gold):
    w, kw, xo, kf = _unet_xl(gi)
    d = C.create_gaussian_diffusion(timestep_respacing="ddim50")
    x = gi["x"].to(DEV)
    for t in (0, 49):
        o = d.ddim_reverse_sample(w, x, [t, t], model_kwargs=kw)
        assert step_gate(o["pred_xstart"], gold[f"unet.t{t}.pred_xstart"], t, "unet xl pred_xstart", False)
        assert step_gate(o["sample"], gold[f"unet.t{t}.sample"], t, "unet xl sample", True)
    # 4 steps t = 20..23, each from the engine's previous state, against the reference's segment from the same x
    seg = x
    for t in range(20, 24):
        seg = d.ddim_reverse_sample(w, seg, [t, t], model_kwargs=kw)["sample"]
    assert step_gate(seg, gold["unet.seg20_24.sample"], 23, "unet xl 4-step segment", True)
    # guidance on the bf16x3 UNet keeps its existing error
    y2 = dict(kw["y"], reconstruction_guidance=True, reconstruction_weight=20.0, gradient_schedule=None, diffusion_steps=1000,
              stop_recguidance_at=0, inpainted_motion=xo, inpainting_mask=kf)
    with pytest.raises(RuntimeError, match="transformer"):
        d.ddim_reverse_sample_loop(w, x, model_kwargs={"y": y2, "obs_x0": xo, "obs_mask": kf})


# ------------------------------------------------------------------------------------------------
# teacher-forced over every step of whole inversions, against the oracle on the engine's own states
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("Bn", [2, 64])
def test_every_step_teacher_forced_vs_oracle(plain, Bn):
    m, sd = plain
    g = torch.Generator().manual_seed(31 + Bn)
    x0 = torch.randn(Bn, D, 1, L, generator=g)
    d = C.create_gaussian_diffusion(timestep_respacing="ddim50")
    states, preds = [x0.to(DEV)], []
    for o in d.ddim_reverse_sample_loop_progressive(m, x0.to(DEV), model_kwargs={"y": {}}):
        states.append(o["sample"].clone())
        preds.append(o["pred_xstart"].clone())
    assert len(preds) == 50
    fused = d.ddim_reverse_sample_loop(m, x0.to(DEV), model_kwargs={"y": {}})
    assert torch.equal(fused, states[-1])  # the generator == the fused loop, bit for bit
    bad = []
    for t in range(50):
        o = R.ddim_reverse_sample(sd, TAB, states[t].cpu(), torch.tensor([t] * Bn), O.Conditioning())
        if not x0_gate(preds[t], o["pred_xstart"], states[t], t, f"B={Bn} pred_xstart"):
            bad.append((t, "pred_xstart"))
        if not sample_gate(states[t + 1], o["sample"], states[t], t, f"B={Bn} sample"):
            bad.append((t, "sample"))
    assert not bad, bad


# ------------------------------------------------------------------------------------------------
# fp16 UNet: the A / F gates of test_gpu_unet_fp16.py
# ------------------------------------------------------------------------------------------------
def test_fp16_unet_xl_steps_and_segment():
    Bn = 2
    m, sd = xl_module(Bn)
    w = C.ClassifierFreeSampleModel(m)
    x, xo, kf, cond, _, scale = xl_inputs(Bn, seed=41)
    table = {str(i): cond[i].to(DEV) for i in range(Bn)}
    m.encode_text = lambda texts: torch.stack([table[s] for s in texts])
    d = C.create_gaussian_diffusion(timestep_respacing="ddim50")
    d.precision = C.PRECISION_FP16
    kw = {"y": {"text": [str(i) for i in range(Bn)], "text_scale": scale.to(DEV)}, "obs_x0": xo.to(DEV), "obs_mask": kf.to(DEV)}
    c = O.Conditioning(cond_emb=cond, cfg=True, text_scale=scale, obs_x0=xo, obs_mask=kf)
    sdd = to_dev(sd)
    UF = O.unet_forward
    want = {}
    try:
        for name, autocast in (("A", True), ("F", False)):
            def gpu_forward(sd_, x_, t_, cond_emb=None, uncond=False, obs_x0=None, obs_mask=None, _ac=autocast):
                return fp16_oracle(sdd, x_, t_, cond_emb, uncond, obs_x0, obs_mask, autocast=_ac).cpu()
            O.unet_forward = gpu_forward
            want[name] = {t: R.ddim_reverse_sample(sd, TAB, x, torch.tensor([t] * Bn), c) for t in (0, 10, 49)}
            want[name]["seg"] = R.ddim_reverse_sample_loop(sd, TAB, x, c, t_start=30, max_steps=4)
    finally:
        O.unet_forward = UF
    for t in (0, 10, 49):
        got = d.ddim_reverse_sample(w, x.to(DEV), [t, t], model_kwargs=kw)
        # a CFG output: the 1.5x margin test_gpu_unet_fp16.py gives CFG combines
        fp16_gate(got["pred_xstart"], want["A"][t]["pred_xstart"], want["F"][t]["pred_xstart"], f"fp16 xl cfg t={t} pred_xstart", track=1.5)
        fp16_gate(got["sample"], want["A"][t]["sample"], want["F"][t]["sample"], f"fp16 xl cfg t={t} sample", track=1.5)
    seg = x.to(DEV)
    for t in range(30, 34):
        seg = d.ddim_reverse_sample(w, seg, [t, t], model_kwargs=kw)["sample"]
    fp16_gate(seg, want["A"]["seg"], want["F"]["seg"], "fp16 xl cfg 4-step segment t=30..33", track=1.5)


def test_fp16_unet_guided_steps():
    Bn = 2
    m, w, sd, x_obs, kf, y, c, g = guided_setup(Bn, seed=43)
    x = torch.randn(Bn, D, 1, L, generator=g)
    d = C.create_gaussian_diffusion(timestep_respacing="ddim50")
    d.precision = C.PRECISION_FP16
    kw = {"y": y, "obs_x0": x_obs.to(DEV), "obs_mask": kf.to(DEV)}
    got = d.ddim_reverse_sample(w, x.to(DEV), [12, 12], model_kwargs=kw)
    a, f = oracle_loop(sd, lambda: R.ddim_reverse_sample(sd, TAB, x, torch.tensor([12] * Bn), c))
    guided_gate(got["pred_xstart"], a["pred_xstart"].detach(), f["pred_xstart"].detach(), "fp16 guided t=12 pred_xstart", track=1.5)
    guided_gate(got["sample"], a["sample"].detach(), f["sample"].detach(), "fp16 guided t=12 sample", track=1.5)


# ------------------------------------------------------------------------------------------------
# identities, state, errors, launches
# ------------------------------------------------------------------------------------------------
def test_step_equals_fused_first_step_and_graph_equals_direct(plain, gi):
    m, _ = plain
    d = C.create_gaussian_diffusion(timestep_respacing="ddim50")
    x = gi["x"].to(DEV)
    eng = m.engine_for(torch.device(DEV), max_batch=B)
    one = d.ddim_reverse_sample(m, x, torch.tensor([0, 0]), model_kwargs={"y": {}})
    fused1 = eng.sample(B, sampler=C.capi.SAMPLER_DDIM_REVERSE, num_steps=1, x_T=x, want_pred_xstart=True)
    assert torch.equal(one["sample"], fused1["sample"]) and torch.equal(one["pred_xstart"], fused1["pred_xstart"])
    graph = d.ddim_reverse_sample_loop(m, x, model_kwargs={"y": {}})
    d.use_graph = False
    direct = d.ddim_reverse_sample_loop(m, x, model_kwargs={"y": {}})
    assert torch.equal(graph, direct)
    # partial inversion: skip_timesteps counts the iterations already done, upwards
    part = eng.sample(B, sampler=C.capi.SAMPLER_DDIM_REVERSE, num_steps=3, skip_timesteps=0, x_T=x)["sample"]
    rest = eng.sample(B, sampler=C.capi.SAMPLER_DDIM_REVERSE, skip_timesteps=3, x_T=part)["sample"]
    assert torch.equal(rest, graph)


def test_torch_generator_untouched(plain, gi):
    m, _ = plain
    d = C.create_gaussian_diffusion(timestep_respacing="ddim50")
    torch.manual_seed(9)
    before = torch.cuda.get_rng_state(DEV)
    d.ddim_reverse_sample_loop(m, gi["x"].to(DEV), model_kwargs={"y": {}})
    list(d.ddim_reverse_sample_loop_progressive(m, gi["x"].to(DEV), model_kwargs={"y": {}}))
    d.ddim_reverse_sample(m, gi["x"].to(DEV), [5, 5], model_kwargs={"y": {}})
    torch.cuda.synchronize()
    assert torch.equal(torch.cuda.get_rng_state(DEV), before)


def test_inverting_engine_leaves_other_samplers_alone(gi):
    """DDPM / DDIM / PLMS on an engine that has inverted: the results and launch counts of a fresh engine"""
    tape = gi["tape"][:5].to(DEV)

    def runs(m, invert_first):
        eng = m.engine_for(torch.device(DEV), max_batch=B)
        d = C.create_gaussian_diffusion(timestep_respacing="ddim50")
        d.noise_tape = tape
        d.ddim_sample_loop(m, SHAPE, model_kwargs={"y": {}}, skip_timesteps=48)  # the engine's one-time setup, in both runs
        if invert_first:
            d.ddim_reverse_sample_loop(m, gi["x"].to(DEV), model_kwargs={"y": {}})
        res = []
        for fn, kw in ((d.p_sample_loop, {}), (d.ddim_sample_loop, {}), (d.plms_sample_loop, {"order": 3})):
            n0 = eng.launch_count
            out = fn(m, SHAPE, model_kwargs={"y": {}}, skip_timesteps=46, **kw)
            torch.cuda.synchronize()
            res.append((out, eng.launch_count - n0))
        return res

    inverted = runs(_model(False)[0], True)
    fresh = runs(_model(False)[0], False)
    for (a, na), (b, nb) in zip(inverted, fresh):
        assert torch.equal(a, b) and na == nb


def test_launch_accounting(plain, gi):
    """a reverse step costs a DDIM step's launches: the same passes and one step kernel"""
    m, _ = plain
    eng = m.engine_for(torch.device(DEV), max_batch=B)
    x = gi["x"].to(DEV)

    def launches(**kw):
        n0 = eng.launch_count
        eng.sample(B, x_T=x, **kw)
        torch.cuda.synchronize()
        return eng.launch_count - n0

    rev = {n: launches(sampler=C.capi.SAMPLER_DDIM_REVERSE, num_steps=n) for n in (4, 5)}
    ddim = {n: launches(sampler=C.capi.SAMPLER_DDIM, num_steps=n) for n in (4, 5)}
    assert rev[5] - rev[4] == ddim[5] - ddim[4] > 0
    assert rev[4] == ddim[4]


def test_errors(plain, gi):
    m, _ = plain
    d = C.create_gaussian_diffusion(timestep_respacing="ddim50")
    x = gi["x"].to(DEV)
    with pytest.raises(AssertionError, match="Reverse ODE"):
        d.ddim_reverse_sample(m, x, [0, 0], model_kwargs={"y": {}}, eta=0.3)
    with pytest.raises(NotImplementedError):
        d.ddim_reverse_sample(m, x, torch.tensor([0, 1]), model_kwargs={"y": {}})
    eng = m.engine_for(torch.device(DEV), max_batch=B)
    S = C.capi.SAMPLER_DDIM_REVERSE
    z = torch.zeros(SHAPE, device=DEV)
    for field, kw in (("noise_tape", {"noise_tape": torch.zeros((2,) + SHAPE, device=DEV)}), ("init_image", {"init_image": z}),
                      ("dump_xstart", {"dump_steps": [0]}), ("eta", {"eta": 0.5})):
        with pytest.raises(RuntimeError, match=field):
            eng.sample(B, sampler=S, x_T=x, **kw)
    # the PLMS fields: the Python layer never sends them with this sampler; the ABI refuses them
    for field, value in (("plms_order", 2), ("plms_old_eps_out", z.data_ptr())):
        a = C.capi.SampleArgs(B, S, 0.0, 0, 1, 0, None, x.data_ptr())
        setattr(a, field, value)
        out = torch.empty_like(x)
        with torch.cuda.device(eng.device):
            rc = eng.lib.cmdi_sample(eng._h, ctypes.byref(a), out.data_ptr(), torch.cuda.current_stream(DEV).cuda_stream)
        assert rc != 0 and field.encode() in C.capi.load().cmdi_last_error()
    with pytest.raises(RuntimeError, match="x_T"):
        eng.sample(B, sampler=S)

"""GPU: overlapping windows (GaussianDiffusion.window = Window(frames, overlap)) behind the public API and the C ABI:
  - one window (window_count = 1) == the plain loop bit for bit, for every in-scope sampler, the three noise modes,
    the transformer and the UNet xl, with torch's generator left where the plain loop leaves it;
  - every window covering a frame holds the same bits there after every step (window_out), for every sampler, with CFG,
    imputation and reconstruction guidance;
  - whole ddim20 loops at B = 2 and DDPM / DDIM tails with 64 window rows against oracle/windowed_oracle.py at
    rtol 1e-3 / atol 1e-4 (bf16x3), including per-window prompts, guidance at w = 20, the UNet xl with keyframe input,
    K = 2, K = 4 and a frame covered three times;
  - noise drawn in the global layout in all three modes, generator == fused loop, graph replay == direct launches,
    launches per step == an unwindowed loop at B * K sequences, global outputs, and the errors.
"""
import ctypes

import numpy as np
import pytest
import torch

import condmdi_b200 as C
import test_gpu_dpm_solver as TD
import test_gpu_unet_guidance as TG
from condmdi_b200.diffusion import _torch_stream_args
from oracle import condmdi_oracle as O
from oracle import windowed_oracle as W

pytestmark = pytest.mark.gpu
D = 263
DEV = "cuda:0"
close = TD.close
SAMPLERS = ["p_sample_loop", "ddim_sample_loop", "plms_sample_loop", "dpm_solver_sample_loop", "unipc_sample_loop",
            "dpm_solver_sde_sample_loop"]
ENGINE_SAMPLER = {"p_sample_loop": C.capi.SAMPLER_DDPM, "ddim_sample_loop": C.capi.SAMPLER_DDIM,
                  "plms_sample_loop": C.capi.SAMPLER_PLMS, "dpm_solver_sample_loop": C.capi.SAMPLER_DPM_SOLVER,
                  "unipc_sample_loop": C.capi.SAMPLER_UNIPC, "dpm_solver_sde_sample_loop": C.capi.SAMPLER_DPM_SOLVER_SDE}
STOCHASTIC = {"p_sample_loop", "dpm_solver_sde_sample_loop"}  # one draw per step after x_T


def texts_model(kind, table):
    """The bf16x3 transformer (text) or the keyframe-conditioned UNet xl, with encode_text looking prompts up in `table`."""
    if kind == "unet":
        m, sd = TG.module()
    else:
        sd = O.random_state_dict(seed=7, text=True)
        m = C.MDM(cond_mode="text", cond_mask_prob=0.1)
        assert not any(m.load_state_dict(sd, strict=False))
        m = m.to(DEV)
    m.encode_text = lambda texts: torch.stack([table[t] for t in texts])
    return m, sd


def inputs(B, N, seed):
    g = torch.Generator().manual_seed(seed)
    x_obs = torch.randn(B, D, 1, N, generator=g)
    kf = torch.rand(B, D, 1, N, generator=g) < 0.2
    cond = torch.randn(B, 512, generator=g)
    scale = 0.5 + 2 * torch.rand(B, generator=g)
    return x_obs, kf, cond, scale


def ykw(B, N, x_obs, kf, scale, text, guided=False, unet=False):
    y = {"text": text, "text_scale": scale.to(DEV), "mask": torch.ones(B, 1, 1, N, dtype=torch.bool, device=DEV),
         "imputate": 1, "stop_imputation_at": 1, "replacement_distribution": "conditional",
         "inpainted_motion": x_obs.to(DEV), "inpainting_mask": kf.to(DEV)}
    if guided:
        y.update(reconstruction_guidance=True, reconstruction_weight=20.0, gradient_schedule=None, diffusion_steps=1000,
                 stop_recguidance_at=2)
    kw = {"y": y}
    if unet:
        kw.update(obs_x0=x_obs.to(DEV), obs_mask=kf.to(DEV))
    return kw


def cond_of(x_obs, kf, cond, scale, guided=False, unet=False):
    kw = dict(cond_emb=cond, cfg=True, text_scale=scale, y_mask=torch.ones(x_obs.shape[0], 1, 1, x_obs.shape[-1], dtype=torch.bool),
              imputate=True, stop_imputation_at=1, inpainted_motion=x_obs, inpainting_mask=kf)
    if guided:
        kw.update(reconstruction_guidance=True, reconstruction_weight=20.0, stop_recguidance_at=2)
    if unet:
        kw.update(obs_x0=x_obs, obs_mask=kf)
    return O.Conditioning(**kw)


def run(d, name, model, shape, **kw):
    return getattr(d, name)(model, shape, **kw)


def covering(f0, F, g):
    return [k for k in range(len(f0)) if f0[k] <= g < f0[k] + F]


def assert_shared_frames_agree(xw, f0, F, what):
    """xw: (B * K, D, 1, F) window rows; every window covering a global frame holds the same bits there"""
    K = len(f0)
    xw = xw.reshape(-1, K, *xw.shape[1:]).cpu()
    for g in range(f0[-1] + F):
        cov = covering(f0, F, g)
        for k in cov[1:]:
            assert torch.equal(xw[:, k, ..., g - f0[k]], xw[:, cov[0], ..., g - f0[cov[0]]]), f"{what}: frame {g}, window {k}"


# ------------------------------------------------------------------------------------------------
# one window == the plain loop, bit for bit
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", ["transformer", "unet"])
def test_one_window_is_the_plain_loop_bit_for_bit(kind):
    B, L = 2, 196
    x_obs, kf, cond, scale = inputs(B, L, 3)
    m, _ = texts_model(kind, {"a": cond[0].to(DEV), "b": cond[1].to(DEV)})
    w = C.ClassifierFreeSampleModel(m)
    kw = ykw(B, L, x_obs, kf, scale, ["a", "b"], unet=kind == "unet")
    shape = (B, D, 1, L)
    g = torch.Generator().manual_seed(4)
    tape = torch.randn(11, B, D, 1, L, generator=g).to(DEV)
    # the engine with window_count = 1: its window path (crop, gather, global noise indexing) at K = 1
    eng = m.engine_for(torch.device(DEV), max_batch=2 * B, nframes=L)
    d = C.create_gaussian_diffusion(timestep_respacing="ddim10")
    eng.set_schedule(d.betas, d.timestep_map)
    ce = cond.to(DEV)
    args = dict(batch=B, cond_emb=ce, cfg=True, text_scale=scale.to(DEV), y_mask=torch.ones(B, L, dtype=torch.uint8, device=DEV),
                imputate=True, stop_imputation_at=1, inpainted_motion=x_obs.to(DEV), inpainting_mask=kf.to(DEV),
                want_pred_xstart=True)
    if kind == "unet":
        args.update(obs_x0=x_obs.to(DEV), obs_mask=kf.to(DEV))
    for name in SAMPLERS:
        extra = dict(sampler=ENGINE_SAMPLER[name])
        if name in ("dpm_solver_sample_loop", "dpm_solver_sde_sample_loop"):
            extra["dpm_order"] = 2
        numel = B * D * L
        modes = {"tape": dict(x_T=tape[0], noise_tape=tape[1:] if name in STOCHASTIC else None),
                 "engine": dict(seed=1234, sample_offset=5),
                 "torch": dict(_torch_stream_args(torch.device(DEV), numel, 11, lazy=True))}
        for mode, nz in modes.items():
            a = eng.sample(**args, **extra, **nz)
            b = eng.sample(**args, **extra, **nz, window_frames0=[0], global_frames=L, want_window_out=True)
            assert torch.equal(a["sample"], b["sample"]), f"{kind} {name} {mode}"
            assert torch.equal(a["pred_xstart"], b["pred_xstart"]), f"{kind} {name} {mode} pred_xstart"
            assert torch.equal(a["sample"], b["windows"]), f"{kind} {name} {mode} window_out"
    # the public API: a Window no shorter than the motion is the plain loop, with torch's generator where it leaves it
    for name in SAMPLERS:
        outs, states = [], []
        for window in (None, C.Window(196, 48)):
            d = C.create_gaussian_diffusion(timestep_respacing="ddim10")
            d.window = window
            torch.manual_seed(77)
            outs.append(run(d, name, w, shape, model_kwargs=kw))
            states.append(torch.cuda.get_rng_state(DEV))
        assert torch.equal(outs[0], outs[1]), f"{kind} {name} public API"
        assert torch.equal(states[0], states[1]), f"{kind} {name} torch generator"


# ------------------------------------------------------------------------------------------------
# shared frames: identical bits in every covering window after every step
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", SAMPLERS)
def test_shared_frames_hold_identical_bits_after_every_step(name):
    B, N, F, O_ = 2, 250, 120, 60
    f0 = W.placement(N, F, O_)
    K = len(f0)
    assert f0 == [0, 60, 120, 130]  # frames 130..179 are covered by three windows
    x_obs, kf, cond, scale = inputs(B, N, 5)
    m, _ = texts_model("transformer", {})
    eng = m.engine_for(torch.device(DEV), max_batch=B * K, nframes=F)
    d = C.create_gaussian_diffusion(timestep_respacing="ddim10")
    eng.set_schedule(d.betas, d.timestep_map)
    T = d.num_timesteps
    g = torch.Generator().manual_seed(6)
    tape = torch.randn(T + 1, B, D, 1, N, generator=g).to(DEV)
    cw = torch.randn(B * K, 512, generator=g).to(DEV)
    crop = lambda t: W.crop(t, f0, F).contiguous()  # noqa: E731
    args = dict(batch=B * K, sampler=ENGINE_SAMPLER[name], cond_emb=cw, cfg=True, text_scale=scale.repeat_interleave(K).to(DEV),
                y_mask=torch.ones(B * K, F, dtype=torch.uint8, device=DEV), imputate=True, stop_imputation_at=0,
                inpainted_motion=crop(x_obs).to(DEV), inpainting_mask=crop(kf).to(DEV), recon_guidance=True,
                stop_recguidance_at=0, recon_coef=np.full(T, 0.05, np.float32), window_frames0=f0, global_frames=N,
                want_window_out=True, want_pred_xstart=True)
    if name in ("dpm_solver_sample_loop", "dpm_solver_sde_sample_loop"):
        args["dpm_order"] = 2
    state = tape[0]
    for k in range(T):
        res = eng.sample(**args, skip_timesteps=k, num_steps=1, resume=k > 0, x_T=state,
                         noise_tape=tape[1 + k:] if name in STOCHASTIC else None)
        assert_shared_frames_agree(res["windows"], f0, F, f"{name} step {k}")
        assert torch.equal(crop(res["sample"]), res["windows"].reshape(B * K, D, 1, F)), f"{name} step {k}: gather"
        state = res["sample"]
    assert torch.isfinite(state).all()


# ------------------------------------------------------------------------------------------------
# against the restatement
# ------------------------------------------------------------------------------------------------
def test_ddim20_whole_loops_vs_restatement():
    tab = O.make_tables("ddim20")
    B = 2
    # K = 2: 300 frames in windows of 196 overlapping 92; text, CFG, imputation, DDIM
    N, F, O_ = 300, 196, 48
    f0 = W.placement(N, F, O_)
    assert f0 == [0, 104]
    x_obs, kf, cond, scale = inputs(B, N, 11)
    m, sd = texts_model("transformer", {"a": cond[0].to(DEV), "b": cond[1].to(DEV)})
    tape = torch.randn(21, B, D, 1, N, generator=torch.Generator().manual_seed(12))
    d = C.create_gaussian_diffusion(timestep_respacing="ddim20")
    d.window, d.noise_tape = C.Window(F, O_), tape.to(DEV)
    got = d.ddim_sample_loop(C.ClassifierFreeSampleModel(m), (B, D, 1, N), model_kwargs=ykw(B, N, x_obs, kf, scale, ["a", "b"]))
    assert got.shape == (B, D, 1, N)
    want = W.sample_loop(sd, tab, (B, D, 1, N), cond_of(x_obs, kf, cond, scale), tape, f0, F, sampler="ddim")
    assert close(got, want, "ddim20 K=2 cfg + imputation")
    # K = 4 with a frame covered three times, per-window prompts, guidance w = 20 (stop_recguidance_at = 2), DDPM
    N, F, O_ = 250, 120, 60
    f0 = W.placement(N, F, O_)
    K = len(f0)
    x_obs, kf, cond, scale = inputs(B, N, 13)
    cw = torch.randn(B * K, 512, generator=torch.Generator().manual_seed(14))
    table = {f"w{i}": cw[i].to(DEV) for i in range(B * K)}
    m, sd = texts_model("transformer", table)
    tape = torch.randn(21, B, D, 1, N, generator=torch.Generator().manual_seed(15))
    d = C.create_gaussian_diffusion(timestep_respacing="ddim20")
    d.window, d.noise_tape = C.Window(F, O_), tape.to(DEV)
    prompts = [[f"w{b * K + k}" for k in range(K)] for b in range(B)]
    got = d.p_sample_loop(C.ClassifierFreeSampleModel(m), (B, D, 1, N),
                          model_kwargs=ykw(B, N, x_obs, kf, scale, prompts, guided=True))
    want = W.sample_loop(sd, tab, (B, D, 1, N), cond_of(x_obs, kf, None, scale, guided=True), tape, f0, F, sampler="ddpm",
                         cond_emb=cw)
    assert close(got, want, "ddim20 K=4 per-window prompts, cfg + imputation + guidance w=20")
    # the rows follow the prompts: swapping two windows' prompts moves the result
    prompts[0][1], prompts[0][2] = prompts[0][2], prompts[0][1]
    swapped = d.p_sample_loop(C.ClassifierFreeSampleModel(m), (B, D, 1, N),
                              model_kwargs=ykw(B, N, x_obs, kf, scale, prompts, guided=True))
    assert not torch.equal(swapped[0], got[0]) and torch.equal(swapped[1], got[1])


def test_64_window_rows_ddpm_tail_transformer_vs_restatement():
    B, N, F, O_ = 16, 600, 196, 48
    f0 = W.placement(N, F, O_)
    assert len(f0) == 4
    x_obs, kf, cond, scale = inputs(B, N, 21)
    m, sd = texts_model("transformer", {f"s{i}": cond[i].to(DEV) for i in range(B)})
    tape = torch.randn(4, B, D, 1, N, generator=torch.Generator().manual_seed(22))
    d = C.create_gaussian_diffusion(timestep_respacing="ddim50")
    d.window, d.noise_tape = C.Window(F, O_), tape.to(DEV)
    got = d.p_sample_loop(C.ClassifierFreeSampleModel(m), (B, D, 1, N), skip_timesteps=47, init_image=x_obs.to(DEV),
                          model_kwargs=ykw(B, N, x_obs, kf, scale, [f"s{i}" for i in range(B)]))
    want = W.sample_loop(sd, O.make_tables("ddim50"), (B, D, 1, N), cond_of(x_obs, kf, cond, scale), tape, f0, F,
                         sampler="ddpm", skip_timesteps=47, init_image=x_obs)
    assert close(got, want, "64 window rows, DDPM tail, cfg + imputation")


def test_64_window_rows_ddim_tail_unet_xl_keyframes_vs_restatement():
    B, N, F, O_ = 16, 600, 196, 48
    f0 = W.placement(N, F, O_)
    x_obs, kf, cond, scale = inputs(B, N, 31)
    m, sd = texts_model("unet", {f"s{i}": cond[i].to(DEV) for i in range(B)})
    tape = torch.randn(4, B, D, 1, N, generator=torch.Generator().manual_seed(32))
    d = C.create_gaussian_diffusion(timestep_respacing="ddim50")
    d.window, d.noise_tape = C.Window(F, O_), tape.to(DEV)
    got = d.ddim_sample_loop(C.ClassifierFreeSampleModel(m), (B, D, 1, N), skip_timesteps=47, init_image=x_obs.to(DEV),
                             model_kwargs=ykw(B, N, x_obs, kf, scale, [f"s{i}" for i in range(B)], unet=True))
    want = TD._unet_fp32_on_gpu(sd, lambda: W.sample_loop(sd, O.make_tables("ddim50"), (B, D, 1, N),
                                                          cond_of(x_obs, kf, cond, scale, unet=True), tape, f0, F,
                                                          sampler="ddim", skip_timesteps=47, init_image=x_obs))
    assert close(got, want, "64 window rows, UNet xl keyframes, DDIM tail", **TD.unet_gate("ddim50", 47, 1))


# ------------------------------------------------------------------------------------------------
# noise in the global layout, generator == fused, graph == direct, launches, outputs
# ------------------------------------------------------------------------------------------------
def _engine_normal(B, per, seed, stream_id):
    out = torch.empty(B, per, device=DEV)
    lib = C.capi.load()
    C.capi.check(lib.cmdi_test_normal(ctypes.c_void_p(out.data_ptr()), B, per, seed, stream_id, 0,
                                      ctypes.c_void_p(torch.cuda.current_stream(DEV).cuda_stream)), "cmdi_test_normal")
    return out


@pytest.mark.parametrize("N", [250, 600])  # 600: the engine generator's quad path in every window; 250: its scalar path
def test_noise_is_drawn_in_the_global_layout(N):
    B, F, O_ = 2, 196 if N == 600 else 120, 48 if N == 600 else 60
    m, _ = texts_model("transformer", {})
    shape = (B, D, 1, N)
    T = 10
    kw = {"y": {"text": ["x", "y"]}}
    m.encode_text = lambda texts: torch.zeros(len(texts), 512, device=DEV)

    def diff(**attrs):
        d = C.create_gaussian_diffusion(timestep_respacing="ddim10")
        d.window = C.Window(F, O_)
        for k, v in attrs.items():
            setattr(d, k, v)
        return d
    # torch: the draws of randn(B, D, 1, N) and randn_like of it, and torch's generator left after them
    torch.manual_seed(5)
    got = diff(rng="torch").p_sample_loop(m, shape, model_kwargs=kw)
    after = torch.cuda.get_rng_state(DEV)
    torch.manual_seed(5)
    tape = torch.stack([torch.randn(*shape, device=DEV) for _ in range(T + 1)])
    assert torch.equal(torch.cuda.get_rng_state(DEV), after)
    assert torch.equal(got, diff(noise_tape=tape).p_sample_loop(m, shape, model_kwargs=kw)), "torch stream"
    # engine generator: x_T from stream 0, step t from stream t + 1, keyed by the global sample and element c * N + g
    seed = 99
    tape = [_engine_normal(B, D * N, seed, 0)] + [_engine_normal(B, D * N, seed, T - k) for k in range(T)]
    tape = torch.stack(tape).view(T + 1, B, D, 1, N)
    got = diff(rng="engine", engine_seed=seed).p_sample_loop(m, shape, model_kwargs=kw)
    assert torch.equal(got, diff(noise_tape=tape).p_sample_loop(m, shape, model_kwargs=kw)), "engine generator"


@pytest.mark.parametrize("name", SAMPLERS)
def test_generator_equals_fused_and_graph_equals_direct(name):
    B, N, F, O_ = 2, 250, 120, 60
    x_obs, kf, cond, scale = inputs(B, N, 41)
    m, _ = texts_model("transformer", {"a": cond[0].to(DEV), "b": cond[1].to(DEV)})
    w = C.ClassifierFreeSampleModel(m)
    kw = ykw(B, N, x_obs, kf, scale, ["a", "b"], guided=True)
    outs = {}
    for mode in ("fused", "direct", "generator"):
        d = C.create_gaussian_diffusion(timestep_respacing="ddim10")
        d.window, d.rng, d.engine_seed = C.Window(F, O_), "engine", 7
        d.use_graph = mode != "direct"
        if mode == "generator":
            steps = list(getattr(d, name + "_progressive")(w, (B, D, 1, N), model_kwargs=kw))
            assert len(steps) == 10 and steps[-1]["pred_xstart"].shape == (B, D, 1, N)
            outs[mode] = steps[-1]["sample"]
        else:
            outs[mode] = run(d, name, w, (B, D, 1, N), model_kwargs=kw)
    assert torch.equal(outs["fused"], outs["generator"]), name
    assert torch.equal(outs["fused"], outs["direct"]), name


def test_launches_per_step_equal_an_unwindowed_loop_at_B_times_K():
    B, N, F, O_ = 2, 250, 120, 60
    K = len(W.placement(N, F, O_))
    m, _ = texts_model("transformer", {})
    m.encode_text = lambda texts: torch.zeros(len(texts), 512, device=DEV)

    def launches(shape, window, steps):
        d = C.create_gaussian_diffusion(timestep_respacing=f"ddim{steps}")
        d.window, d.rng = window, "engine"
        d.p_sample_loop(m, shape, model_kwargs={"y": {"text": ["t"] * shape[0]}})  # warm: step graphs captured
        eng = m.engine_for(torch.device(DEV), max_batch=B * K, nframes=F)
        n0 = eng.launch_count
        d.p_sample_loop(m, shape, model_kwargs={"y": {"text": ["t"] * shape[0]}})
        return eng.launch_count - n0
    win = [launches((B, D, 1, N), C.Window(F, O_), s) for s in (5, 10)]
    plain = [launches((B * K, D, 1, F), None, s) for s in (5, 10)]
    assert win[1] - win[0] == plain[1] - plain[0]  # per step
    assert win[0] == plain[0] + 1  # per call: the crop of x_T


def test_outputs_are_global():
    B, N, F, O_ = 2, 250, 120, 60
    m, _ = texts_model("transformer", {})
    m.encode_text = lambda texts: torch.zeros(len(texts), 512, device=DEV)
    d = C.create_gaussian_diffusion(timestep_respacing="ddim10")
    d.window, d.rng, d.engine_seed = C.Window(F, O_), "engine", 3
    kw = {"y": {"text": ["t", "u"]}}
    sample = d.p_sample_loop(m, (B, D, 1, N), model_kwargs=kw)
    dumps = d.p_sample_loop(m, (B, D, 1, N), model_kwargs=kw, dump_steps=[0, 9])
    assert sample.shape == (B, D, 1, N) and [t.shape for t in dumps] == [(B, D, 1, N)] * 2
    assert torch.equal(dumps[1], sample)  # at t = 0 the DDPM sample is x0 (posterior coefficients 1 and 0)
    steps = list(d.plms_sample_loop_progressive(m, (B, D, 1, N), model_kwargs=kw))
    assert steps[-1]["sample"].shape == (B, D, 1, N) and "old_eps" not in steps[-1]


# ------------------------------------------------------------------------------------------------
# errors
# ------------------------------------------------------------------------------------------------
def test_errors():
    m, _ = texts_model("transformer", {})
    m.encode_text = lambda texts: torch.zeros(len(texts), 512, device=DEV)
    kw = {"y": {"text": ["t", "u"]}}
    d = C.create_gaussian_diffusion(timestep_respacing="ddim10")
    d.window = C.Window(208, 48)  # the transformer engine takes at most 207 frames
    with pytest.raises(RuntimeError, match="nframes = 208"):
        d.p_sample_loop(m, (2, D, 1, 400), model_kwargs=kw)
    with pytest.raises(ValueError, match="overlap"):
        C.Window(196, 99)
    d.window = C.Window(120, 60)
    x = torch.randn(2, D, 1, 400, device=DEV)
    with pytest.raises(NotImplementedError, match="overlapping windows"):
        d.ddim_reverse_sample_loop(m, x, model_kwargs=kw)
    with pytest.raises(NotImplementedError, match="overlapping windows"):
        d.ddim_reverse_sample(m, x, torch.zeros(2, dtype=torch.long), model_kwargs=kw)
    with pytest.raises(NotImplementedError, match="overlapping windows"):
        d.repaint_sample_loop(m, (2, D, 1, 400), model_kwargs=kw)
    with pytest.raises(NotImplementedError, match="overlapping windows"):
        d.repaint_sample_loop_progressive(m, (2, D, 1, 400), model_kwargs=kw)
    with pytest.raises(ValueError, match="one prompt per window"):
        d.p_sample_loop(m, (2, D, 1, 400), model_kwargs={"y": {"text": [["a", "b"], ["c"]]}})
    # the C ABI names the field
    eng = m.engine_for(torch.device(DEV), max_batch=8, nframes=120)
    eng.set_schedule(d.betas, d.timestep_map)
    ce = torch.zeros(8, 512, device=DEV)
    cases = [(dict(batch=6, window_frames0=[0, 60, 120, 130], global_frames=250), "window_count 4 does not divide batch 6"),
             (dict(batch=8, window_frames0=[0, 60, 60, 130], global_frames=250), r"window_frames0\[2\] = 60"),
             (dict(batch=8, window_frames0=[0, 60, 120, 131], global_frames=250), r"window_frames0\[3\] = 131"),
             (dict(batch=8, window_frames0=[0, 60, 190, 200], global_frames=320), r"window_frames0\[2\] = 190"),
             (dict(batch=8, window_frames0=[0, 1, 2, 3], global_frames=100), "global_frames 100 is shorter"),
             (dict(batch=8, global_frames=250), "global_frames is a window field"),
             (dict(batch=8, want_window_out=True), "window_out is a window field"),
             (dict(batch=8, sampler=C.capi.SAMPLER_REPAINT, repaint_jump_length=2, repaint_jump_n_sample=2,
                   window_frames0=[0, 60, 120, 130], global_frames=250), "window_count: sampler 7")]
    for args, match in cases:
        with pytest.raises(RuntimeError, match=match):
            eng.sample(cond_emb=ce[:args["batch"]], seed=1, **args)


# ------------------------------------------------------------------------------------------------
# the reference-driven fixtures (oracle/make_golden_windowed.py)
# ------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def gold(golden_dir):
    from oracle.golden_io import load_golden
    return load_golden(golden_dir, "windowed")


@pytest.mark.parametrize("name", sorted(W.FIXTURES))
def test_reference_driven_fixtures(name, gold):
    N, F, O_, sampler, respacing, skip, guided, unet = W.FIXTURES[name]
    K = len(W.placement(N, F, O_))
    x_obs, kf, cond_w, scale, tape = W.fixture_inputs(name)
    m, _ = texts_model("unet" if unet else "transformer", {f"w{i}": cond_w[i].to(DEV) for i in range(2 * K)})
    prompts = [[f"w{b * K + k}" for k in range(K)] for b in range(2)]
    y = {"text": prompts, "text_scale": scale.to(DEV), "mask": torch.ones(2, 1, 1, N, dtype=torch.bool, device=DEV)}
    kw = {"y": y}
    if unet:
        kw.update(obs_x0=x_obs.to(DEV), obs_mask=kf.to(DEV))
    else:
        y.update(imputate=1, stop_imputation_at=1, replacement_distribution="conditional", inpainted_motion=x_obs.to(DEV),
                 inpainting_mask=kf.to(DEV))
    if guided:
        y.update(reconstruction_guidance=True, reconstruction_weight=20.0, gradient_schedule=None, diffusion_steps=1000,
                 stop_recguidance_at=2)
    d = C.create_gaussian_diffusion(timestep_respacing=respacing)
    d.window, d.noise_tape = C.Window(F, O_), tape.to(DEV)
    loop = d.p_sample_loop if sampler == "ddpm" else d.ddim_sample_loop
    got = loop(C.ClassifierFreeSampleModel(m), (2, D, 1, N), model_kwargs=kw, skip_timesteps=skip, init_image=x_obs.to(DEV))
    tol = TD.unet_gate(respacing, skip, 1) if unet else {}
    assert close(got, gold[f"{name}.ref"], f"fixture {name}", **tol)


# ------------------------------------------------------------------------------------------------
# the multistep samplers against their own restatements, blended
# ------------------------------------------------------------------------------------------------
def test_ddim20_multistep_loops_vs_restatement():
    from oracle import dpm_solver_oracle, dpm_solver_sde_oracle, plms_oracle, unipc_oracle
    B, N, F, O_ = 2, 250, 120, 60
    f0 = W.placement(N, F, O_)
    x_obs, kf, cond, scale = inputs(B, N, 61)
    m, sd = texts_model("transformer", {"a": cond[0].to(DEV), "b": cond[1].to(DEV)})
    tape = torch.randn(21, B, D, 1, N, generator=torch.Generator().manual_seed(62))
    tab = O.make_tables("ddim20")
    loops = {"plms_sample_loop": lambda *a, **k: plms_oracle.plms_sample_loop(*a, order=2, **k),
             "dpm_solver_sample_loop": lambda *a, **k: dpm_solver_oracle.dpm_solver_sample_loop(*a, order=2, **k),
             "unipc_sample_loop": lambda *a, **k: unipc_oracle.unipc_sample_loop(*a, order=2, **k),
             "dpm_solver_sde_sample_loop": lambda *a, **k: dpm_solver_sde_oracle.dpm_solver_sde_sample_loop(*a, order=2, **k)}
    for name, loop in loops.items():
        d = C.create_gaussian_diffusion(timestep_respacing="ddim20")
        d.window, d.noise_tape = C.Window(F, O_), tape.to(DEV)
        got = run(d, name, C.ClassifierFreeSampleModel(m), (B, D, 1, N), model_kwargs=ykw(B, N, x_obs, kf, scale, ["a", "b"]))
        want = W.sample_loop(sd, tab, (B, D, 1, N), cond_of(x_obs, kf, cond, scale), tape, f0, F, loop=loop)
        assert close(got, want, f"ddim20 {name} K=4, cfg + imputation")


# ------------------------------------------------------------------------------------------------
# PRECISION_BF16 transformer and fp16 UNet: the A/F gates of the sampler tests
# ------------------------------------------------------------------------------------------------
def test_bf16_transformer_windowed_loop_meets_the_contract():
    import test_gpu_bf16 as TB
    m, sd = TB.module(text=False)
    sdd = {k: v.to(DEV) for k, v in sd.items()}
    B, N, F, O_, skip = 2, 250, 120, 60, 14
    f0 = W.placement(N, F, O_)
    tape = torch.randn(21 - skip, B, D, 1, N, generator=torch.Generator().manual_seed(71))
    d = C.create_gaussian_diffusion(timestep_respacing="ddim20")
    d.window, d.noise_tape, d.precision = C.Window(F, O_), tape.to(DEV), TB.BF16
    got = d.p_sample_loop(m, (B, D, 1, N), model_kwargs={"y": {}}, skip_timesteps=skip)
    real = O.mdm_forward
    want = {}
    try:
        for name, q in (("A", TB.bf16r), ("F", TB.exact)):
            def fwd(sd_, x, t, cond_emb=None, uncond=False, num_heads=4, _q=q):
                with torch.no_grad():
                    return TB.mdm_model(_q, sdd, x.to(DEV), t.to(DEV), cond_emb, uncond).float().cpu()
            O.mdm_forward = fwd
            want[name] = W.sample_loop(sd, O.make_tables("ddim20"), (B, D, 1, N), O.Conditioning(), tape, f0, F,
                                       sampler="ddpm", skip_timesteps=skip)
    finally:
        O.mdm_forward = real
    TB.gate(got, want["A"], want["F"], f"PRECISION_BF16 windowed DDPM, K=4, last {20 - skip} steps")


def test_fp16_unet_xl_windowed_loop_meets_the_gates():
    B, N, F, O_, skip = 2, 250, 120, 60, 45
    f0 = W.placement(N, F, O_)
    x_obs, kf, cond, scale = inputs(B, N, 81)
    m, sd = texts_model("unet", {"a": cond[0].to(DEV), "b": cond[1].to(DEV)})
    tape = torch.randn(51 - skip, B, D, 1, N, generator=torch.Generator().manual_seed(82))
    kw = {"y": {"text": ["a", "b"], "text_scale": scale.to(DEV)}, "obs_x0": x_obs.to(DEV), "obs_mask": kf.to(DEV)}
    d = C.create_gaussian_diffusion(timestep_respacing="ddim50")
    d.window, d.noise_tape, d.precision = C.Window(F, O_), tape.to(DEV), C.PRECISION_FP16
    got = d.ddim_sample_loop(C.ClassifierFreeSampleModel(m), (B, D, 1, N), model_kwargs=kw, skip_timesteps=skip,
                             init_image=x_obs.to(DEV))
    c = O.Conditioning(cond_emb=cond, cfg=True, text_scale=scale, obs_x0=x_obs, obs_mask=kf)
    a, f = TG.oracle_loop(sd, lambda: W.sample_loop(sd, O.make_tables("ddim50"), (B, D, 1, N), c, tape, f0, F, sampler="ddim",
                                                    skip_timesteps=skip, init_image=x_obs))
    # loops are gated at track 1.5, as in test_gpu_unet_fp16.py / test_gpu_unet_guidance.py
    TG.gate(got, a, f, "fp16 UNet xl windowed, CFG + keyframe input, K=4, last 5 steps", track=1.5)


def test_resume_refuses_another_window_placement():
    m, _ = texts_model("transformer", {})
    m.encode_text = lambda texts: torch.zeros(len(texts), 512, device=DEV)
    eng = m.engine_for(torch.device(DEV), max_batch=8, nframes=120)
    d = C.create_gaussian_diffusion(timestep_respacing="ddim10")
    eng.set_schedule(d.betas, d.timestep_map)
    args = dict(batch=8, sampler=C.capi.SAMPLER_DPM_SOLVER, dpm_order=2, cond_emb=torch.zeros(8, 512, device=DEV), seed=1)
    first = eng.sample(**args, num_steps=1, window_frames0=[0, 60, 120, 130], global_frames=250)
    for f0, n in (([0, 60, 120, 140], 260), ([0, 60, 100, 130], 250)):
        with pytest.raises(RuntimeError, match="does not continue the running history"):
            eng.sample(**args, skip_timesteps=1, num_steps=1, resume=True, x_T=first["sample"][:, :, :, :n]
                       if n <= 250 else torch.zeros(2, D, 1, n, device=DEV), window_frames0=f0, global_frames=n)
    eng.sample(**args, skip_timesteps=1, num_steps=1, resume=True, x_T=first["sample"], window_frames0=[0, 60, 120, 130],
               global_frames=250)

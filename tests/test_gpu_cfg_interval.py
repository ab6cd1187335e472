"""GPU: classifier-free guidance limited to an interval of steps (y['stop_cfg_at'] / y['start_cfg_at']).

  - bit identities for all eight samplers (DDPM, DDIM, PLMS, DPM-Solver++, UniPC, SDE-DPM-Solver++, RePaint, DDIM
    inversion), on the bf16x3 transformer with CFG and the fp16 UNet xl with keyframe CFG: an interval covering every
    step is the guided loop, one covering none is the loop of the unwrapped model;
  - mixed intervals against oracle/cfg_interval_oracle.py: ddim20 loops of every sampler with boundaries inside (PLMS's
    first step evaluates t = 19 outside and t = 18 inside; RePaint's walk revisits the lower boundary) at each sampler's
    bf16x3 gate, fp16 UNet tails at the A / F gates, a B = 64 DDIM tail, a windowed loop (K = 3) and a guided loop
    (reconstruction + joint guidance) whose guidance and interval boundaries differ;
  - generator == fused loop, graph replay == direct launches, calls with interval A, then B, then none == each on a
    fresh engine, launches per step, merged run_eval_jobs == unmerged, sharded == single-GPU;
  - the C ABI's refusals.
"""
import numpy as np
import pytest
import torch

import condmdi_b200 as C
import test_gpu_bf16 as TB
import test_gpu_joint_guidance as TJ
import test_gpu_keyframe_cfg as TK
import test_gpu_transformer_guidance as TT
import test_gpu_unet_guidance as TG
from condmdi_b200.distributed import shard_model_kwargs
from oracle import cfg_interval_oracle as CI
from oracle import condmdi_oracle as O
from oracle import ddim_reverse_oracle as RV
from oracle import joint_guidance_oracle as J
from oracle import keyframe_cfg_oracle as K
from oracle import plms_oracle as P
from oracle import repaint_oracle as R
from oracle import windowed_oracle as W

pytestmark = pytest.mark.gpu
D, L = 263, 196
DEV = "cuda:0"
GATE = dict(rtol=1e-3, atol=1e-4)
close = TK.close
SAMPLERS = TK.SAMPLERS
ALL = SAMPLERS + ["ddim_reverse_sample_loop"]
STOP, START = 6, 18  # the mixed ddim20 loops: guidance at t = 18 .. 6


def interval(kw, stop, start):
    """model_kwargs with y['stop_cfg_at'] / y['start_cfg_at'] (None: the key is left out)"""
    y = dict(kw["y"])
    if stop is not None:
        y["stop_cfg_at"] = stop
    if start is not None:
        y["start_cfg_at"] = start
    return dict(kw, y=y)


def tf_case(B, seed):
    """the bf16x3 text transformer with a per-sample text table, keyframes and per-sample CFG scales"""
    m, sd = TB.module()
    x_obs, _, kf, cond, scale = TG.inputs(B, seed)
    table = {str(i): cond[i].to(DEV) for i in range(B)}
    m.encode_text = lambda texts: torch.stack([table[s] for s in texts])
    return m, sd, x_obs, kf, cond, scale


def tf_kw(B, xo, kf, scale, imputate=True):
    y = {"text": [str(i) for i in range(B)], "text_scale": scale.to(DEV),
         "mask": torch.ones(B, 1, 1, xo.shape[-1], dtype=torch.bool, device=DEV)}
    if imputate:
        y.update(imputate=1, stop_imputation_at=0, replacement_distribution="conditional", inpainted_motion=xo.to(DEV),
                 inpainting_mask=kf.to(DEV))
    return {"y": y}


def tf_cond(B, xo, kf, cond, scale, imputate=True):
    kw = dict(cond_emb=cond, cfg=True, text_scale=scale, y_mask=torch.ones(B, 1, 1, xo.shape[-1], dtype=torch.bool))
    if imputate:
        kw.update(imputate=True, stop_imputation_at=0, inpainted_motion=xo, inpainting_mask=kf)
    return O.Conditioning(**kw)


def run(d, model, name, kw, shape, x=None, **extra):
    if name == "ddim_reverse_sample_loop":
        return d.ddim_reverse_sample_loop(model, x.to(DEV), model_kwargs=kw)
    if name == "repaint_sample_loop":
        extra.update(jump_length=TK.J_LEN, jump_n_sample=TK.J_N)
    return getattr(d, name)(model, shape, model_kwargs=kw, **extra)


def tf_oracle(sd, fn):
    """fn() with the transformer restatement evaluated on the GPU in exact fp32"""
    return TT.oracle_loop(sd, fn, exact_fp32=True)


# ------------------------------------------------------------------------------------------------
# bit identities
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ALL)
@pytest.mark.parametrize("arch", ["transformer", "unet_fp16"])
def test_whole_and_empty_intervals_are_bit_identities(arch, name):
    B, T = 2, 10
    if arch == "transformer":
        m, _, xo, kf, _, scale = tf_case(B, 21)
        guided, kw, x = C.ClassifierFreeSampleModel(m), tf_kw(B, xo, kf, scale), xo
    else:
        m, _, _ = TK.text_model(B)
        x, xo, kf, w_t, w_k = TK.inputs(B, 21)
        guided, kw = C.KeyframeClassifierFreeSampleModel(m), TK.ykw(B, xo, kf, w_t, w_k, imputate=True)

    def loop(model, kw_):
        d = C.create_gaussian_diffusion(timestep_respacing=f"ddim{T}")
        d.rng, d.engine_seed = "engine", 7
        if arch != "transformer":
            d.precision = C.PRECISION_FP16
        return run(d, model, name, kw_, (B, D, 1, L), x=x)
    want_guided, want_plain = loop(guided, kw), loop(m, kw)
    assert not torch.equal(want_guided, want_plain)
    for stop, start in ((0, T - 1), (None, T - 1), (0, None), (-5, 100)):
        assert torch.equal(loop(guided, interval(kw, stop, start)), want_guided), (stop, start)
    for stop, start in ((T, T), (T, None), (None, -1)):
        assert torch.equal(loop(guided, interval(kw, stop, start)), want_plain), (stop, start)


# ------------------------------------------------------------------------------------------------
# mixed intervals against the restatement
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", SAMPLERS)
def test_mixed_ddim20_loops_vs_restatement(name):
    B = 2
    m, sd, xo, kf, cond, scale = tf_case(B, 22)
    tab = O.make_tables("ddim20")
    draws = 1 + (len(R.build_walk(tab.num_timesteps - 1, TK.J_LEN, TK.J_N)) if name == "repaint_sample_loop"
                 else tab.num_timesteps)
    tape = torch.randn(draws, B, D, 1, L, generator=torch.Generator().manual_seed(23))
    d = C.create_gaussian_diffusion(timestep_respacing="ddim20")
    d.noise_tape = tape.to(DEV)
    got = run(d, C.ClassifierFreeSampleModel(m), name, interval(tf_kw(B, xo, kf, scale), STOP, START), (B, D, 1, L))
    c = tf_cond(B, xo, kf, cond, scale)
    with CI.cfg_interval(tab, STOP, START):
        want = tf_oracle(sd, lambda: TK.restated_loop(name, sd, tab, (B, D, 1, L), c, tape))
    assert close(got, want, f"{name} ddim20, CFG at t = {STOP} .. {START}", **TK.loop_gate(name))


def test_mixed_ddim20_inversion_vs_restatement():
    B = 2
    m, sd, xo, kf, cond, scale = tf_case(B, 24)
    x = torch.randn(B, D, 1, L, generator=torch.Generator().manual_seed(25))
    tab = O.make_tables("ddim20")
    d = C.create_gaussian_diffusion(timestep_respacing="ddim20")
    got = d.ddim_reverse_sample_loop(C.ClassifierFreeSampleModel(m), x.to(DEV),
                                     model_kwargs=interval(tf_kw(B, xo, kf, scale), STOP, START))
    c = tf_cond(B, xo, kf, cond, scale)
    with CI.cfg_interval(tab, STOP, START):
        want = tf_oracle(sd, lambda: RV.ddim_reverse_sample_loop(sd, tab, x, c))
    err = (got.cpu() - want).abs().max().item()
    print(f"[ddim_reverse ddim20, CFG at t = {STOP} .. {START}] max_abs={err:.3e} max|x_T|={want.abs().max():.1f}")
    # test_gpu_keyframe_cfg's relative bound for the grown state of the reverse ODE
    assert err <= 1e-4 * want.abs().max().item()


@pytest.mark.parametrize("name", ["ddim_sample_loop", "plms_sample_loop"])
def test_fp16_unet_keyframe_cfg_tails_meet_the_gates(name):
    """ddim50 t = 5 .. 0, keyframe CFG with text CFG and imputation at t = 4 .. 2: PLMS's first step evaluates t = 5
    outside the interval and t = 4 inside it"""
    B = 2
    m, sd, cond = TK.text_model(B)
    x, xo, kf, w_t, w_k = TK.inputs(B, 26)
    tape = torch.randn(7, B, D, 1, L, generator=torch.Generator().manual_seed(27))
    d = C.create_gaussian_diffusion(timestep_respacing="ddim50")
    d.precision, d.noise_tape = C.PRECISION_FP16, tape.to(DEV)
    got = getattr(d, name)(C.KeyframeClassifierFreeSampleModel(m), (B, D, 1, L), skip_timesteps=44, init_image=x.to(DEV),
                           model_kwargs=interval(TK.ykw(B, xo, kf, w_t, w_k, imputate=True), 2, 4))
    c = TK.cond_of(B, xo, kf, cond, w_t, imputate=True)
    tab = O.make_tables("ddim50")

    def restated():
        if name == "plms_sample_loop":
            return P.plms_sample_loop(sd, tab, (B, D, 1, L), c, tape, skip_timesteps=44, init_image=x)
        return O.sample_loop(sd, tab, (B, D, 1, L), c, tape, sampler="ddim", skip_timesteps=44, init_image=x)
    with K.keyframe_cfg(w_k), CI.cfg_interval(tab, 2, 4):
        a, f = TG.oracle_loop(sd, restated)
    TG.gate(got, a, f, f"fp16 UNet xl {name} t = 5 .. 0, keyframe CFG at t = 4 .. 2", track=1.5)


def test_b64_ddim_tail_vs_restatement():
    B = 64
    m, sd, xo, kf, cond, scale = tf_case(B, 28)
    tape = torch.randn(7, B, D, 1, L, generator=torch.Generator().manual_seed(29))
    d = C.create_gaussian_diffusion(timestep_respacing="ddim50")
    d.noise_tape = tape.to(DEV)
    got = d.ddim_sample_loop(C.ClassifierFreeSampleModel(m), (B, D, 1, L), skip_timesteps=44, init_image=xo.to(DEV),
                             model_kwargs=interval(tf_kw(B, xo, kf, scale), 2, 4))
    tab = O.make_tables("ddim50")
    with CI.cfg_interval(tab, 2, 4):
        want = tf_oracle(sd, lambda: O.sample_loop(sd, tab, (B, D, 1, L), tf_cond(B, xo, kf, cond, scale), tape, sampler="ddim",
                                                   skip_timesteps=44, init_image=xo))
    assert close(got, want, "B=64 ddim50 t = 5 .. 0, CFG at t = 4 .. 2", **GATE)


def test_windowed_ddim20_loop_vs_blended_restatement():
    B, N, F, O_ = 2, 440, 196, 48
    f0 = W.placement(N, F, O_)
    assert len(f0) == 3
    K_ = len(f0)
    m, sd, _, _, cond, _ = tf_case(B * K_, 30)
    scale = torch.tensor([2.5, 1.5])
    tape = torch.randn(21, B, D, 1, N, generator=torch.Generator().manual_seed(31))
    d = C.create_gaussian_diffusion(timestep_respacing="ddim20")
    d.window, d.noise_tape = C.Window(F, O_), tape.to(DEV)
    kw = {"y": {"text": [[str(K_ * b + k) for k in range(K_)] for b in range(B)], "text_scale": scale.to(DEV),
                "mask": torch.ones(B, 1, 1, N, dtype=torch.bool, device=DEV)}}
    got = d.ddim_sample_loop(C.ClassifierFreeSampleModel(m), (B, D, 1, N), model_kwargs=interval(kw, STOP, START))
    c = O.Conditioning(cfg=True, text_scale=scale)
    tab = O.make_tables("ddim20")
    with CI.cfg_interval(tab, STOP, START):
        want = tf_oracle(sd, lambda: W.sample_loop(sd, tab, (B, D, 1, N), c, tape, f0, F, sampler="ddim", cond_emb=cond))
    assert close(got, want, f"windowed K=3 ddim20, CFG at t = {STOP} .. {START}", **GATE)


def test_guided_ddim50_tail_with_different_boundaries():
    """ddim50 t = 5 .. 0 at B = 2: CFG at t = 4 .. 1, reconstruction guidance down to t = 3, joint guidance down to t = 2;
    held like test_gpu_joint_guidance's guided tails (every step's pred_xstart and sample, rtol 1e-3 / atol 1e-4)"""
    B, n = 2, 6
    w, sd, x_obs, kw, c, g = TT.loop_case(B, seed=32, stop_recguidance_at=3)
    space, term = TJ.add_joint(kw["y"], B, L, True, 0.1, 2, seed=10)
    tape = torch.randn(1 + n, B, D, 1, L, generator=g)
    d = C.create_gaussian_diffusion(timestep_respacing="ddim50")
    d.joint_space, d.noise_tape = space, tape.to(DEV)
    got = TT.engine_steps(d.ddim_sample_loop_progressive(w, (B, D, 1, L), model_kwargs=interval(kw, 1, 4), skip_timesteps=44,
                                                         init_image=x_obs.to(DEV)), n)
    tab = O.make_tables("ddim50")
    with J.joint_guided(term), CI.cfg_interval(tab, 1, 4):
        want = tf_oracle(sd, lambda: O.sample_loop(sd, tab, (B, D, 1, L), c, tape, "ddim", skip_timesteps=44, init_image=x_obs,
                                                   max_steps=n, return_all=True))
    TJ.gate_fp32(got, want, "guided ddim50, CFG at t = 4 .. 1")


# ------------------------------------------------------------------------------------------------
# invariants
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", SAMPLERS)
def test_generator_equals_fused_and_graph_equals_direct(name):
    B = 2
    m, _, xo, kf, _, scale = tf_case(B, 33)
    w = C.ClassifierFreeSampleModel(m)
    kw = interval(tf_kw(B, xo, kf, scale), 3, 6)
    outs = {}
    for mode in ("fused", "direct", "generator"):
        d = C.create_gaussian_diffusion(timestep_respacing="ddim10")
        d.rng, d.engine_seed, d.use_graph = "engine", 9, mode != "direct"
        extra = dict(jump_length=2, jump_n_sample=2) if name == "repaint_sample_loop" else {}
        if mode == "generator":
            outs[mode] = list(getattr(d, name + "_progressive")(w, (B, D, 1, L), model_kwargs=kw, **extra))[-1]["sample"]
        else:
            outs[mode] = getattr(d, name)(w, (B, D, 1, L), model_kwargs=kw, **extra)
    assert torch.isfinite(outs["fused"]).all()
    assert torch.equal(outs["fused"], outs["generator"]), name
    assert torch.equal(outs["fused"], outs["direct"]), name


@pytest.mark.parametrize("name", ["ddim_sample_loop", "plms_sample_loop", "repaint_sample_loop"])
def test_later_calls_equal_a_fresh_engine(name):
    """Calls with interval A, then B, then none on one engine each equal the same call on a fresh engine: the step
    graphs are keyed by the passes of each step."""
    B = 2
    calls = [(2, 6), (5, 8), None]

    def loop(m, iv):
        _, _, xo, kf, _, scale = tf_case(B, 34)
        kw = tf_kw(B, xo, kf, scale)
        d = C.create_gaussian_diffusion(timestep_respacing="ddim10")
        d.rng, d.engine_seed = "engine", 11
        return run(d, C.ClassifierFreeSampleModel(m), name, kw if iv is None else interval(kw, *iv), (B, D, 1, L))
    shared = tf_case(B, 34)[0]
    got = [loop(shared, iv) for iv in calls]
    for iv, g in zip(calls, got):
        assert torch.equal(g, loop(tf_case(B, 34)[0], iv)), iv


def test_launches_per_step():
    """A step inside the interval launches a CFG step's kernels, a step outside a plain step's (the same count: the
    passes run as one batch); a call with the interval launches what the CFG call launches."""
    B = 2
    m, _, xo, kf, _, scale = tf_case(B, 35)
    kw = tf_kw(B, xo, kf, scale)
    eng = m.engine_for(torch.device(DEV), max_batch=B, nframes=L)

    def count(model, kw_, steps):
        d = C.create_gaussian_diffusion(timestep_respacing=f"ddim{steps}")
        d.rng = "engine"
        d.ddim_sample_loop(model, (B, D, 1, L), model_kwargs=kw_)
        n0 = eng.launch_count
        d.ddim_sample_loop(model, (B, D, 1, L), model_kwargs=kw_)
        return eng.launch_count - n0
    w = C.ClassifierFreeSampleModel(m)
    per_step = {}
    for label, model, kw_ in (("cfg", w, kw), ("plain", m, kw), ("inside", w, interval(kw, 0, None)),
                              ("outside", w, interval(kw, 100, None)), ("mixed", w, interval(kw, 3, 6))):
        n5, n10 = count(model, kw_, 5), count(model, kw_, 10)
        per_step[label] = (n10 - n5, n5)
    print(per_step)
    assert per_step["inside"] == per_step["cfg"]
    assert per_step["outside"][0] == per_step["plain"][0]
    assert per_step["mixed"] == per_step["cfg"]


def test_merged_eval_jobs_equal_unmerged():
    B = 2
    m, _, _, _, _, _ = tf_case(2 * B, 36)
    w = C.ClassifierFreeSampleModel(m)
    jobs = []
    for j in range(2):
        _, _, xo, kf, _, scale = tf_case(B, 37 + j)
        kw = interval(tf_kw(B, xo, kf, scale), 2, 6)
        kw["y"]["text"] = [str(2 * j + i) for i in range(B)]
        jobs.append(C.EvalJob(j, 0, (B, D, 1, L), kw, j))
    d = C.create_gaussian_diffusion(timestep_respacing="ddim10")
    merged = C.run_eval_jobs(d, w, jobs, sampler="ddim_sample_loop", seed=5, merge=2)
    single = C.run_eval_jobs(d, w, jobs, sampler="ddim_sample_loop", seed=5, merge=1)
    for j in range(2):
        assert torch.equal(merged[j], single[j]), j


def test_sharded_equals_single_gpu():
    """sharded_sample's per-rank calls (rng = 'engine', sample_offset = first global row, the rank's slice of
    model_kwargs), emulated on one GPU, assemble the single-GPU batch bit for bit."""
    B, G = 4, 2
    m, _, xo, kf, _, scale = tf_case(B, 39)
    w = C.ClassifierFreeSampleModel(m)
    kw = interval(tf_kw(B, xo, kf, scale), 2, 6)
    d = C.create_gaussian_diffusion(timestep_respacing="ddim10")
    d.rng, d.engine_seed = "engine", 13
    full = d.ddim_sample_loop(w, (B, D, 1, L), model_kwargs=kw)
    parts = []
    for r in range(G):
        lo, hi = r * B // G, (r + 1) * B // G
        d.sample_offset = lo
        parts.append(d.ddim_sample_loop(w, (hi - lo, D, 1, L), model_kwargs=shard_model_kwargs(kw, lo, hi, B)))
    d.sample_offset = 0
    assert torch.equal(torch.cat(parts), full)


# ------------------------------------------------------------------------------------------------
# refusals
# ------------------------------------------------------------------------------------------------
def test_c_abi_refusals():
    B = 2
    m, _, _, _, cond, scale = tf_case(B, 40)
    d = C.create_gaussian_diffusion(timestep_respacing="ddim10")
    eng = m.engine_for(torch.device(DEV), max_batch=B, nframes=L)
    eng.set_schedule(d.betas, d.timestep_map)
    args = dict(batch=B, sampler=C.capi.SAMPLER_DDIM, cond_emb=cond.to(DEV), seed=3)
    with pytest.raises(RuntimeError, match="cfg_interval .* needs cfg or keyframe_scale"):
        eng.sample(stop_cfg_at=2, **args)
    with pytest.raises(RuntimeError, match="stop_cfg_at 5 > start_cfg_at 2"):
        eng.sample(cfg=True, text_scale=scale.to(DEV), stop_cfg_at=5, start_cfg_at=2, **args)
    # the refused calls left the engine usable
    ok = eng.sample(cfg=True, text_scale=scale.to(DEV), stop_cfg_at=2, start_cfg_at=5, **args)["sample"]
    assert torch.isfinite(ok).all() and np.isfinite(ok.sum().item())

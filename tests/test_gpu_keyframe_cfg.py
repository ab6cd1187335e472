"""GPU: classifier-free guidance over keyframes (KeyframeClassifierFreeSampleModel) on the keyframe-conditioned UNet xl.

  - forwards against oracle/keyframe_cfg_oracle.py: bf16x3 within rtol 1e-3 / atol 1e-4; fp16 within the A / F gate
    test_gpu_unet_fp16.py holds CFG outputs to (A: the restatement under CUDA autocast, F: in exact fp32);
  - whole ddim20 loops at B = 2 of all eight samplers (DDPM, DDIM, PLMS, DPM-Solver++, UniPC, SDE-DPM-Solver++,
    RePaint, DDIM inversion) against their restatements run under oracle/keyframe_cfg_oracle.keyframe_cfg, and a
    B = 64 DDIM tail with imputation (192 sequences at max_batch 96);
  - generator == fused loop, graph replay == direct launches, launches per step == a CFG step's;
  - the fp16 input-VJP of the three passes against autograd after CUDA autocast, with exact zeros where a weight
    vanishes, the same with the joint-position term in the seed, and guided DDPM / DDIM tails;
  - one windowed loop (K = 2) against the blended restatement; merged run_eval_jobs == unmerged;
  - a CFG loop after keyframe-CFG calls == the same loop on a fresh engine; the ABI's refusals.
"""
import numpy as np
import pytest
import torch

import condmdi_b200 as C
import test_gpu_dpm_solver as TD
import test_gpu_dpm_solver_sde as TSDE
import test_gpu_unet_guidance as TG
import test_gpu_unipc as TU
from oracle import condmdi_oracle as O
from oracle import ddim_reverse_oracle as RV
from oracle import dpm_solver_oracle as DS
from oracle import dpm_solver_sde_oracle as SDE
from oracle import joint_guidance_oracle as J
from oracle import keyframe_cfg_oracle as K
from oracle import plms_oracle as P
from oracle import repaint_oracle as R
from oracle import unipc_oracle as U
from oracle import windowed_oracle as W

pytestmark = pytest.mark.gpu
D, L = 263, 196
DEV = "cuda:0"
close = TD.close
GATE = dict(rtol=1e-3, atol=1e-4)
SAMPLERS = ["p_sample_loop", "ddim_sample_loop", "plms_sample_loop", "dpm_solver_sample_loop", "unipc_sample_loop",
            "dpm_solver_sde_sample_loop", "repaint_sample_loop"]


def text_model(B, seed=11):
    m, sd = TG.module(seed=seed)
    g = torch.Generator().manual_seed(seed + 100)
    cond = torch.randn(B, 512, generator=g)
    table = {f"p{i}": cond[i].to(DEV) for i in range(B)}
    m.encode_text = lambda texts: torch.stack([table[t] for t in texts])
    return m, sd, cond


def inputs(B, seed, N=L):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, D, 1, N, generator=g)
    xo = torch.randn(B, D, 1, N, generator=g)
    kf = torch.zeros(B, D, 1, N, dtype=torch.bool)
    kf[..., ::20] = True  # sparse keyframes, every feature
    w_t = 1.5 + 2 * torch.rand(B, generator=g)
    w_k = 0.5 + 2 * torch.rand(B, generator=g)  # per sample, != w_t
    return x, xo, kf, w_t, w_k


def ykw(B, xo, kf, w_t, w_k, imputate=False, guided=False, text=True):
    N = xo.shape[-1]
    y = {"keyframe_scale": w_k.to(DEV), "mask": torch.ones(B, 1, 1, N, dtype=torch.bool, device=DEV)}
    if text:
        y.update(text=[f"p{i}" for i in range(B)], text_scale=w_t.to(DEV))
    if imputate:
        y.update(imputate=1, stop_imputation_at=0, replacement_distribution="conditional", inpainted_motion=xo.to(DEV),
                 inpainting_mask=kf.to(DEV))
    if guided:
        y.update(reconstruction_guidance=True, reconstruction_weight=20.0, gradient_schedule=None, diffusion_steps=1000,
                 stop_recguidance_at=0, inpainted_motion=xo.to(DEV), inpainting_mask=kf.to(DEV))
    return {"y": y, "obs_x0": xo.to(DEV), "obs_mask": kf.to(DEV)}


def cond_of(B, xo, kf, cond, w_t, imputate=False, guided=False):
    kw = dict(cond_emb=cond, cfg=cond is not None, text_scale=w_t, y_mask=torch.ones(B, 1, 1, xo.shape[-1], dtype=torch.bool),
              obs_x0=xo, obs_mask=kf)
    if imputate or guided:
        kw.update(inpainted_motion=xo, inpainting_mask=kf)
    if imputate:
        kw.update(imputate=True, stop_imputation_at=0)
    if guided:
        kw.update(reconstruction_guidance=True, reconstruction_weight=20.0, stop_recguidance_at=0)
    return O.Conditioning(**kw)


def oracle_forward(sd, x, t, c, w_k, autocast=False):
    sdd = {k: v.to(DEV) for k, v in sd.items()}
    dev = lambda v: None if v is None else v.to(DEV)  # noqa: E731
    cc = O.Conditioning(cond_emb=dev(c.cond_emb), cfg=c.cfg, text_scale=dev(c.text_scale), obs_x0=dev(c.obs_x0),
                        obs_mask=dev(c.obs_mask))
    tt = torch.full((x.shape[0],), t, device=DEV)
    with TG.ctx_of(autocast), torch.no_grad():
        passes = K.passes(sdd, x.to(DEV), tt, cc)
    with TG.exact_fp32():
        return K.combine(*passes, dev(c.text_scale), w_k.to(DEV)).cpu()


def combine_gate(w_t, w_k, base=GATE):
    """The bf16x3 gate for loops: x0's error is the passes' errors weighted by |1 - w_k| + |w_k - w_t| + |w_t|, against
    |1 - s| + |s| = 4 for the CFG 2.5 the loop gates were set on, so atol scales by that ratio (never below 1)."""
    amp = ((1 - w_k).abs() + (w_k - w_t).abs() + w_t.abs()).max().item() / 4.0
    return dict(rtol=base["rtol"], atol=base["atol"] * max(1.0, amp))


def oracle_loop(sd, w_k, run):
    with K.keyframe_cfg(w_k):
        return TD._unet_fp32_on_gpu(sd, run)


# ------------------------------------------------------------------------------------------------
# forwards
# ------------------------------------------------------------------------------------------------
def test_forward_bf16x3_vs_oracle():
    B = 2
    m, sd, cond = text_model(B)
    x, xo, kf, w_t, w_k = inputs(B, 1)
    wm = C.KeyframeClassifierFreeSampleModel(m)
    for t in (500, 30):
        got = wm(x.to(DEV), torch.full((B,), t, device=DEV), **ykw(B, xo, kf, w_t, w_k))
        want = oracle_forward(sd, x, t, cond_of(B, xo, kf, cond, w_t), w_k)
        assert close(got, want, f"bf16x3 forward t={t}", **GATE)
    # w_k = 1: the CFG wrapper's output up to fp32 rounding
    ones = torch.ones(B)
    got = wm(x.to(DEV), torch.full((B,), 500, device=DEV), **ykw(B, xo, kf, w_t, ones))
    kw = ykw(B, xo, kf, w_t, ones)
    cfg = C.ClassifierFreeSampleModel(m)(x.to(DEV), torch.full((B,), 500, device=DEV), **kw)
    assert close(got, cfg, "w_k = 1 vs CFG", rtol=0, atol=1e-5)
    # the no_cond keyframe model: two passes, n + w_k (c - n)
    mn, sdn = TG.module(text=False, seed=12)
    got = C.KeyframeClassifierFreeSampleModel(mn)(x.to(DEV), torch.full((B,), 500, device=DEV),
                                                   **ykw(B, xo, kf, w_t, w_k, text=False))
    want = oracle_forward(sdn, x, 500, cond_of(B, xo, kf, None, w_t), w_k)
    assert close(got, want, "bf16x3 no_cond forward", **GATE)


def test_forward_fp16_meets_the_cfg_gate():
    B = 2
    m, sd, cond = text_model(B)
    x, xo, kf, w_t, w_k = inputs(B, 2)
    eng = m.engine_for(DEV, max_batch=C.model.keyframe_cfg_max_batch(B, True), precision=C.PRECISION_FP16, nframes=L)
    for t in (500, 30):
        got = eng.forward(x.to(DEV), t, cond_emb=cond.to(DEV), cfg=True, text_scale=w_t, obs_x0=xo.to(DEV),
                          obs_mask=kf.to(DEV), keyframe_scale=w_k)
        c = cond_of(B, xo, kf, cond, w_t)
        TG.gate(got, oracle_forward(sd, x, t, c, w_k, autocast=True), oracle_forward(sd, x, t, c, w_k), f"fp16 kf-cfg t={t}",
                track=1.5)


# ------------------------------------------------------------------------------------------------
# loops
# ------------------------------------------------------------------------------------------------
J_LEN, J_N = 2, 2  # RePaint's jumps in the loop tests


def restated_loop(name, sd, tab, shape, c, tape):
    """The restatement of sampler `name` (the engine's defaults: order 2, UniPC bh2 with the corrector)."""
    if name in ("p_sample_loop", "ddim_sample_loop"):
        return O.sample_loop(sd, tab, shape, c, tape, sampler="ddpm" if name == "p_sample_loop" else "ddim")
    if name == "plms_sample_loop":
        return P.plms_sample_loop(sd, tab, shape, c, tape, order=2)
    if name == "dpm_solver_sample_loop":
        return DS.dpm_solver_sample_loop(sd, tab, shape, c, tape, order=2)
    if name == "unipc_sample_loop":
        return U.unipc_sample_loop(sd, tab, shape, c, tape, order=2)
    if name == "dpm_solver_sde_sample_loop":
        return SDE.dpm_solver_sde_sample_loop(sd, tab, shape, c, tape, 2)
    return R.repaint_sample_loop(sd, tab, shape, c, tape, J_LEN, J_N)


def loop_gate(name):
    """Each sampler's bf16x3 loop gate for the UNet, as its own tests derive it: the multistep samplers weight each
    step's x0 error by their coefficients (test_gpu_dpm_solver.unet_gate and its SDE / UniPC counterparts)."""
    if name == "dpm_solver_sample_loop":
        return TD.unet_gate("ddim20", 0, 2)
    if name == "dpm_solver_sde_sample_loop":
        return TSDE.unet_gate("ddim20", 0, 2)
    if name == "unipc_sample_loop":
        return TU.weighted_gate("ddim20", 0, 2, "bh2", True)
    if name == "repaint_sample_loop":
        return dict(rtol=1e-3, atol=3e-4)  # test_gpu_repaint's gate for the UNet xl walk: more passes than steps
    return GATE


@pytest.mark.parametrize("name", SAMPLERS)
def test_ddim20_loops_vs_restatement(name):
    B = 2
    m, sd, cond = text_model(B)
    _, xo, kf, w_t, w_k = inputs(B, 3)
    tab = O.make_tables("ddim20")
    draws = 1 + (len(R.build_walk(tab.num_timesteps - 1, J_LEN, J_N)) if name == "repaint_sample_loop" else tab.num_timesteps)
    tape = torch.randn(draws, B, D, 1, L, generator=torch.Generator().manual_seed(4))
    d = C.create_gaussian_diffusion(timestep_respacing="ddim20")
    d.noise_tape = tape.to(DEV)
    kw = dict(jump_length=J_LEN, jump_n_sample=J_N) if name == "repaint_sample_loop" else {}
    got = getattr(d, name)(C.KeyframeClassifierFreeSampleModel(m), (B, D, 1, L), model_kwargs=ykw(B, xo, kf, w_t, w_k, imputate=True),
                           **kw)
    c = cond_of(B, xo, kf, cond, w_t, imputate=True)
    want = oracle_loop(sd, w_k, lambda: restated_loop(name, sd, tab, (B, D, 1, L), c, tape))
    assert close(got, want, f"{name} ddim20 kf-cfg + imputation", **combine_gate(w_t, w_k, loop_gate(name)))


def test_ddim20_inversion_vs_restatement():
    """The whole inversion end to end, with test_gpu_ddim_reverse's end-to-end bound: the reverse ODE amplifies, so each
    step may add the per-step gate e_t = atol + rtol |x_{t+1}| (atol scaled by combine_gate), which the later steps
    multiply by their state factors J_t; bound = sum_t e_t prod_{s>t} J_s, |x_{t+1}| from the restated loop."""
    B = 2
    m, sd, cond = text_model(B)
    x, xo, kf, w_t, w_k = inputs(B, 8)
    tab = O.make_tables("ddim20")
    d = C.create_gaussian_diffusion(timestep_respacing="ddim20")
    got = d.ddim_reverse_sample_loop(C.KeyframeClassifierFreeSampleModel(m), x.to(DEV), model_kwargs=ykw(B, xo, kf, w_t, w_k, imputate=True))
    c = cond_of(B, xo, kf, cond, w_t, imputate=True)
    outs = oracle_loop(sd, w_k, lambda: RV.ddim_reverse_sample_loop(sd, tab, x, c, return_all=True))
    an = RV.alphas_cumprod_next(tab)
    J = [float(np.sqrt(1 - an[t]) * tab.sqrt_recip_alphas_cumprod[t] / tab.sqrt_recipm1_alphas_cumprod[t])
         for t in range(tab.num_timesteps)]
    g = combine_gate(w_t, w_k)
    bound = sum((g["atol"] + g["rtol"] * o["sample"].abs().max().item()) * np.prod(J[t + 1:]) for t, o in enumerate(outs))
    err = (got.cpu() - outs[-1]["sample"]).abs().max().item()
    print(f"[ddim_reverse_sample_loop ddim20 kf-cfg + imputation] max_abs={err:.3e} max|x_T|={outs[-1]['sample'].abs().max():.1f} "
          f"bound={bound:.3e} ratio={err / bound:.3f}")
    assert err <= bound
    # and relative to the grown state: the bf16x3 operands carry it to 2^-16, a few roundings per step
    assert err <= 1e-4 * outs[-1]["sample"].abs().max().item()


def test_b64_ddim_tail_with_imputation_vs_restatement():
    B = 64
    m, sd, cond = text_model(B)
    x, xo, kf, w_t, w_k = inputs(B, 5)
    tape = torch.randn(4, B, D, 1, L, generator=torch.Generator().manual_seed(6))
    d = C.create_gaussian_diffusion(timestep_respacing="ddim50")
    d.noise_tape = tape.to(DEV)
    got = d.ddim_sample_loop(C.KeyframeClassifierFreeSampleModel(m), (B, D, 1, L), skip_timesteps=47, init_image=x.to(DEV),
                             model_kwargs=ykw(B, xo, kf, w_t, w_k, imputate=True))
    eng = m.engine_for(torch.device(DEV), max_batch=96, nframes=L)
    assert eng.max_batch == 96  # 3 x 64 sequences
    want = oracle_loop(sd, w_k, lambda: O.sample_loop(sd, O.make_tables("ddim50"), (B, D, 1, L),
                                                      cond_of(B, xo, kf, cond, w_t, imputate=True), tape, sampler="ddim",
                                                      skip_timesteps=47, init_image=x))
    assert close(got, want, "B=64 ddim tail", **combine_gate(w_t, w_k, TD.unet_gate("ddim50", 47, 1)))


@pytest.mark.parametrize("name", SAMPLERS)
def test_generator_equals_fused_and_graph_equals_direct(name):
    B = 2
    m, _, _ = text_model(B)
    _, xo, kf, w_t, w_k = inputs(B, 7)
    wm = C.KeyframeClassifierFreeSampleModel(m)
    outs = {}
    for mode in ("fused", "direct", "generator"):
        d = C.create_gaussian_diffusion(timestep_respacing="ddim10")
        d.rng, d.engine_seed, d.use_graph = "engine", 9, mode != "direct"
        kw = dict(model_kwargs=ykw(B, xo, kf, w_t, w_k, imputate=True))
        if name == "repaint_sample_loop":
            kw.update(jump_length=2, jump_n_sample=2)
        if mode == "generator":
            outs[mode] = list(getattr(d, name + "_progressive")(wm, (B, D, 1, L), **kw))[-1]["sample"]
        else:
            outs[mode] = getattr(d, name)(wm, (B, D, 1, L), **kw)
    assert torch.isfinite(outs["fused"]).all()
    assert torch.equal(outs["fused"], outs["generator"]), name
    assert torch.equal(outs["fused"], outs["direct"]), name


def test_launches_per_step_equal_a_cfg_step():
    B = 2
    m, _, _ = text_model(B)
    _, xo, kf, w_t, w_k = inputs(B, 9)

    def per_step(model):
        n = []
        for steps in (5, 10):
            d = C.create_gaussian_diffusion(timestep_respacing=f"ddim{steps}")
            d.rng = "engine"
            d.ddim_sample_loop(model, (B, D, 1, L), model_kwargs=ykw(B, xo, kf, w_t, w_k))
            eng = m.engine_for(torch.device(DEV), max_batch=3, nframes=L)
            n0 = eng.launch_count
            d.ddim_sample_loop(model, (B, D, 1, L), model_kwargs=ykw(B, xo, kf, w_t, w_k))
            n.append(eng.launch_count - n0)
        return n[1] - n[0], n[0]
    kf_step, kf_call = per_step(C.KeyframeClassifierFreeSampleModel(m))
    cfg_step, cfg_call = per_step(C.ClassifierFreeSampleModel(m))
    assert kf_step == cfg_step and kf_call == cfg_call


# ------------------------------------------------------------------------------------------------
# fp16 input-VJP and guided tails
# ------------------------------------------------------------------------------------------------
def oracle_vjp3(sd, x, t, xo, M, cond, w_t, w_k, autocast):
    """The three pass gradients of sum((xo - x0_hat)^2 * M) w.r.t. x, autograd after the forward (autocast or fp32)."""
    sdd = {k: v.to(DEV) for k, v in sd.items()}
    x, xo, M, cond = x.to(DEV), xo.to(DEV), M.to(DEV), cond.to(DEV)
    tt = torch.full((x.shape[0],), int(t), device=DEV)
    z = x.detach().requires_grad_(True)
    with TG.ctx_of(autocast):
        outs = K.passes(sdd, z, tt, O.Conditioning(cond_emb=cond, cfg=True, obs_x0=xo, obs_mask=M))
    with TG.ctx_of(False):
        hat = K.combine(*outs, w_t.to(DEV), w_k.to(DEV))
        loss = ((xo - hat).square() * M).sum()
        seeds = torch.autograd.grad(loss, outs, retain_graph=True)
        return torch.stack([torch.autograd.grad(o, z, s_, retain_graph=True)[0] for o, s_ in zip(outs, seeds)])


def test_fp16_input_vjp_of_the_three_passes():
    B = 2
    m, sd, cond = text_model(B)
    x, xo, kf, w_t, w_k = inputs(B, 10)
    eng = m.engine_for(DEV, max_batch=3, precision=C.PRECISION_FP16, nframes=L)
    for t in (500, 30):
        got = eng.test_input_vjp(x, t, xo, kf, cond_emb=cond, cfg=True, text_scale=w_t, obs_x0=xo, obs_mask=kf, keyframe_scale=w_k)
        assert got.shape == (3, B, D, 1, L)
        a = oracle_vjp3(sd, x, t, xo, kf, cond, w_t, w_k, True)
        f = oracle_vjp3(sd, x, t, xo, kf, cond, w_t, w_k, False)
        for p, name in enumerate(("c", "u", "n")):
            TG.gate(got[p], a[p], f[p], f"vjp t={t} pass {name}", track=1.5)
        # the keyframe passes see no gradient at keyframes (the blend replaced x_t there); the keyframe-free pass does
        assert (got[0][kf.to(DEV)] == 0).all() and (got[1][kf.to(DEV)] == 0).all()
        assert (got[2][kf.to(DEV)] != 0).any()
    # w_k = w_t: the u pass's seed w_k G - w_t G is exactly 0; w_k = 1: the n pass's seed G - G is exactly 0
    got = eng.test_input_vjp(x, 500, xo, kf, cond_emb=cond, cfg=True, text_scale=w_t, obs_x0=xo, obs_mask=kf, keyframe_scale=w_t)
    assert (got[1] == 0).all() and (got[0] != 0).any()
    got = eng.test_input_vjp(x, 500, xo, kf, cond_emb=cond, cfg=True, text_scale=w_t, obs_x0=xo, obs_mask=kf,
                             keyframe_scale=torch.ones(B))
    assert (got[2] == 0).all() and (got[1] != 0).any()


@pytest.mark.parametrize("name,sampler", [("p_sample_loop", "ddpm"), ("ddim_sample_loop", "ddim")])
def test_fp16_guided_tails_meet_the_gates(name, sampler):
    B = 2
    m, sd, cond = text_model(B)
    x, xo, kf, w_t, w_k = inputs(B, 11)
    tape = torch.randn(4, B, D, 1, L, generator=torch.Generator().manual_seed(12))
    d = C.create_gaussian_diffusion(timestep_respacing="ddim50")
    d.noise_tape, d.precision = tape.to(DEV), C.PRECISION_FP16
    got = getattr(d, name)(C.KeyframeClassifierFreeSampleModel(m), (B, D, 1, L), skip_timesteps=47, init_image=x.to(DEV),
                           model_kwargs=ykw(B, xo, kf, w_t, w_k, imputate=True, guided=True))
    c = cond_of(B, xo, kf, cond, w_t, imputate=True, guided=True)

    def loop(autocast):
        sdd = {k: v.to(DEV) for k, v in sd.items()}

        def fwd(sd_, x_, t_, cond_emb=None, uncond=False, obs_x0=None, obs_mask=None):
            dev = lambda v: None if v is None else v.to(DEV)  # noqa: E731
            with TG.ctx_of(autocast):
                return TG.UNET_FORWARD(sdd, dev(x_), dev(t_), dev(cond_emb), uncond, dev(obs_x0), dev(obs_mask)).float().cpu()
        try:
            O.unet_forward = fwd
            with K.keyframe_cfg(w_k):
                return O.sample_loop(sd, O.make_tables("ddim50"), (B, D, 1, L), c, tape, sampler=sampler, skip_timesteps=47,
                                     init_image=x)
        finally:
            O.unet_forward = TG.UNET_FORWARD
    TG.gate(got, loop(True), loop(False), f"guided {sampler} tail", track=1.5)


def oracle_joint_vjp3(sd, x, t, xo, M, c_r, jt, jm, mean, std, c_j, cond, w_t, w_k, autocast):
    """The three pass gradients of c_r sum((xo - x0_hat)^2 M) + c_j L_j(x0_hat) w.r.t. x (L_j: joint_guidance_oracle's
    joint loss, abs_3d), autograd after the forward (autocast or fp32)."""
    sdd = {k: v.to(DEV) for k, v in sd.items()}
    dev = lambda v: v.to(DEV)  # noqa: E731
    x, xo, M, cond = dev(x), dev(xo), dev(M), dev(cond)
    tt = torch.full((x.shape[0],), int(t), device=DEV)
    z = x.detach().requires_grad_(True)
    with TG.ctx_of(autocast):
        outs = K.passes(sdd, z, tt, O.Conditioning(cond_emb=cond, cfg=True, obs_x0=xo, obs_mask=M))
    with TG.ctx_of(False):
        hat = K.combine(*outs, dev(w_t), dev(w_k)).float()
        loss = c_r * ((xo - hat).square() * M).sum() + c_j * J.joint_loss(hat, dev(jt), dev(jm), dev(mean), dev(std), True)
        seeds = torch.autograd.grad(loss, outs, retain_graph=True)
        return torch.stack([torch.autograd.grad(o, z, s_, retain_graph=True)[0] for o, s_ in zip(outs, seeds)])


def test_fp16_joint_input_vjp_of_the_three_passes():
    """Joint-position guidance's seed under keyframe CFG (joint_seed_kernel's three-pass x0_hat and the seed split over
    the passes) against autograd, per pass, at the gates of the VJP above."""
    B = 2
    m, sd, cond = text_model(B)
    x, xo, kf, w_t, w_k = inputs(B, 13)
    mean, std, jt, jm, _ = J.inputs(B, L, seed=6)
    c_r, c_j = 10.0, 0.05
    eng = m.engine_for(DEV, max_batch=3, precision=C.PRECISION_FP16, nframes=L)
    for t in (500, 30):
        got = eng.test_joint_input_vjp(x, t, jt, jm, mean, std, True, c_j, inpainted_motion=xo, inpainting_mask=kf, c_r=c_r,
                                       cond_emb=cond, cfg=True, text_scale=w_t, obs_x0=xo, obs_mask=kf, keyframe_scale=w_k)
        assert got.shape == (3, B, D, 1, L)
        a, f = [oracle_joint_vjp3(sd, x, t, xo, kf, c_r, jt, jm, mean, std, c_j, cond, w_t, w_k, ac) for ac in (True, False)]
        for p, name in enumerate(("c", "u", "n")):
            TG.gate(got[p], a[p], f[p], f"joint vjp t={t} pass {name}", track=1.5)


# ------------------------------------------------------------------------------------------------
# windows, sharding, isolation, refusals
# ------------------------------------------------------------------------------------------------
def test_windowed_ddim20_loop_vs_blended_restatement():
    B, N, F, O_ = 2, 300, 196, 48
    f0 = W.placement(N, F, O_)
    assert len(f0) == 2
    m, sd, _ = text_model(B * 2)
    cond = torch.stack([m.encode_text([f"p{i}"])[0].cpu() for i in range(B * 2)])
    _, xo, kf, w_t, w_k = inputs(B, 15, N=N)
    tape = torch.randn(21, B, D, 1, N, generator=torch.Generator().manual_seed(16))
    d = C.create_gaussian_diffusion(timestep_respacing="ddim20")
    d.window, d.noise_tape = C.Window(F, O_), tape.to(DEV)
    kw = ykw(B, xo, kf, w_t, w_k, imputate=True)
    kw["y"]["text"] = [[f"p{2 * b}", f"p{2 * b + 1}"] for b in range(B)]
    got = d.ddim_sample_loop(C.KeyframeClassifierFreeSampleModel(m), (B, D, 1, N), model_kwargs=kw)
    c = cond_of(B, xo, kf, None, w_t, imputate=True)
    c.cfg = True
    want = oracle_loop(sd, w_k.repeat_interleave(2), lambda: W.sample_loop(sd, O.make_tables("ddim20"), (B, D, 1, N), c, tape,
                                                                           f0, F, sampler="ddim", cond_emb=cond))
    assert close(got, want, "windowed ddim20 kf-cfg", **combine_gate(w_t, w_k))


def test_merged_eval_jobs_equal_unmerged():
    B = 2
    m, _, _ = text_model(2 * B)
    wm = C.KeyframeClassifierFreeSampleModel(m)
    jobs = []
    for j in range(2):
        _, xo, kf, w_t, w_k = inputs(B, 17 + j)
        kw = ykw(B, xo, kf, w_t, w_k, imputate=True)
        kw["y"]["text"] = [f"p{2 * j + i}" for i in range(B)]
        jobs.append(C.EvalJob(j, 0, (B, D, 1, L), kw, j))
    d = C.create_gaussian_diffusion(timestep_respacing="ddim10")
    merged = C.run_eval_jobs(d, wm, jobs, sampler="ddim_sample_loop", seed=5, merge=2)
    single = C.run_eval_jobs(d, wm, jobs, sampler="ddim_sample_loop", seed=5, merge=1)
    for j in range(2):
        assert torch.equal(merged[j], single[j]), j


def test_cfg_after_keyframe_cfg_equals_a_fresh_engine():
    B = 2
    _, xo, kf, w_t, w_k = inputs(B, 19)

    def cfg_loop(m):
        d = C.create_gaussian_diffusion(timestep_respacing="ddim10")
        d.rng, d.engine_seed, d.max_batch = "engine", 4, 3
        return d.ddim_sample_loop(C.ClassifierFreeSampleModel(m), (B, D, 1, L), model_kwargs=ykw(B, xo, kf, w_t, w_k, imputate=True))
    m, _, _ = text_model(B)
    d = C.create_gaussian_diffusion(timestep_respacing="ddim10")
    d.rng, d.engine_seed = "engine", 4
    d.ddim_sample_loop(C.KeyframeClassifierFreeSampleModel(m), (B, D, 1, L), model_kwargs=ykw(B, xo, kf, w_t, w_k, imputate=True))
    after = cfg_loop(m)
    fresh, _, _ = text_model(B)
    assert torch.equal(after, cfg_loop(fresh))


def test_refusals():
    B = 2
    m, _, cond = text_model(B)
    x, xo, kf, w_t, w_k = inputs(B, 20)
    # the wrapper: the transformer and a UNet without keyframe input
    with pytest.raises(ValueError):
        C.KeyframeClassifierFreeSampleModel(C.MDM(cond_mode="text", cond_mask_prob=0.1))
    with pytest.raises(ValueError):
        C.KeyframeClassifierFreeSampleModel(TG.module(kf_cond=False)[0])
    # the ABI: no keyframes; passes x batch beyond 2 * max_batch
    eng = m.engine_for(DEV, max_batch=2, nframes=L)
    assert eng.max_batch == 2
    with pytest.raises(RuntimeError, match="obs_x0 and obs_mask"):
        eng.forward(x.to(DEV), 500, cond_emb=cond.to(DEV), cfg=True, text_scale=w_t, keyframe_scale=w_k)
    with pytest.raises(RuntimeError, match="2 \\* max_batch"):
        eng.forward(x.to(DEV), 500, cond_emb=cond.to(DEV), cfg=True, text_scale=w_t, obs_x0=xo.to(DEV), obs_mask=kf.to(DEV),
                    keyframe_scale=w_k)
    # the transformer engine refuses keyframe_scale
    mt = C.MDM(cond_mode="text", cond_mask_prob=0.1).to(DEV)
    et = mt.engine_for(DEV, max_batch=4, nframes=L)
    with pytest.raises(RuntimeError, match="keyframe-conditioned MDM_UNET"):
        et.forward(x.to(DEV), 500, cond_emb=cond.to(DEV), cfg=True, text_scale=w_t, obs_x0=xo.to(DEV), obs_mask=kf.to(DEV),
                   keyframe_scale=w_k)
    # reconstruction guidance at bf16x3 keeps its refusal
    d = C.create_gaussian_diffusion(timestep_respacing="ddim10")
    d.rng = "engine"
    with pytest.raises(RuntimeError, match="PRECISION_FP16"):
        d.ddim_sample_loop(C.KeyframeClassifierFreeSampleModel(m), (B, D, 1, L),
                           model_kwargs=ykw(B, xo, kf, w_t, w_k, guided=True))


def test_forwards_vs_reference_fixtures():
    import os
    from oracle import make_golden_keyframe_cfg as MG
    from oracle.golden_io import load_golden
    gold = load_golden(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden"), "keyframe_cfg")
    gi = MG.inputs()
    sd, sdn = MG.weights()
    B = gi["x"].shape[0]
    for name, w, text in (("fwd.t500", sd, True), ("fwd.t30", sd, True), ("nocond.t500", sdn, False)):
        m = C.MDM_UNET(keyframe_conditioned=True, **({"cond_mode": "text", "cond_mask_prob": 0.1} if text else {}))
        assert not any(m.load_state_dict(w, strict=False))
        m = m.to(DEV)
        m.encode_text = lambda texts: gi["cond"].to(DEV)
        t = int(name.split(".t")[1])
        kw = ykw(B, gi["x_obs"], gi["kf_mask"], gi["text_scale"], gi["keyframe_scale"], text=text)
        kw["y"]["text"] = ["a", "b"]
        got = C.KeyframeClassifierFreeSampleModel(m)(gi["x"].to(DEV), torch.full((B,), t, device=DEV), **kw)
        assert close(got, torch.from_numpy(gold[f"{name}.ref"]), f"fixture {name}", **GATE)

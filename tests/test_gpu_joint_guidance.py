"""GPU: joint-position guidance -- the joint seed kernel (cmdi_joint_guidance_seed) against fp64 autograd of the oracle's
de-normalisation + recover_from_ric, the guided input-VJP with the joint term, guided loops against
oracle/joint_guidance_oracle.py, and the invariants of the step path (graph replay, generators, unguided and
reconstruction-only calls after joint-guided ones, launch counts, refusals)."""
import pytest
import torch

import condmdi_b200 as C
import test_gpu_bf16 as TB
import test_gpu_dpm_solver as TD
import test_gpu_transformer_guidance as TT
import test_gpu_unet_guidance as TG
from condmdi_b200.engine import joint_guidance_seed
from oracle import condmdi_oracle as O
from oracle import dpm_solver_oracle as S
from oracle import joint_guidance_oracle as J
from oracle import repaint_oracle as R

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
# max |E - F| / max |F| of the seed kernel (fp32 FK and block scans over <= 224 frames); measured on H100: at most
# 1.5e-7 (abs3d) and 6.8e-7 (relative, L = 224)
SEED_GATE = 5e-6


# ---------------------------------------------------------------------------------------------------------------------
# the joint seed kernel
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("abs_3d", [True, False], ids=["abs3d", "rel"])
@pytest.mark.parametrize("B,L", [(2, 196), (2, 224), (2, 2), (64, 196)])
def test_joint_seed_kernel(abs_3d, B, L):
    mean, std, target, mask, g = J.inputs(B, L, seed=B * 1000 + L + abs_3d)
    x0 = torch.randn(B, 263, 1, L, generator=g)
    mask[-1] = False  # the last sample observes nothing
    got = joint_guidance_seed(x0.to(DEV), target.to(DEV), mask.to(DEV), mean.to(DEV), std.to(DEV), abs_3d).cpu()
    want = J.joint_seed(x0.to(DEV).double(), target.to(DEV).double(), mask.to(DEV), mean.to(DEV).double(),
                        std.to(DEV).double(), abs_3d).cpu()
    assert (got[:, 67:] == 0).all(), "channels >= 67 must be exact zeros"
    assert (got[-1] == 0).all(), "a sample with an empty mask must have a zero gradient"
    ratio = ((got.double() - want).abs().max() / want.abs().max()).item()
    print(f"[joint seed {'abs3d' if abs_3d else 'rel'} B={B} L={L}] max|E-F| / max|F| = {ratio:.3e} "
          f"(max|F| = {want.abs().max().item():.3e})")
    assert ratio <= SEED_GATE


@pytest.mark.parametrize("abs_3d", [True, False], ids=["abs3d", "rel"])
@pytest.mark.parametrize("ld", [264, 272])
def test_joint_seed_kernel_frame_major(abs_3d, ld):
    """the engine's layout: frame-major rows of ld >= D_pad columns.  The seed equals the reference-layout call's bit for
    bit on the 263 features, and every column from 67 on, the pad included, is an exact zero (the output is prefilled
    with NaN)"""
    B, L = 3, 196
    mean, std, target, mask, g = J.inputs(B, L, seed=40 + ld)
    x0 = torch.randn(B, 263, 1, L, generator=g).to(DEV)
    rows = torch.full((B, L, ld), float("nan"), device=DEV)
    rows[:, :, :263] = x0[:, :, 0].transpose(1, 2)
    args = (target.to(DEV), mask.to(DEV), mean.to(DEV), std.to(DEV), abs_3d)
    out = torch.full((B, L, ld), float("nan"), device=DEV)
    got = joint_guidance_seed(rows, *args, ld=ld, out=out)
    ref = joint_guidance_seed(x0, *args)
    assert (got[:, :, 67:] == 0).all(), "columns >= 67 (pad included) must be exact zeros"
    assert torch.equal(got[:, :, :263], ref[:, :, 0].transpose(1, 2))


# ---------------------------------------------------------------------------------------------------------------------
# input-VJP of c_r L_r + c_j L_j per pass (the transformer against tests/test_gpu_bf16.py's fp64 models A and F)
# ---------------------------------------------------------------------------------------------------------------------
def joint_pass_vjps(forward, x, t, xo, M, c_r, jt, jm, mean, std, abs_3d, c_j, cond_emb, scale):
    """TB.pass_vjps for the loss c_r sum((xo - x0_hat)^2 M) + c_j L_j(x0_hat), CFG, fp64 on the GPU"""
    dbl = lambda v: v.to(DEV).double()  # noqa: E731
    z = x.detach().to(DEV).double().requires_grad_(True)
    outs = [forward(z, t.to(DEV), dbl(cond_emb), False), forward(z, t.to(DEV), dbl(cond_emb), True)]
    hat = outs[1] + dbl(scale).view(-1, 1, 1, 1) * (outs[0] - outs[1])
    loss = c_j * J.joint_loss(hat, dbl(jt), jm.to(DEV), dbl(mean), dbl(std), abs_3d)
    if xo is not None:
        loss = loss + c_r * ((dbl(xo) - hat).square() * dbl(M)).sum()
    seeds = torch.autograd.grad(loss, outs, retain_graph=True)
    return torch.stack([torch.autograd.grad(o, z, s_, retain_graph=True)[0] for o, s_ in zip(outs, seeds)]).cpu()


@pytest.mark.parametrize("recon", [True, False], ids=["recon+joint", "joint"])
@pytest.mark.parametrize("abs_3d", [True, False], ids=["abs3d", "rel"])
def test_transformer_joint_input_vjp(recon, abs_3d):
    B, L = 2, 196
    m, sd = TB.module()
    x, xo, M, cond, scale = TT.vjp_case_inputs(263, L, B, seed=17)
    mean, std, jt, jm, _ = J.inputs(B, L, seed=5)
    c_r, c_j = (10.0 if recon else 0.0), (0.05 if abs_3d else 0.002)
    sdd = {k: v.to(DEV).double() for k, v in sd.items()}
    failures = []
    for t in (500, 30):
        tt = torch.full((B,), t)
        a, f = [joint_pass_vjps(lambda z, t_, c, u, q=q: TB.mdm_model(q, sdd, z, t_, c, u), x, tt, xo if recon else None, M,
                                c_r, jt, jm, mean, std, abs_3d, c_j, cond, scale) for q in (TB.bf16r, TB.exact)]
        for name, prec in (("bf16x3", C.PRECISION_BF16X3), ("bf16", C.PRECISION_BF16)):
            eng = m.engine_for(DEV, max_batch=B, precision=prec, nframes=L)
            got = eng.test_joint_input_vjp(x, t, jt, jm, mean, std, abs_3d, c_j, inpainted_motion=xo if recon else None,
                                           inpainting_mask=M if recon else None, c_r=c_r, cond_emb=cond, cfg=True,
                                           text_scale=scale)
            for k, which in enumerate(["cond", "uncond"]):
                try:
                    TB.gate(got[k], a[k], f[k], f"joint vjp {name} {'recon+' if recon else ''}joint "
                            f"{'abs3d' if abs_3d else 'rel'} t={t} {which}", c=TT.GATES[name])
                except AssertionError as err:
                    failures.append(str(err))
    assert not failures, failures


def unet_joint_vjp(sdd, x, t, xo, M, c_r, jt, jm, mean, std, c_j, cond=None, uncond=False, obs=None, kf=None, scale=None,
                   autocast=True):
    """TG.oracle_vjp for c_r sum((xo - x0_hat)^2 M) + c_j L_j(x0_hat): autograd after a forward under autocast (or fp32)"""
    dev = lambda v: None if v is None else v.to(DEV)  # noqa: E731
    x, xo, M, cond, obs, kf = dev(x), dev(xo), dev(M), dev(cond), dev(obs), dev(kf)
    tt = torch.full((x.shape[0],), int(t), device=DEV)
    z = x.detach().requires_grad_(True)
    with TG.ctx_of(autocast):
        outs = [TG.UNET_FORWARD(sdd, z, tt, cond, uncond, obs, kf)]
        if scale is not None:
            outs.append(TG.UNET_FORWARD(sdd, z, tt, cond, True, obs, kf))
    with TG.ctx_of(False):
        hat = outs[0] if scale is None else outs[1] + (scale.to(DEV).view(-1, 1, 1, 1) * (outs[0] - outs[1]))
        hat = hat.float()
        loss = c_r * ((xo - hat).square() * M).sum() + c_j * J.joint_loss(hat, dev(jt), dev(jm), dev(mean), dev(std), True)
        seeds = torch.autograd.grad(loss, outs, retain_graph=True)
        return torch.stack([torch.autograd.grad(o, z, s_, retain_graph=True)[0] for o, s_ in zip(outs, seeds)])


@pytest.mark.parametrize("mode,B", [("text", 2), ("uncond", 2), ("cfg", 2), ("cfg", 64)])
def test_unet_fp16_joint_input_vjp(mode, B):
    """the keyframe-conditioned xl MDM_UNET at PRECISION_FP16 against autograd after an autocast forward (A) and an fp32
    one (F), with test_gpu_unet_guidance.py's gates: |E - A| <= |A - F| and |E - F| <= 2 |A - F|, max and mean"""
    m, sd = TG.module()
    sdd = {k: v.to(DEV) for k, v in sd.items()}
    x, xo, kf, cond, scale = TG.inputs(B, seed=70 + B)
    mean, std, jt, jm, _ = J.inputs(B, TG.L, seed=6)
    c_r, c_j = 10.0, 0.05
    kw = {"cond": cond, "uncond": mode == "uncond"}
    cfg = mode == "cfg"
    eng = m.engine_for(DEV, max_batch=B, precision=C.PRECISION_FP16, nframes=TG.L)
    for t in (500, 30):
        got = eng.test_joint_input_vjp(x, t, jt, jm, mean, std, True, c_j, inpainted_motion=xo, inpainting_mask=kf, c_r=c_r,
                                       cond_emb=cond, uncond=kw["uncond"], cfg=cfg, text_scale=scale if cfg else None,
                                       obs_x0=xo, obs_mask=kf)
        a, f = [unet_joint_vjp(sdd, x, t, xo, kf, c_r, jt, jm, mean, std, c_j, obs=xo, kf=kf, scale=scale if cfg else None,
                               autocast=ac, **kw) for ac in (True, False)]
        assert got.shape == a.shape
        for k, what in enumerate(["cond", "uncond"][: got.shape[0]]):
            TG.gate(got[k], a[k], f[k], f"unet fp16 joint vjp {mode} B={B} t={t} {what} pass")


# ---------------------------------------------------------------------------------------------------------------------
# loops against the oracle with its model evaluated on the GPU
# ---------------------------------------------------------------------------------------------------------------------
def add_joint(y, B, L, abs_3d, weight, stop, seed):
    mean, std, jt, jm, _ = J.inputs(B, L, seed=seed)
    y.update(joint_guidance=True, joint_target=jt.to(DEV), joint_target_mask=jm.to(DEV), joint_guidance_weight=weight,
             joint_gradient_schedule=None, stop_jointguidance_at=stop, diffusion_steps=1000)
    return C.JointSpace(mean, std, abs_3d), J.JointTerm(jt, jm, mean, std, abs_3d, weight, None, 1000, stop)


def gate_fp32(got, want, what, sample_atol=1e-4):
    """rtol 1e-3 / atol 1e-4 on every step's pred_xstart, and rtol 1e-3 / sample_atol on every step's sample"""
    failures = []
    for k, (e, r) in enumerate(zip(got, want)):
        for key in ("pred_xstart", "sample"):
            ge, gr = e[key].cpu().double(), r[key].double()
            err = (ge - gr).abs()
            atol = sample_atol if key == "sample" else 1e-4
            viol = (err > atol + 1e-3 * gr.abs()).double().mean().item()
            print(f"[{what} step {k} {key}] max_abs={err.max():.3e} max|ref|={gr.abs().max():.3e} violations={viol:.2e}")
            if viol > 0:
                failures.append((k, key, err.max().item(), viol))
    assert not failures, failures


def test_bf16x3_ddim50_tail_joint_b64():
    """ddim50 t = 5 .. 0 at B = 64: CFG, imputation, reconstruction guidance down to t = 3, joint guidance down to t = 2"""
    w, sd, x_obs, kw, tape, run, B, n = TT.ddim50_b64_case()
    space, term = add_joint(kw["y"], B, 196, True, 0.1, 2, seed=8)
    d = C.create_gaussian_diffusion(timestep_respacing="ddim50")
    d.joint_space = space
    d.noise_tape = tape.to(DEV)
    got = TT.engine_steps(d.ddim_sample_loop_progressive(w, (B, 263, 1, 196), model_kwargs=kw, skip_timesteps=44,
                                                         init_image=x_obs.to(DEV)), n)
    with J.joint_guided(term):
        want = TT.oracle_loop(sd, run, exact_fp32=True)
    gate_fp32(got, want, "bf16x3 B=64 ddim50 joint")


@pytest.mark.parametrize("abs_3d", [True, False], ids=["abs3d", "rel"])
def test_bf16x3_ddpm_tail_joint_b2(abs_3d):
    """t = 49 .. 46 of the 1000-step schedule, every step guided by both terms"""
    B, n = 2, 4
    w, sd, x_obs, kw, c, g = TT.loop_case(B, seed=63, stop_recguidance_at=0)
    space, term = add_joint(kw["y"], B, 196, abs_3d, 0.1 if abs_3d else 0.005, 0, seed=9)
    tape = torch.randn(1 + n, B, 263, 1, 196, generator=g)
    d = C.create_gaussian_diffusion()
    d.joint_space = space
    d.noise_tape = tape.to(DEV)
    got = TT.engine_steps(d.p_sample_loop_progressive(w, (B, 263, 1, 196), model_kwargs=kw, skip_timesteps=950,
                                                      init_image=x_obs.to(DEV)), n)
    with J.joint_guided(term):
        want = TT.oracle_loop(sd, lambda: O.sample_loop(sd, O.make_tables(""), (B, 263, 1, 196), c, tape, "ddpm",
                                                        skip_timesteps=950, init_image=x_obs, max_steps=n, return_all=True),
                              exact_fp32=True)
    gate_fp32(got, want, f"bf16x3 B=2 ddpm joint {'abs3d' if abs_3d else 'rel'}")


def test_bf16x3_dpm_solver_order2_joint_b2():
    """DPM-Solver++ order 2 on ddim50, t = 5 .. 0: CFG, imputation, reconstruction and joint guidance on every step.
    Every step's x0 is held to rtol 1e-3 / atol 1e-4.  The sample weights the x0 errors of the last two steps by
    sum_j |B_j| where DDIM weights one by |B0| (test_gpu_dpm_solver.py's unet_gate), and a guided x0 already sits near
    atol (max 9e-5 in the ddim50 loop above), so the samples' atol is scaled by that ratio of weights, as the existing
    DPM-Solver++ tests scale it."""
    B, n = 2, 6
    w, sd, x_obs, kw, c, g = TT.loop_case(B, seed=65, stop_recguidance_at=0)
    space, term = add_joint(kw["y"], B, 196, True, 0.1, 0, seed=13)
    tape = torch.randn(1, B, 263, 1, 196, generator=g)
    d = C.create_gaussian_diffusion(timestep_respacing="ddim50")
    d.joint_space = space
    d.noise_tape = tape.to(DEV)
    got = TT.engine_steps(d.dpm_solver_sample_loop_progressive(w, (B, 263, 1, 196), model_kwargs=kw, skip_timesteps=44,
                                                               init_image=x_obs.to(DEV), order=2), n)
    with J.joint_guided(term):
        want = TT.oracle_loop(sd, lambda: S.dpm_solver_sample_loop(sd, O.make_tables("ddim50"), (B, 263, 1, 196), c, tape, 2,
                                                                   skip_timesteps=44, init_image=x_obs, return_all=True),
                              exact_fp32=True)
    gate_fp32(got, want, "bf16x3 B=2 dpm-solver++ order 2 joint", sample_atol=TD.unet_gate("ddim50", 44, 2)["atol"])


def test_bf16x3_repaint_walk_joint_b2():
    """RePaint on ddim50 from t = 5, jump_length 2, jump_n_sample 2: CFG, imputation, reconstruction guidance and joint
    guidance stopping at 2, so the revisited stretch is guided by position"""
    B, skip, j, r = 2, 44, 2, 2
    w, sd, x_obs, kw, c, g = TT.loop_case(B, seed=66, stop_recguidance_at=0)
    space, term = add_joint(kw["y"], B, 196, True, 0.1, 2, seed=14)
    n_ops = len(C.diffusion._repaint_walk(49 - skip, j, r))
    tape = torch.randn(1 + n_ops, B, 263, 1, 196, generator=g)
    d = C.create_gaussian_diffusion(timestep_respacing="ddim50")
    d.joint_space = space
    d.noise_tape = tape.to(DEV)
    got = d.repaint_sample_loop(w, (B, 263, 1, 196), model_kwargs=kw, skip_timesteps=skip, init_image=x_obs.to(DEV),
                                jump_length=j, jump_n_sample=r)
    with J.joint_guided(term):
        want = TT.oracle_loop(sd, lambda: R.repaint_sample_loop(sd, O.make_tables("ddim50"), (B, 263, 1, 196), c, tape, j, r,
                                                                skip_timesteps=skip, init_image=x_obs), exact_fp32=True)
    gate_fp32([{"sample": got, "pred_xstart": got}], [{"sample": want, "pred_xstart": want}], "bf16x3 B=2 repaint joint")


def test_unet_fp16_ddpm_tail_joint_b2():
    B = 2
    m, w, sd, x_obs, kf, y, c, g = TG.setup(B, seed=22)
    y.update(imputate=1, stop_imputation_at=1, replacement_distribution="conditional")
    c.imputate, c.stop_imputation_at = True, 1
    space, term = add_joint(y, B, TG.L, True, 0.1, 0, seed=10)
    tape = torch.randn(5, B, TG.D, 1, TG.L, generator=g)
    d = C.create_gaussian_diffusion()
    d.precision = C.PRECISION_FP16
    d.joint_space = space
    d.noise_tape = tape.to(DEV)
    kw = {"y": y, "obs_x0": x_obs.to(DEV), "obs_mask": kf.to(DEV)}
    got = d.p_sample_loop(w, (B, TG.D, 1, TG.L), model_kwargs=kw, skip_timesteps=996, init_image=x_obs.to(DEV))
    with J.joint_guided(term):
        a, f = TG.oracle_loop(sd, lambda: O.sample_loop(sd, O.make_tables(""), (B, TG.D, 1, TG.L), c, tape, "ddpm",
                                                        skip_timesteps=996, init_image=x_obs))
    TG.gate(got, a, f, "UNet fp16 B=2 ddpm 4-step tail, cfg + imputation + recon + joint", track=1.5)


# ---------------------------------------------------------------------------------------------------------------------
# invariants
# ---------------------------------------------------------------------------------------------------------------------
def joint_case(B=2, seed=64):
    w, sd, x_obs, kw, c, g = TT.loop_case(B, seed=seed, stop_recguidance_at=0)
    y = dict(kw["y"])
    space, _ = add_joint(y, B, 196, True, 0.1, 2, seed=11)
    return w, x_obs, kw, {"y": y}, space


def run_ddim(w, kw, x_obs, space=None, use_graph=True, progressive=False, skip=44):
    d = C.create_gaussian_diffusion(timestep_respacing="ddim50")
    d.joint_space, d.use_graph, d.rng = space, use_graph, "engine"
    d.engine_seed = 123
    args = dict(model_kwargs=kw, skip_timesteps=skip, init_image=x_obs.to(DEV), noise=torch.zeros(2, 263, 1, 196, device=DEV))
    if progressive:
        return [o["sample"].clone() for o in d.ddim_sample_loop_progressive(w, (2, 263, 1, 196), **args)][-1]
    return d.ddim_sample_loop(w, (2, 263, 1, 196), **args)


def test_graph_replay_generator_and_other_calls_are_unchanged():
    w, x_obs, kw_recon, kw_joint, space = joint_case()
    unguided = {"y": {k: v for k, v in kw_recon["y"].items() if k != "reconstruction_guidance"}}
    before = [run_ddim(w, kw, x_obs) for kw in (unguided, kw_recon)]
    graph = run_ddim(w, kw_joint, x_obs, space)
    direct = run_ddim(w, kw_joint, x_obs, space, use_graph=False)
    gen = run_ddim(w, kw_joint, x_obs, space, progressive=True)
    assert torch.equal(graph, direct), "graph replay differs from direct launches"
    assert torch.equal(graph, gen), "the generator differs from the fused loop"
    after = [run_ddim(w, kw, x_obs) for kw in (unguided, kw_recon)]
    for b, a_, what in zip(before, after, ("unguided", "reconstruction-only")):
        assert torch.equal(a_, b), f"a {what} loop changed after joint-guided calls"
    recon_only = run_ddim(w, kw_recon, x_obs)
    assert not torch.equal(graph, recon_only), "joint guidance had no effect"


def test_launch_counts():
    """Per guided step of the 8-layer transformer, a reconstruction-guided loop launches the parent's formula: the unchained
    guided pass (token rows, frame embedding, 7 per layer, output head: 59), the step kernel (1) and the backward pass
    (seed, head, 8 per layer, input: 68), 128 in all; a joint-guided call adds the joint seed kernel at every guided
    evaluation (its coefficient is 0 where joint guidance has stopped, so one step graph serves every guided step).  The
    per-step count is the difference between a 6-step and a 3-step call, so the per-call launches cancel."""
    w, x_obs, kw_recon, kw_joint, space = joint_case()
    eng = C.resolve_model(w)[0].engine_for(DEV, max_batch=2, precision=C.PRECISION_BF16X3, nframes=196)

    def count(kw, skip, sp=None):
        n0 = eng.launch_count
        run_ddim(w, kw, x_obs, sp, skip=skip)
        return eng.launch_count - n0

    per_step = {}
    for name, kw, sp in (("recon", kw_recon, None), ("recon+joint", kw_joint, space)):
        count(kw, 44, sp)  # capture the step graphs first
        per_step[name] = (count(kw, 44, sp) - count(kw, 47, sp)) / 3
    print(f"[launches per guided step] {per_step}")
    assert per_step["recon"] == 59 + 1 + 68
    assert per_step["recon+joint"] == 59 + 1 + 68 + 1


def test_graphs_follow_the_root_representation():
    """an abs_3d joint-guided call, then a relative one of the same configuration on the same engine (step graphs on):
    the second equals the same call on a fresh engine, bit for bit"""
    w, x_obs, _, kw_joint, space_abs = joint_case()
    space_rel = C.JointSpace(space_abs.mean, space_abs.std, abs_3d=False)
    kw_joint["y"]["joint_guidance_weight"] = 0.005
    run_ddim(w, kw_joint, x_obs, space_abs)
    rel_after_abs = run_ddim(w, kw_joint, x_obs, space_rel)
    w2 = joint_case()[0]
    rel_fresh = run_ddim(w2, kw_joint, x_obs, space_rel)
    assert torch.equal(rel_after_abs, rel_fresh)
    assert not torch.equal(rel_fresh, run_ddim(w2, kw_joint, x_obs, space_abs))


def test_refusals():
    w, x_obs, _, kw_joint, space = joint_case()
    d = C.create_gaussian_diffusion(timestep_respacing="ddim50")
    with pytest.raises(NotImplementedError, match="joint_space"):
        d.ddim_sample_loop(w, (2, 263, 1, 196), model_kwargs=kw_joint, skip_timesteps=44)
    d.joint_space = space
    d.window = C.Window(196, 0)
    with pytest.raises(NotImplementedError, match="windows"):
        d.ddim_sample_loop(w, (2, 263, 1, 196), model_kwargs=kw_joint, skip_timesteps=44)
    # MDM_UNET at bf16x3 and bf16: the reconstruction-guidance refusal
    m, wu, sd, xo, kf, y, c, g = TG.setup(2, seed=23)
    add_joint(y, 2, TG.L, True, 0.1, 0, seed=12)
    y["reconstruction_guidance"] = False
    for precision in (C.PRECISION_BF16X3, C.PRECISION_BF16):
        du = C.create_gaussian_diffusion(timestep_respacing="ddim50")
        du.precision, du.joint_space = precision, space
        with pytest.raises(RuntimeError, match="transformer"):
            du.ddim_sample_loop(wu, (2, TG.D, 1, TG.L), model_kwargs={"y": y}, skip_timesteps=48)

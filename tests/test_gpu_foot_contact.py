"""GPU: foot-contact guidance -- the FC instance of the joint seed kernel (cmdi_foot_contact_seed) against fp64 autograd
of oracle/foot_contact_oracle.py, the guided input-VJP with the contact term (alone and with joint targets), guided
loops against the restatement, and the invariants of the step path (graph replay, generators, calls after
foot-contact-guided ones, launch counts, refusals)."""
import pytest
import torch

import condmdi_b200 as C
import test_gpu_bf16 as TB
import test_gpu_dpm_solver as TD
import test_gpu_joint_guidance as TJ
import test_gpu_keyframe_cfg as TK
import test_gpu_transformer_guidance as TT
import test_gpu_unet_guidance as TG
from condmdi_b200.engine import foot_contact_seed
from oracle import condmdi_oracle as O
from oracle import dpm_solver_oracle as S
from oracle import foot_contact_oracle as FC
from oracle import joint_guidance_oracle as J
from oracle import keyframe_cfg_oracle as K
from oracle import repaint_oracle as R

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
# joint guidance's gate for the seed kernel (fp32 FK and block scans over <= 224 frames); measured on H100 for the
# foot-contact instance: at most 1.3e-7 (abs3d) and 7.7e-7 (relative, L = 224)
SEED_GATE = TJ.SEED_GATE


def stats(seed, B=2, L=196):
    """joint_guidance_oracle.inputs' statistics and targets, with contact channels whose labels a denoiser output cannot
    move across 0.5 (std 1e-6): feet 7, 10 and 8 in contact on every frame, foot 11 on none.  Held fixed, the labels are
    the same in the engine and in an oracle whose x0_hat differs from it by rounding."""
    mean, std, jt, jm, g = J.inputs(B, L, seed=seed)
    std[259:263] = 1e-6
    mean[259:263] = torch.tensor([1.0, 1.0, 1.0, 0.0])
    return mean, std, jt, jm, g


def ragged(B, L, seed):
    lengths = torch.randint(max(1, L // 4), L + 1, (B,), generator=torch.Generator().manual_seed(seed))
    lengths[0] = L
    return torch.arange(L)[None] < lengths[:, None]


# ---------------------------------------------------------------------------------------------------------------------
# the seed kernel
# ---------------------------------------------------------------------------------------------------------------------
def fp64_seed(x0, mean, std, abs_3d, valid, c_c, target=None, mask=None, c_j=0.0):
    """c_j dL_j/dx0 + c_c dL_c/dx0 in fp64 on the GPU, with the contact labels formed in fp32 (the kernel's rounding of
    x0 * std + mean, so that a label near 0.5 falls on the same side)"""
    w = FC.contact_weights(x0.to(DEV), mean.to(DEV), std.to(DEV), valid.to(DEV)).double()
    d = lambda v: v.to(DEV).double()  # noqa: E731
    with torch.enable_grad():
        z = d(x0).requires_grad_(True)
        P = J.joint_positions(z, d(mean), d(std), abs_3d)
        feet = P[:, :, list(FC.FOOT_JOINTS)]
        loss = c_c * ((feet[:, 1:] - feet[:, :-1]).square().sum(-1) * w).sum()
        if target is not None:
            loss = loss + c_j * ((P - d(target)).square() * mask.to(DEV)).sum()
        return torch.autograd.grad(loss, z)[0].cpu()


@pytest.mark.parametrize("abs_3d", [True, False], ids=["abs3d", "rel"])
@pytest.mark.parametrize("B,L", [(2, 196), (2, 224), (2, 2), (64, 196)])
def test_contact_seed_kernel(abs_3d, B, L):
    """c_c = 1 alone, and 0.3 L_c + 0.7 L_j, over ragged masks, with labels exactly at 0.5 on every 7th frame"""
    mean, std, x0, g = FC.inputs(B, L, seed=B * 1000 + L + abs_3d)
    x0[:, 259:263, 0, ::7] = 0.0   # de-normalises to exactly 0.5: not a contact
    _, _, jt, jm, _ = J.inputs(B, L, seed=7)
    valid = ragged(B, L, seed=L + B)
    if B > 2:
        valid[-1] = False          # the last sample has no valid frame
    exactly_half = (x0[:, 259:263, 0] * std[259:263, None] + mean[259:263, None] == 0.5)
    assert exactly_half.any()
    assert FC.contact_weights(x0, mean, std, valid).sum() > 0 or L == 2
    args = (mean.to(DEV), std.to(DEV), abs_3d, valid.to(DEV))
    for c_c, c_j, with_joint in ((1.0, 0.0, False), (0.3, 0.7, True)):
        tgt = dict(target=jt.to(DEV), mask=jm.to(DEV), c_j=c_j) if with_joint else {}
        got = foot_contact_seed(x0.to(DEV), *args, c_c=c_c, **tgt).cpu()
        want = fp64_seed(x0, mean, std, abs_3d, valid, c_c, jt if with_joint else None, jm, c_j)
        assert (got[:, 67:] == 0).all(), "channels >= 67 (the contact labels included) must be exact zeros"
        if B > 2 and not with_joint:
            assert (got[-1] == 0).all(), "a sample without valid frames must have a zero gradient"
        scale = want.abs().max().item()
        ratio = ((got.double() - want).abs().max() / max(scale, 1e-30)).item()
        print(f"[contact seed {'abs3d' if abs_3d else 'rel'} B={B} L={L} c_c={c_c} joint={with_joint}] "
              f"max|E-F| / max|F| = {ratio:.3e} (max|F| = {scale:.3e})")
        if scale == 0:
            assert (got == 0).all()
        else:
            assert ratio <= SEED_GATE


@pytest.mark.parametrize("abs_3d", [True, False], ids=["abs3d", "rel"])
def test_contact_seed_frame_major_and_limits(abs_3d):
    """the engine's layout equals the reference layout bit for bit (pad columns exact zeros; output prefilled with NaN);
    no label above 0.5, or no two consecutive valid frames: an exact zero"""
    B, L, ld = 3, 196, 264
    mean, std, x0, g = FC.inputs(B, L, seed=50)
    x0 = x0.to(DEV)
    rows = torch.full((B, L, ld), float("nan"), device=DEV)
    rows[:, :, :263] = x0[:, :, 0].transpose(1, 2)
    args = (mean.to(DEV), std.to(DEV), abs_3d)
    out = torch.full((B, L, ld), float("nan"), device=DEV)
    got = foot_contact_seed(rows, *args, ld=ld, out=out)
    ref = foot_contact_seed(x0, *args)
    assert (got[:, :, 67:] == 0).all()
    assert torch.equal(got[:, :, :263], ref[:, :, 0].transpose(1, 2))
    assert ref.abs().max() > 0
    no_contact = mean.clone()
    no_contact[259:263] = -100.0
    assert (foot_contact_seed(x0, no_contact.to(DEV), std.to(DEV), abs_3d) == 0).all()
    alternate = (torch.arange(L) % 2 == 0).expand(B, L).to(DEV)
    assert (foot_contact_seed(x0, *args, valid=alternate) == 0).all()


# ---------------------------------------------------------------------------------------------------------------------
# input-VJP with the contact term per pass
# ---------------------------------------------------------------------------------------------------------------------
def fc_loss(hat, mean, std, abs_3d, valid, c_c, jt=None, jm=None, c_j=0.0):
    d = lambda v: v.to(hat)  # noqa: E731
    loss = c_c * FC.contact_loss(hat, d(mean), d(std), abs_3d, valid.to(hat.device))
    if jt is not None:
        loss = loss + c_j * J.joint_loss(hat, d(jt), jm.to(hat.device), d(mean), d(std), abs_3d)
    return loss


def transformer_vjps(forward, x, t, mode, cond, scale, loss_of):
    """the pass gradients of loss_of(x0_hat) w.r.t. x, fp64 on the GPU: text (one conditional pass), uncond, or CFG"""
    z = x.detach().to(DEV).double().requires_grad_(True)
    cd = cond.to(DEV).double()
    if mode == "cfg":
        outs = [forward(z, t.to(DEV), cd, False), forward(z, t.to(DEV), cd, True)]
        hat = outs[1] + scale.to(DEV).double().view(-1, 1, 1, 1) * (outs[0] - outs[1])
    else:
        outs = [forward(z, t.to(DEV), cd, mode == "uncond")]
        hat = outs[0]
    seeds = torch.autograd.grad(loss_of(hat), outs, retain_graph=True)
    return torch.stack([torch.autograd.grad(o, z, s_, retain_graph=True)[0] for o, s_ in zip(outs, seeds)]).cpu()


@pytest.mark.parametrize("joint", [False, True], ids=["contact", "contact+joint"])
@pytest.mark.parametrize("mode", ["text", "uncond", "cfg"])
def test_transformer_contact_input_vjp(mode, joint):
    """bf16x3 and bf16 against the fp64 models A (bf16-rounded operands) and F (exact) at the guidance gates, relative
    representation with joint targets, abs_3d without (the transformer takes no keyframe input, so keyframe CFG is
    MDM_UNET's and is covered below)"""
    B, L = 2, 196
    m, sd = TB.module()
    x, xo, M, cond, scale = TT.vjp_case_inputs(263, L, B, seed=19)
    mean, std, jt, jm, _ = stats(5, B, L)
    valid = ragged(B, L, seed=3)
    abs_3d = not joint
    c_c, c_j = (0.05 if abs_3d else 0.002), (0.002 if joint else 0.0)
    sdd = {k: v.to(DEV).double() for k, v in sd.items()}
    loss_of = lambda hat: fc_loss(hat, mean, std, abs_3d, valid, c_c, jt if joint else None, jm, c_j)  # noqa: E731
    failures = []
    for t in (500, 30):
        tt = torch.full((B,), t)
        a, f = [transformer_vjps(lambda z, t_, c, u, q=q: TB.mdm_model(q, sdd, z, t_, c, u), x, tt, mode, cond, scale, loss_of)
                for q in (TB.bf16r, TB.exact)]
        for name, prec in (("bf16x3", C.PRECISION_BF16X3), ("bf16", C.PRECISION_BF16)):
            eng = m.engine_for(DEV, max_batch=B, precision=prec, nframes=L)
            got = eng.test_foot_contact_input_vjp(x, t, mean, std, abs_3d, c_c, valid=valid,
                                                  joint_target=jt if joint else None, joint_mask=jm if joint else None,
                                                  c_j=c_j, cond_emb=cond, uncond=mode == "uncond", cfg=mode == "cfg",
                                                  text_scale=scale if mode == "cfg" else None)
            assert got.shape == a.shape
            for k in range(got.shape[0]):
                try:
                    TB.gate(got[k], a[k], f[k], f"contact vjp {name} {mode} joint={joint} t={t} pass {k}", c=TT.GATES[name])
                except AssertionError as err:
                    failures.append(str(err))
    assert not failures, failures


def unet_vjps(sd, x, t, mode, xo, kf, cond, w_t, w_k, loss_of, autocast):
    """the pass gradients of loss_of(x0_hat) w.r.t. x, autograd after the forward under CUDA autocast (or fp32): text,
    uncond, CFG, or keyframe CFG's three passes"""
    sdd = {k: v.to(DEV) for k, v in sd.items()}
    dev = lambda v: None if v is None else v.to(DEV)  # noqa: E731
    x, xo, kf, cond = dev(x), dev(xo), dev(kf), dev(cond)
    tt = torch.full((x.shape[0],), int(t), device=DEV)
    z = x.detach().requires_grad_(True)
    with TG.ctx_of(autocast):
        if mode == "kfcfg":
            outs = K.passes(sdd, z, tt, O.Conditioning(cond_emb=cond, cfg=True, obs_x0=xo, obs_mask=kf))
        else:
            outs = [TG.UNET_FORWARD(sdd, z, tt, cond, mode == "uncond", xo, kf)]
            if mode == "cfg":
                outs.append(TG.UNET_FORWARD(sdd, z, tt, cond, True, xo, kf))
    with TG.ctx_of(False):
        if mode == "kfcfg":
            hat = K.combine(*outs, dev(w_t), dev(w_k))
        elif mode == "cfg":
            hat = outs[1] + (dev(w_t).view(-1, 1, 1, 1) * (outs[0] - outs[1]))
        else:
            hat = outs[0]
        hat = hat.float()
        seeds = torch.autograd.grad(loss_of(hat), outs, retain_graph=True)
        return torch.stack([torch.autograd.grad(o, z, s_, retain_graph=True)[0] for o, s_ in zip(outs, seeds)])


@pytest.mark.parametrize("joint", [False, True], ids=["contact", "contact+joint"])
@pytest.mark.parametrize("mode", ["text", "uncond", "cfg", "kfcfg"])
def test_unet_fp16_contact_input_vjp(mode, joint):
    """the keyframe-conditioned xl MDM_UNET at PRECISION_FP16 with reconstruction guidance too, against autograd after a
    CUDA-autocast forward (A) and an fp32 one (F), at test_gpu_unet_guidance.py's gates: text, uncond and CFG on
    test_gpu_joint_guidance.py's model and inputs, keyframe CFG's three passes on test_gpu_keyframe_cfg.py's.  Under CFG
    and keyframe CFG the max |E - A| is held to 1.5 |A - F| as test_gpu_keyframe_cfg.py holds its combined passes:
    measured on H100, 1.02-1.06 of max |A - F| for CFG at t = 500 (the means 0.88-0.90)"""
    B = 2
    kfcfg = mode == "kfcfg"
    if kfcfg:
        m, sd, cond = TK.text_model(B)
        x, xo, kf, w_t, w_k = TK.inputs(B, 13)
    else:
        m, sd = TG.module()
        x, xo, kf, cond, w_t = TG.inputs(B, seed=70 + B)
        w_k = None
    mean, std, jt, jm, _ = stats(6, B, TG.L)
    valid = ragged(B, TG.L, seed=4)
    c_r, c_c, c_j = 10.0, 0.05, (0.05 if joint else 0.0)

    def loss_of(hat):
        d = lambda v: v.to(DEV)  # noqa: E731
        return c_r * ((d(xo) - hat).square() * d(kf)).sum() + fc_loss(hat, mean, std, True, valid, c_c,
                                                                      jt if joint else None, jm, c_j)

    eng = m.engine_for(DEV, max_batch=3 if kfcfg else B, precision=C.PRECISION_FP16, nframes=TG.L)
    for t in (500, 30):
        got = eng.test_foot_contact_input_vjp(x, t, mean, std, True, c_c, valid=valid, joint_target=jt if joint else None,
                                              joint_mask=jm if joint else None, c_j=c_j, inpainted_motion=xo,
                                              inpainting_mask=kf, c_r=c_r, cond_emb=cond, uncond=mode == "uncond",
                                              cfg=mode in ("cfg", "kfcfg"),
                                              text_scale=w_t if mode in ("cfg", "kfcfg") else None, obs_x0=xo, obs_mask=kf,
                                              keyframe_scale=w_k if kfcfg else None)
        a, f = [unet_vjps(sd, x, t, mode, xo, kf, cond, w_t, w_k, loss_of, ac) for ac in (True, False)]
        assert got.shape == a.shape
        for p in range(got.shape[0]):
            TG.gate(got[p], a[p], f[p], f"unet fp16 contact vjp {mode} joint={joint} t={t} pass {p}",
                    track=1.5 if mode in ("cfg", "kfcfg") else 1.0)


# ---------------------------------------------------------------------------------------------------------------------
# loops against the restatement with its model evaluated on the GPU
# ---------------------------------------------------------------------------------------------------------------------
def add_contact(y, B, L, abs_3d, weight, stop, seed, joint=None):
    """y['foot_contact_*'] (and y['joint_*'] with joint = (weight, stop)); the JointSpace and the oracle's terms"""
    mean, std, jt, jm, _ = stats(seed, B, L)
    y.update(foot_contact_guidance=True, foot_contact_weight=weight, foot_contact_gradient_schedule=None,
             stop_footcontact_at=stop, diffusion_steps=1000)
    fc = FC.FootContactTerm(mean, std, abs_3d, weight, None, 1000, stop)
    j = None
    if joint is not None:
        y.update(joint_guidance=True, joint_target=jt.to(DEV), joint_target_mask=jm.to(DEV), joint_guidance_weight=joint[0],
                 joint_gradient_schedule=None, stop_jointguidance_at=joint[1])
        j = J.JointTerm(jt, jm, mean, std, abs_3d, joint[0], None, 1000, joint[1])
    return C.JointSpace(mean, std, abs_3d), fc, j


def test_bf16x3_ddim50_tail_contact_b64():
    """ddim50 t = 5 .. 0 at B = 64: CFG, imputation, reconstruction guidance down to t = 3, foot contact down to t = 2"""
    w, sd, x_obs, kw, tape, run, B, n = TT.ddim50_b64_case()
    space, fc, _ = add_contact(kw["y"], B, 196, True, 0.1, 2, seed=8)
    d = C.create_gaussian_diffusion(timestep_respacing="ddim50")
    d.joint_space = space
    d.noise_tape = tape.to(DEV)
    got = TT.engine_steps(d.ddim_sample_loop_progressive(w, (B, 263, 1, 196), model_kwargs=kw, skip_timesteps=44,
                                                         init_image=x_obs.to(DEV)), n)
    with FC.foot_contact_guided(fc):
        want = TT.oracle_loop(sd, run, exact_fp32=True)
    TJ.gate_fp32(got, want, "bf16x3 B=64 ddim50 contact")


@pytest.mark.parametrize("abs_3d", [True, False], ids=["abs3d", "rel"])
def test_bf16x3_ddpm_tail_contact_and_joint_b2(abs_3d):
    """t = 49 .. 46 of the 1000-step schedule, every step guided by all three terms"""
    B, n = 2, 4
    w, sd, x_obs, kw, c, g = TT.loop_case(B, seed=67, stop_recguidance_at=0)
    wt = 0.1 if abs_3d else 0.005
    space, fc, j = add_contact(kw["y"], B, 196, abs_3d, wt, 0, seed=9, joint=(wt, 0))
    tape = torch.randn(1 + n, B, 263, 1, 196, generator=g)
    d = C.create_gaussian_diffusion()
    d.joint_space = space
    d.noise_tape = tape.to(DEV)
    got = TT.engine_steps(d.p_sample_loop_progressive(w, (B, 263, 1, 196), model_kwargs=kw, skip_timesteps=950,
                                                      init_image=x_obs.to(DEV)), n)
    with FC.foot_contact_guided(fc, j):
        want = TT.oracle_loop(sd, lambda: O.sample_loop(sd, O.make_tables(""), (B, 263, 1, 196), c, tape, "ddpm",
                                                        skip_timesteps=950, init_image=x_obs, max_steps=n, return_all=True),
                              exact_fp32=True)
    TJ.gate_fp32(got, want, f"bf16x3 B=2 ddpm contact+joint {'abs3d' if abs_3d else 'rel'}")


# With three feet in contact on every valid frame the contact term is dense: these two loops guide with a fifth of the
# weight, on the cases (seeds) of test_gpu_joint_guidance.py's DPM-Solver++ and RePaint loops
LIGHT = 0.02


def test_bf16x3_dpm_solver_order2_contact_b2():
    """DPM-Solver++ order 2 on ddim50, t = 5 .. 0, every step guided, with the samples' atol scaled as
    test_gpu_joint_guidance.py scales it"""
    B, n = 2, 6
    w, sd, x_obs, kw, c, g = TT.loop_case(B, seed=65, stop_recguidance_at=0)
    space, fc, _ = add_contact(kw["y"], B, 196, True, LIGHT, 0, seed=13)
    tape = torch.randn(1, B, 263, 1, 196, generator=g)
    d = C.create_gaussian_diffusion(timestep_respacing="ddim50")
    d.joint_space = space
    d.noise_tape = tape.to(DEV)
    got = TT.engine_steps(d.dpm_solver_sample_loop_progressive(w, (B, 263, 1, 196), model_kwargs=kw, skip_timesteps=44,
                                                               init_image=x_obs.to(DEV), order=2), n)
    with FC.foot_contact_guided(fc):
        want = TT.oracle_loop(sd, lambda: S.dpm_solver_sample_loop(sd, O.make_tables("ddim50"), (B, 263, 1, 196), c, tape, 2,
                                                                   skip_timesteps=44, init_image=x_obs, return_all=True),
                              exact_fp32=True)
    TJ.gate_fp32(got, want, "bf16x3 B=2 dpm-solver++ order 2 contact", sample_atol=TD.unet_gate("ddim50", 44, 2)["atol"])


def test_bf16x3_repaint_walk_contact_b2():
    """RePaint on ddim50 from t = 5, jump_length 2, jump_n_sample 2, foot contact stopping at 2"""
    B, skip, jl, r = 2, 44, 2, 2
    w, sd, x_obs, kw, c, g = TT.loop_case(B, seed=66, stop_recguidance_at=0)
    space, fc, _ = add_contact(kw["y"], B, 196, True, LIGHT, 2, seed=14)
    n_ops = len(C.diffusion._repaint_walk(49 - skip, jl, r))
    tape = torch.randn(1 + n_ops, B, 263, 1, 196, generator=g)
    d = C.create_gaussian_diffusion(timestep_respacing="ddim50")
    d.joint_space = space
    d.noise_tape = tape.to(DEV)
    got = d.repaint_sample_loop(w, (B, 263, 1, 196), model_kwargs=kw, skip_timesteps=skip, init_image=x_obs.to(DEV),
                                jump_length=jl, jump_n_sample=r)
    with FC.foot_contact_guided(fc):
        want = TT.oracle_loop(sd, lambda: R.repaint_sample_loop(sd, O.make_tables("ddim50"), (B, 263, 1, 196), c, tape, jl, r,
                                                                skip_timesteps=skip, init_image=x_obs), exact_fp32=True)
    TJ.gate_fp32([{"sample": got, "pred_xstart": got}], [{"sample": want, "pred_xstart": want}], "bf16x3 B=2 repaint contact")


def test_unet_fp16_ddpm_tail_contact_b2():
    B = 2
    m, w, sd, x_obs, kf, y, c, g = TG.setup(B, seed=24)
    y.update(imputate=1, stop_imputation_at=1, replacement_distribution="conditional")
    c.imputate, c.stop_imputation_at = True, 1
    space, fc, _ = add_contact(y, B, TG.L, True, 0.1, 0, seed=10)
    tape = torch.randn(5, B, TG.D, 1, TG.L, generator=g)
    d = C.create_gaussian_diffusion()
    d.precision = C.PRECISION_FP16
    d.joint_space = space
    d.noise_tape = tape.to(DEV)
    kw = {"y": y, "obs_x0": x_obs.to(DEV), "obs_mask": kf.to(DEV)}
    got = d.p_sample_loop(w, (B, TG.D, 1, TG.L), model_kwargs=kw, skip_timesteps=996, init_image=x_obs.to(DEV))
    with FC.foot_contact_guided(fc):
        a, f = TG.oracle_loop(sd, lambda: O.sample_loop(sd, O.make_tables(""), (B, TG.D, 1, TG.L), c, tape, "ddpm",
                                                        skip_timesteps=996, init_image=x_obs))
    TG.gate(got, a, f, "UNet fp16 B=2 ddpm 4-step tail, cfg + imputation + recon + foot contact", track=1.5)


# ---------------------------------------------------------------------------------------------------------------------
# invariants
# ---------------------------------------------------------------------------------------------------------------------
def contact_case(B=2, seed=64, alone=False):
    """TJ.joint_case's model and keyframes, with (kw_recon, kw_joint, kw_contact) model_kwargs; alone: the contact
    term without keyframes or reconstruction guidance (plain text-to-motion with CFG)"""
    w, x_obs, kw_recon, kw_joint, space_j = TJ.joint_case(B, seed)
    y = dict(kw_recon["y"])
    if alone:
        y = {k: v for k, v in y.items() if k in ("text", "text_scale", "mask")}
    space, _, _ = add_contact(y, B, 196, True, 0.1, 2, seed=11)
    return w, x_obs, kw_recon, kw_joint, {"y": y}, space


def test_graph_replay_generator_and_other_calls_are_unchanged():
    w, x_obs, kw_recon, kw_joint, kw_fc, space = contact_case()
    unguided = {"y": {k: v for k, v in kw_recon["y"].items() if k != "reconstruction_guidance"}}
    before = [TJ.run_ddim(w, kw, x_obs, sp) for kw, sp in ((unguided, None), (kw_recon, None), (kw_joint, space))]
    graph = TJ.run_ddim(w, kw_fc, x_obs, space)
    direct = TJ.run_ddim(w, kw_fc, x_obs, space, use_graph=False)
    gen = TJ.run_ddim(w, kw_fc, x_obs, space, progressive=True)
    assert torch.equal(graph, direct), "graph replay differs from direct launches"
    assert torch.equal(graph, gen), "the generator differs from the fused loop"
    after = [TJ.run_ddim(w, kw, x_obs, sp) for kw, sp in ((unguided, None), (kw_recon, None), (kw_joint, space))]
    w2 = TJ.joint_case()[0]
    fresh = [TJ.run_ddim(w2, kw, x_obs, sp) for kw, sp in ((unguided, None), (kw_recon, None), (kw_joint, space))]
    for b, a_, f_, what in zip(before, after, fresh, ("unguided", "reconstruction-only", "joint-only")):
        assert torch.equal(a_, b) and torch.equal(a_, f_), f"a {what} loop changed after foot-contact-guided calls"
    assert not torch.equal(graph, before[1]), "foot-contact guidance had no effect"


def test_contact_alone_guides_plain_text_to_motion():
    """no keyframes (M = 0): graph replay equals direct launches, and the result differs from the unguided loop"""
    w, x_obs, _, _, kw_fc, space = contact_case(alone=True)
    graph = TJ.run_ddim(w, kw_fc, x_obs, space)
    direct = TJ.run_ddim(w, kw_fc, x_obs, space, use_graph=False)
    plain = TJ.run_ddim(w, {"y": {k: v for k, v in kw_fc["y"].items() if not k.startswith(("foot_", "stop_foot"))}}, x_obs)
    assert torch.equal(graph, direct)
    assert torch.isfinite(graph).all() and not torch.equal(graph, plain)


def test_launch_counts():
    """a foot-contact-guided step launches what a joint-guided step launches (128 + the joint seed kernel), with or
    without joint targets; the per-step count is the difference between a 6-step and a 3-step call"""
    w, x_obs, kw_recon, kw_joint, kw_fc, space = contact_case()
    kw_both = {"y": dict(kw_fc["y"], **{k: v for k, v in kw_joint["y"].items() if k.startswith(("joint_", "stop_joint"))})}
    eng = C.resolve_model(w)[0].engine_for(DEV, max_batch=2, precision=C.PRECISION_BF16X3, nframes=196)

    def count(kw, skip, sp=None):
        n0 = eng.launch_count
        TJ.run_ddim(w, kw, x_obs, sp, skip=skip)
        return eng.launch_count - n0

    per_step = {}
    for name, kw, sp in (("recon+joint", kw_joint, space), ("recon+contact", kw_fc, space), ("recon+joint+contact", kw_both, space)):
        count(kw, 44, sp)  # capture the step graphs first
        per_step[name] = (count(kw, 44, sp) - count(kw, 47, sp)) / 3
    print(f"[launches per guided step] {per_step}")
    assert per_step["recon+joint"] == 59 + 1 + 68 + 1
    assert per_step["recon+contact"] == per_step["recon+joint"]
    assert per_step["recon+joint+contact"] == per_step["recon+joint"]


def test_refusals():
    w, x_obs, _, _, kw_fc, space = contact_case()
    d = C.create_gaussian_diffusion(timestep_respacing="ddim50")
    with pytest.raises(NotImplementedError, match="joint_space"):
        d.ddim_sample_loop(w, (2, 263, 1, 196), model_kwargs=kw_fc, skip_timesteps=44)
    d.joint_space = space
    d.window = C.Window(196, 0)
    with pytest.raises(NotImplementedError, match="windows"):
        d.ddim_sample_loop(w, (2, 263, 1, 196), model_kwargs=kw_fc, skip_timesteps=44)
    d.window = None
    bad = {"y": dict(kw_fc["y"], foot_contact_weight=None)}
    with pytest.raises(ValueError, match="foot_contact_weight"):
        d.ddim_sample_loop(w, (2, 263, 1, 196), model_kwargs=bad, skip_timesteps=44)
    # MDM_UNET at bf16x3 and bf16: the reconstruction-guidance refusal, message unchanged
    m, wu, sd, xo, kf, y, c, g = TG.setup(2, seed=25)
    add_contact(y, 2, TG.L, True, 0.1, 0, seed=12)
    y["reconstruction_guidance"] = False
    for precision in (C.PRECISION_BF16X3, C.PRECISION_BF16):
        du = C.create_gaussian_diffusion(timestep_respacing="ddim50")
        du.precision, du.joint_space = precision, space
        with pytest.raises(RuntimeError, match="transformer"):
            du.ddim_sample_loop(wu, (2, TG.D, 1, TG.L), model_kwargs={"y": y}, skip_timesteps=48)

"""GPU: obstacle-avoidance guidance -- the obstacle instances of the joint seed kernel (cmdi_obstacle_seed) against fp64
autograd of oracle/obstacle_oracle.py (alone and with the joint and foot-contact terms), the guided input-VJP with the
obstacle term, guided loops against the restatement, and the invariants of the step path (graph replay, generators,
calls after obstacle-guided ones, launch counts, refusals)."""
import pytest
import torch

import condmdi_b200 as C
import test_gpu_bf16 as TB
import test_gpu_dpm_solver as TD
import test_gpu_foot_contact as TF
import test_gpu_joint_guidance as TJ
import test_gpu_transformer_guidance as TT
import test_gpu_unet_guidance as TG
from condmdi_b200.engine import obstacle_seed
from oracle import condmdi_oracle as O
from oracle import dpm_solver_oracle as S
from oracle import foot_contact_oracle as FC
from oracle import joint_guidance_oracle as J
from oracle import obstacle_oracle as OB
from oracle import repaint_oracle as R

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
# joint guidance's gate for the seed kernel (fp32 FK and block scans over <= 224 frames)
SEED_GATE = TJ.SEED_GATE
# the obstacle term alone in the relative representation: the heading is a prefix sum of angular velocities (tens of
# radians over 200 frames of standard-normal features), so its fp32 rounding (~1e-6 rad) turns every later root step,
# the root carries absolute errors ~1e-5 over a walk of ~10, and the term's direction (P - c) / |P - c| divides them by
# a distance below r (~0.3 here).  Measured on H100: at most 5.2e-5.  Every other case is held to SEED_GATE.
REL_OBSTACLE_GATE = 1e-4


# ---------------------------------------------------------------------------------------------------------------------
# the seed kernel
# ---------------------------------------------------------------------------------------------------------------------
def fp64_seed(x0, mean, std, abs_3d, obstacles, joints, valid, c_o, c_c=0.0, target=None, mask=None, c_j=0.0):
    """c_j dL_j/dx0 + c_c dL_c/dx0 + c_o dL_o/dx0 in fp64 on the GPU (contact labels formed in fp32, as the kernel)"""
    d = lambda v: v.to(DEV).double()  # noqa: E731
    w = FC.contact_weights(x0.to(DEV), mean.to(DEV), std.to(DEV), valid.to(DEV)).double()
    with torch.enable_grad():
        z = d(x0).requires_grad_(True)
        loss = c_o * OB.obstacle_loss(z, d(mean), d(std), abs_3d, d(obstacles), joints, valid.to(DEV))
        P = J.joint_positions(z, d(mean), d(std), abs_3d)
        if c_c:
            feet = P[:, :, list(FC.FOOT_JOINTS)]
            loss = loss + c_c * ((feet[:, 1:] - feet[:, :-1]).square().sum(-1) * w).sum()
        if target is not None:
            loss = loss + c_j * ((P - d(target)).square() * mask.to(DEV)).sum()
        return torch.autograd.grad(loss, z)[0].cpu()


@pytest.mark.parametrize("abs_3d", [True, False], ids=["abs3d", "rel"])
@pytest.mark.parametrize("B,L,K,joints", [(2, 196, 1, (0,)), (2, 224, 16, (0, 7, 10, 8, 11, 21)), (2, 2, 3, (0, 15)),
                                          (64, 196, 8, tuple(range(22)))])
def test_obstacle_seed_kernel(abs_3d, B, L, K, joints):
    """c_o = 1 alone; 0.5 L_o + 0.3 L_c + 0.2 L_j; per-sample obstacles with radius-0 padding rows, over ragged masks"""
    pad = 1 if 1 < K < 16 else 0
    mean, std, x0, obstacles, _ = OB.inputs(B, L, seed=B * 1000 + L + abs_3d, K=K - pad, joints=joints, abs_3d=abs_3d,
                                            pad=pad)
    fmean, fstd, jt, jm, _ = TF.stats(7, B, L)
    mean[259:263], std[259:263] = fmean[259:263], fstd[259:263]
    valid = TF.ragged(B, L, seed=L + B)
    if B > 2:
        valid[-1] = False          # the last sample has no valid frame
    assert OB.obstacle_loss(x0.double(), mean.double(), std.double(), abs_3d, obstacles.double(), joints, valid) > 0 or L == 2
    args = (mean.to(DEV), std.to(DEV), abs_3d, obstacles.to(DEV))
    mask = OB.joint_mask(joints)
    for c_o, c_c, c_j in ((1.0, 0.0, 0.0), (0.5, 0.3, 0.2)):
        extra = dict(foot_contact=True, c_c=c_c, target=jt.to(DEV), mask=jm.to(DEV), c_j=c_j) if c_c else {}
        got = obstacle_seed(x0.to(DEV), *args, obstacle_joints=mask, c_o=c_o, valid=valid.to(DEV), **extra).cpu()
        want = fp64_seed(x0, mean, std, abs_3d, obstacles, joints, valid, c_o, c_c, jt if c_c else None, jm, c_j)
        assert (got[:, 67:] == 0).all(), "channels >= 67 must be exact zeros"
        if B > 2 and not c_c:
            assert (got[-1] == 0).all(), "a sample without valid frames must have a zero gradient"
        scale = want.abs().max().item()
        ratio = ((got.double() - want).abs().max() / max(scale, 1e-30)).item()
        print(f"[obstacle seed {'abs3d' if abs_3d else 'rel'} B={B} L={L} K={K} |S|={len(joints)} c=({c_o}, {c_c}, {c_j})] "
              f"max|E-F| / max|F| = {ratio:.3e} (max|F| = {scale:.3e})")
        if scale == 0:
            assert (got == 0).all()
        else:
            assert ratio <= (REL_OBSTACLE_GATE if not abs_3d and not c_c else SEED_GATE)


@pytest.mark.parametrize("abs_3d", [True, False], ids=["abs3d", "rel"])
def test_obstacle_seed_frame_major_zero_radii_and_subgradients(abs_3d):
    """the engine's layout equals the reference layout bit for bit (pad columns exact zeros; output prefilled with NaN);
    radii all 0 (also on the joints themselves) or no obstacle at all: an exact zero; distance 0 and distance r give
    torch's subgradients"""
    B, L, ld = 3, 196, 264
    mean, std, x0, obstacles, _ = OB.inputs(B, L, seed=50, K=5, abs_3d=abs_3d)
    x0 = x0.to(DEV)
    rows = torch.full((B, L, ld), float("nan"), device=DEV)
    rows[:, :, :263] = x0[:, :, 0].transpose(1, 2)
    args = (mean.to(DEV), std.to(DEV), abs_3d)
    out = torch.full((B, L, ld), float("nan"), device=DEV)
    got = obstacle_seed(rows, *args, obstacles.to(DEV), ld=ld, out=out)
    ref = obstacle_seed(x0, *args, obstacles.to(DEV))
    assert (got[:, :, 67:] == 0).all()
    assert torch.equal(got[:, :, :263], ref[:, :, 0].transpose(1, 2))
    assert ref.abs().max() > 0
    P = J.joint_positions(x0.cpu().double(), mean.double(), std.double(), abs_3d)[..., [0, 2]].float()
    zero_r = torch.zeros(B, 16, 3)
    zero_r[:, :, :2] = P[:, :16, 0]                                # centred on the pelvis of frames 0 .. 15
    assert (obstacle_seed(x0, *args, zero_r.to(DEV), obstacle_joints=(1 << 22) - 1) == 0).all()
    assert (obstacle_seed(x0, *args, torch.zeros(B, 0, 3, device=DEV)) == 0).all()
    if abs_3d:  # mean 0, std 1: the pelvis XZ of frame f is x0[:, 1:3, 0, f]
        z0 = torch.zeros(1, 263, 1, 4, device=DEV)
        z0[0, 1, 0] = torch.tensor([0.5, 2.0, -3.0, 8.0])
        z0[0, 2, 0] = torch.tensor([0.25, -1.0, 4.0, 8.0])
        m0, s0 = torch.zeros(263, device=DEV), torch.ones(263, device=DEV)
        on = obstacle_seed(z0, m0, s0, True, torch.tensor([[[0.5, 0.25, 1.0]]], device=DEV))
        assert (on == 0).all()                                     # distance 0: (-0, -0), compared by value
        at_r = obstacle_seed(z0, m0, s0, True, torch.tensor([[[1.25, -2.0, 1.25]]], device=DEV)).cpu()
        want = -torch.tensor([0.75, 1.0]) / 1.25 / 4
        assert torch.allclose(at_r[0, 1:3, 0, 1], want, rtol=1e-6, atol=0)


# ---------------------------------------------------------------------------------------------------------------------
# input-VJP with the obstacle term per pass
# ---------------------------------------------------------------------------------------------------------------------
def ob_loss(hat, mean, std, abs_3d, obstacles, joints, valid, c_o, c_c=0.0, jt=None, jm=None, c_j=0.0):
    d = lambda v: v.to(hat)  # noqa: E731
    loss = c_o * OB.obstacle_loss(hat, d(mean), d(std), abs_3d, d(obstacles), joints, valid.to(hat.device))
    if c_c:
        loss = loss + TF.fc_loss(hat, mean, std, abs_3d, valid, c_c, jt, jm, c_j)
    return loss


@pytest.mark.parametrize("combo", ["obstacle", "obstacle+contact+joint"])
@pytest.mark.parametrize("mode", ["text", "cfg"])
def test_transformer_obstacle_input_vjp(mode, combo):
    """bf16x3 and bf16 against the fp64 models A (bf16-rounded operands) and F (exact) at the guidance gates, abs_3d with
    the pelvis alone, relative with three joints and the contact and joint terms"""
    B, L = 2, 196
    m, sd = TB.module()
    x, xo, M, cond, scale = TT.vjp_case_inputs(263, L, B, seed=19)
    mean, std, jt, jm, _ = TF.stats(5, B, L)
    valid = TF.ragged(B, L, seed=3)
    full = combo != "obstacle"
    abs_3d = not full
    joints = (0, 10, 20) if full else (0,)
    # large cylinders around the origin: most frames of x0_hat are inside one
    obstacles = torch.tensor([[0.0, 0.0, 3.0], [0.4, -0.3, 1.5], [5.0, 5.0, 0.0]]).expand(B, -1, -1).contiguous()
    c_o, c_c, c_j = 2.0, (0.002 if full else 0.0), (0.002 if full else 0.0)
    sdd = {k: v.to(DEV).double() for k, v in sd.items()}
    loss_of = lambda hat: ob_loss(hat, mean, std, abs_3d, obstacles, joints, valid, c_o, c_c,  # noqa: E731
                                  jt if full else None, jm, c_j)
    failures = []
    for t in (500, 30):
        tt = torch.full((B,), t)
        a, f = [TF.transformer_vjps(lambda z, t_, c, u, q=q: TB.mdm_model(q, sdd, z, t_, c, u), x, tt, mode, cond, scale,
                                    loss_of) for q in (TB.bf16r, TB.exact)]
        assert f.abs().max() > 0
        for name, prec in (("bf16x3", C.PRECISION_BF16X3), ("bf16", C.PRECISION_BF16)):
            eng = m.engine_for(DEV, max_batch=B, precision=prec, nframes=L)
            got = eng.test_obstacle_input_vjp(x, t, mean, std, abs_3d, obstacles, c_o, OB.joint_mask(joints), valid=valid,
                                              foot_contact=full, c_c=c_c, joint_target=jt if full else None,
                                              joint_mask=jm if full else None, c_j=c_j, cond_emb=cond, cfg=mode == "cfg",
                                              text_scale=scale if mode == "cfg" else None)
            assert got.shape == a.shape
            for k in range(got.shape[0]):
                try:
                    TB.gate(got[k], a[k], f[k], f"obstacle vjp {name} {mode} {combo} t={t} pass {k}", c=TT.GATES[name])
                except AssertionError as err:
                    failures.append(str(err))
    assert not failures, failures


@pytest.mark.parametrize("mode", ["text", "cfg", "kfcfg"])
def test_unet_fp16_obstacle_input_vjp(mode):
    """the keyframe-conditioned xl MDM_UNET at PRECISION_FP16 with reconstruction guidance too, against autograd after a
    CUDA-autocast forward (A) and an fp32 one (F), at test_gpu_foot_contact.py's gates"""
    B = 2
    kfcfg = mode == "kfcfg"
    if kfcfg:
        import test_gpu_keyframe_cfg as TK
        m, sd, cond = TK.text_model(B)
        x, xo, kf, w_t, w_k = TK.inputs(B, 13)
    else:
        m, sd = TG.module()
        x, xo, kf, cond, w_t = TG.inputs(B, seed=70 + B)
        w_k = None
    mean, std, _, _, _ = TF.stats(6, B, TG.L)
    valid = TF.ragged(B, TG.L, seed=4)
    obstacles = torch.tensor([[[0.0, 0.0, 3.0], [0.5, 0.5, 1.0]], [[0.2, -0.1, 2.0], [0.0, 0.0, 0.0]]])
    c_r, c_o = 10.0, 5.0

    def loss_of(hat):
        d = lambda v: v.to(DEV)  # noqa: E731
        return c_r * ((d(xo) - hat).square() * d(kf)).sum() + ob_loss(hat, mean, std, True, obstacles, (0, 12), valid, c_o)

    eng = m.engine_for(DEV, max_batch=3 if kfcfg else B, precision=C.PRECISION_FP16, nframes=TG.L)
    for t in (500, 30):
        got = eng.test_obstacle_input_vjp(x, t, mean, std, True, obstacles, c_o, OB.joint_mask((0, 12)), valid=valid,
                                          inpainted_motion=xo, inpainting_mask=kf, c_r=c_r, cond_emb=cond,
                                          cfg=mode in ("cfg", "kfcfg"), text_scale=w_t if mode in ("cfg", "kfcfg") else None,
                                          obs_x0=xo, obs_mask=kf, keyframe_scale=w_k if kfcfg else None)
        a, f = [TF.unet_vjps(sd, x, t, mode, xo, kf, cond, w_t, w_k, loss_of, ac) for ac in (True, False)]
        assert got.shape == a.shape
        for p in range(got.shape[0]):
            TG.gate(got[p], a[p], f[p], f"unet fp16 obstacle vjp {mode} t={t} pass {p}",
                    track=1.5 if mode in ("cfg", "kfcfg") else 1.0)


# ---------------------------------------------------------------------------------------------------------------------
# loops against the restatement with its model evaluated on the GPU
# ---------------------------------------------------------------------------------------------------------------------
def add_obstacles(y, B, L, abs_3d, weight, stop, seed, joints=(0,), contact=None, joint=None, as_list=False):
    """y['obstacle_*'] (GMD's obs_list form when as_list), and y['foot_contact_*'] / y['joint_*'] with contact / joint =
    (weight, stop); the JointSpace and the oracle's terms.  The cylinders are large and near the origin, so most frames
    of x0_hat are inside one."""
    mean, std, jt, jm, _ = TF.stats(seed, B, L)
    r = 1.5 if abs_3d else 4.0
    obstacles = torch.tensor([[0.0, 0.0, r], [0.3, -0.2, 0.5 * r], [9.0, 9.0, 0.0]]).expand(B, -1, -1).contiguous()
    obs_y = [((float(o[0]), float(o[1])), float(o[2])) for o in obstacles[0]] if as_list else obstacles.to(DEV)
    y.update(obstacle_guidance=True, obstacles=obs_y, obstacle_weight=weight, obstacle_gradient_schedule=None,
             stop_obstacleguidance_at=stop, obstacle_joints=list(joints), diffusion_steps=1000)
    ob = OB.ObstacleTerm(mean, std, obstacles, joints, abs_3d, weight, None, 1000, stop)
    fc = j = None
    if contact is not None:
        y.update(foot_contact_guidance=True, foot_contact_weight=contact[0], foot_contact_gradient_schedule=None,
                 stop_footcontact_at=contact[1])
        fc = FC.FootContactTerm(mean, std, abs_3d, contact[0], None, 1000, contact[1])
    if joint is not None:
        y.update(joint_guidance=True, joint_target=jt.to(DEV), joint_target_mask=jm.to(DEV), joint_guidance_weight=joint[0],
                 joint_gradient_schedule=None, stop_jointguidance_at=joint[1])
        j = J.JointTerm(jt, jm, mean, std, abs_3d, joint[0], None, 1000, joint[1])
    return C.JointSpace(mean, std, abs_3d), ob, fc, j


def test_bf16x3_ddim50_tail_obstacle_b64():
    """ddim50 t = 5 .. 0 at B = 64: CFG, imputation, reconstruction guidance down to t = 3, obstacles down to t = 2"""
    w, sd, x_obs, kw, tape, run, B, n = TT.ddim50_b64_case()
    space, ob, _, _ = add_obstacles(kw["y"], B, 196, True, 20.0, 2, seed=8, as_list=True)
    d = C.create_gaussian_diffusion(timestep_respacing="ddim50")
    d.joint_space = space
    d.noise_tape = tape.to(DEV)
    got = TT.engine_steps(d.ddim_sample_loop_progressive(w, (B, 263, 1, 196), model_kwargs=kw, skip_timesteps=44,
                                                         init_image=x_obs.to(DEV)), n)
    with OB.obstacle_guided(ob):
        want = TT.oracle_loop(sd, run, exact_fp32=True)
    TJ.gate_fp32(got, want, "bf16x3 B=64 ddim50 obstacle")


@pytest.mark.parametrize("abs_3d", [True, False], ids=["abs3d", "rel"])
def test_bf16x3_ddpm_tail_obstacle_contact_and_joint_b2(abs_3d):
    """t = 49 .. 46 of the 1000-step schedule, every step guided by all four terms, three joints in S"""
    B, n = 2, 4
    w, sd, x_obs, kw, c, g = TT.loop_case(B, seed=67, stop_recguidance_at=0)
    # the relative representation's root gradient sums the term over every later frame: a twentieth of the weight, as
    # the foot-contact loop scales its own
    wt = 0.1 if abs_3d else 0.005
    space, ob, fc, j = add_obstacles(kw["y"], B, 196, abs_3d, 20.0 if abs_3d else 1.0, 0, seed=9, joints=(0, 10, 15), contact=(wt, 0),
                                     joint=(wt, 0))
    tape = torch.randn(1 + n, B, 263, 1, 196, generator=g)
    d = C.create_gaussian_diffusion()
    d.joint_space = space
    d.noise_tape = tape.to(DEV)
    got = TT.engine_steps(d.p_sample_loop_progressive(w, (B, 263, 1, 196), model_kwargs=kw, skip_timesteps=950,
                                                      init_image=x_obs.to(DEV)), n)
    with OB.obstacle_guided(ob, fc, j):
        want = TT.oracle_loop(sd, lambda: O.sample_loop(sd, O.make_tables(""), (B, 263, 1, 196), c, tape, "ddpm",
                                                        skip_timesteps=950, init_image=x_obs, max_steps=n, return_all=True),
                              exact_fp32=True)
    TJ.gate_fp32(got, want, f"bf16x3 B=2 ddpm obstacle+contact+joint {'abs3d' if abs_3d else 'rel'}")


def test_bf16x3_dpm_solver_order2_obstacle_b2():
    """DPM-Solver++ order 2 on ddim50, t = 5 .. 0, every step guided"""
    B, n = 2, 6
    w, sd, x_obs, kw, c, g = TT.loop_case(B, seed=65, stop_recguidance_at=0)
    space, ob, _, _ = add_obstacles(kw["y"], B, 196, True, 20.0, 0, seed=13)
    tape = torch.randn(1, B, 263, 1, 196, generator=g)
    d = C.create_gaussian_diffusion(timestep_respacing="ddim50")
    d.joint_space = space
    d.noise_tape = tape.to(DEV)
    got = TT.engine_steps(d.dpm_solver_sample_loop_progressive(w, (B, 263, 1, 196), model_kwargs=kw, skip_timesteps=44,
                                                               init_image=x_obs.to(DEV), order=2), n)
    with OB.obstacle_guided(ob):
        want = TT.oracle_loop(sd, lambda: S.dpm_solver_sample_loop(sd, O.make_tables("ddim50"), (B, 263, 1, 196), c, tape, 2,
                                                                   skip_timesteps=44, init_image=x_obs, return_all=True),
                              exact_fp32=True)
    TJ.gate_fp32(got, want, "bf16x3 B=2 dpm-solver++ order 2 obstacle", sample_atol=TD.unet_gate("ddim50", 44, 2)["atol"])


def test_bf16x3_repaint_walk_obstacle_b2():
    """RePaint on ddim50 from t = 5, jump_length 2, jump_n_sample 2, obstacles stopping at 2"""
    B, skip, jl, r = 2, 44, 2, 2
    w, sd, x_obs, kw, c, g = TT.loop_case(B, seed=66, stop_recguidance_at=0)
    space, ob, _, _ = add_obstacles(kw["y"], B, 196, True, 20.0, 2, seed=14)
    n_ops = len(C.diffusion._repaint_walk(49 - skip, jl, r))
    tape = torch.randn(1 + n_ops, B, 263, 1, 196, generator=g)
    d = C.create_gaussian_diffusion(timestep_respacing="ddim50")
    d.joint_space = space
    d.noise_tape = tape.to(DEV)
    got = d.repaint_sample_loop(w, (B, 263, 1, 196), model_kwargs=kw, skip_timesteps=skip, init_image=x_obs.to(DEV),
                                jump_length=jl, jump_n_sample=r)
    with OB.obstacle_guided(ob):
        want = TT.oracle_loop(sd, lambda: R.repaint_sample_loop(sd, O.make_tables("ddim50"), (B, 263, 1, 196), c, tape, jl, r,
                                                                skip_timesteps=skip, init_image=x_obs), exact_fp32=True)
    TJ.gate_fp32([{"sample": got, "pred_xstart": got}], [{"sample": want, "pred_xstart": want}], "bf16x3 B=2 repaint obstacle")


def test_unet_fp16_ddpm_tail_obstacle_b2():
    B = 2
    m, w, sd, x_obs, kf, y, c, g = TG.setup(B, seed=24)
    y.update(imputate=1, stop_imputation_at=1, replacement_distribution="conditional")
    c.imputate, c.stop_imputation_at = True, 1
    space, ob, _, _ = add_obstacles(y, B, TG.L, True, 20.0, 0, seed=10, joints=(0, 3))
    tape = torch.randn(5, B, TG.D, 1, TG.L, generator=g)
    d = C.create_gaussian_diffusion()
    d.precision = C.PRECISION_FP16
    d.joint_space = space
    d.noise_tape = tape.to(DEV)
    kw = {"y": y, "obs_x0": x_obs.to(DEV), "obs_mask": kf.to(DEV)}
    got = d.p_sample_loop(w, (B, TG.D, 1, TG.L), model_kwargs=kw, skip_timesteps=996, init_image=x_obs.to(DEV))
    with OB.obstacle_guided(ob):
        a, f = TG.oracle_loop(sd, lambda: O.sample_loop(sd, O.make_tables(""), (B, TG.D, 1, TG.L), c, tape, "ddpm",
                                                        skip_timesteps=996, init_image=x_obs))
    TG.gate(got, a, f, "UNet fp16 B=2 ddpm 4-step tail, cfg + imputation + recon + obstacles", track=1.5)


# ---------------------------------------------------------------------------------------------------------------------
# invariants
# ---------------------------------------------------------------------------------------------------------------------
def obstacle_case(B=2, seed=64, alone=False):
    """TJ.joint_case's model and keyframes, with (kw_recon, kw_joint, kw_obstacle) model_kwargs; alone: the obstacle
    term without keyframes or reconstruction guidance (plain text-to-motion with CFG)"""
    w, x_obs, kw_recon, kw_joint, space_j = TJ.joint_case(B, seed)
    y = dict(kw_recon["y"])
    if alone:
        y = {k: v for k, v in y.items() if k in ("text", "text_scale", "mask")}
    space, _, _, _ = add_obstacles(y, B, 196, True, 20.0, 2, seed=11)
    return w, x_obs, kw_recon, kw_joint, {"y": y}, space


def test_graph_replay_generator_and_other_calls_are_unchanged():
    w, x_obs, kw_recon, kw_joint, kw_ob, space = obstacle_case()
    unguided = {"y": {k: v for k, v in kw_recon["y"].items() if k != "reconstruction_guidance"}}
    _, _, _, _, kw_fc, _ = TF.contact_case()
    others = ((unguided, None), (kw_recon, None), (kw_joint, space), (kw_fc, space))
    before = [TJ.run_ddim(w, kw, x_obs, sp) for kw, sp in others]
    graph = TJ.run_ddim(w, kw_ob, x_obs, space)
    direct = TJ.run_ddim(w, kw_ob, x_obs, space, use_graph=False)
    gen = TJ.run_ddim(w, kw_ob, x_obs, space, progressive=True)
    assert torch.equal(graph, direct), "graph replay differs from direct launches"
    assert torch.equal(graph, gen), "the generator differs from the fused loop"
    after = [TJ.run_ddim(w, kw, x_obs, sp) for kw, sp in others]
    w2 = TJ.joint_case()[0]
    fresh = [TJ.run_ddim(w2, kw, x_obs, sp) for kw, sp in others]
    for b, a_, f_, what in zip(before, after, fresh, ("unguided", "reconstruction-only", "joint-only", "foot-contact")):
        assert torch.equal(a_, b) and torch.equal(a_, f_), f"a {what} loop changed after obstacle-guided calls"
    assert not torch.equal(graph, before[1]), "obstacle guidance had no effect"
    # the step-graph key records K: one obstacle fewer captures its own graph and computes what direct launches do
    fewer = {"y": dict(kw_ob["y"], obstacles=kw_ob["y"]["obstacles"][:, :2].contiguous())}
    assert torch.equal(TJ.run_ddim(w, fewer, x_obs, space), TJ.run_ddim(w, fewer, x_obs, space, use_graph=False))
    # and S: another joint set likewise
    other_s = {"y": dict(kw_ob["y"], obstacle_joints=[0, 9, 13])}
    g_s = TJ.run_ddim(w, other_s, x_obs, space)
    assert torch.equal(g_s, TJ.run_ddim(w, other_s, x_obs, space, use_graph=False)) and not torch.equal(g_s, graph)


def test_obstacles_alone_guide_plain_text_to_motion():
    """no keyframes (M = 0): graph replay equals direct launches, the result differs from the unguided loop, and zero
    radii leave it unguided"""
    w, x_obs, _, _, kw_ob, space = obstacle_case(alone=True)
    graph = TJ.run_ddim(w, kw_ob, x_obs, space)
    direct = TJ.run_ddim(w, kw_ob, x_obs, space, use_graph=False)
    plain = TJ.run_ddim(w, {"y": {k: v for k, v in kw_ob["y"].items() if not k.startswith(("obstacle", "stop_obstacle"))}},
                        x_obs)
    assert torch.equal(graph, direct)
    assert torch.isfinite(graph).all() and not torch.equal(graph, plain)
    radius0 = kw_ob["y"]["obstacles"].clone()
    radius0[..., 2] = 0
    zero = TJ.run_ddim(w, {"y": dict(kw_ob["y"], obstacles=radius0)}, x_obs, space)
    assert torch.isfinite(zero).all()


def test_launch_counts():
    """an obstacle-guided step launches what a joint-guided step launches (128 + the joint seed kernel), with or
    without joint targets and foot contact; the per-step count is the difference between a 6-step and a 3-step call"""
    w, x_obs, kw_recon, kw_joint, kw_ob, space = obstacle_case()
    joint_keys = {k: v for k, v in kw_joint["y"].items() if k.startswith(("joint_", "stop_joint"))}
    kw_all = {"y": dict(kw_ob["y"], foot_contact_guidance=True, foot_contact_weight=0.1, stop_footcontact_at=0,
                        **joint_keys)}
    eng = C.resolve_model(w)[0].engine_for(DEV, max_batch=2, precision=C.PRECISION_BF16X3, nframes=196)

    def count(kw, skip, sp=None):
        n0 = eng.launch_count
        TJ.run_ddim(w, kw, x_obs, sp, skip=skip)
        return eng.launch_count - n0

    per_step = {}
    for name, kw in (("recon+joint", kw_joint), ("recon+obstacle", kw_ob), ("recon+joint+contact+obstacle", kw_all)):
        count(kw, 44, space)  # capture the step graphs first
        per_step[name] = (count(kw, 44, space) - count(kw, 47, space)) / 3
    print(f"[launches per guided step] {per_step}")
    assert per_step["recon+joint"] == 59 + 1 + 68 + 1
    assert per_step["recon+obstacle"] == per_step["recon+joint"]
    assert per_step["recon+joint+contact+obstacle"] == per_step["recon+joint"]


def test_refusals():
    w, x_obs, _, _, kw_ob, space = obstacle_case()
    d = C.create_gaussian_diffusion(timestep_respacing="ddim50")
    with pytest.raises(NotImplementedError, match="joint_space"):
        d.ddim_sample_loop(w, (2, 263, 1, 196), model_kwargs=kw_ob, skip_timesteps=44)
    d.joint_space = space
    d.window = C.Window(196, 0)
    with pytest.raises(NotImplementedError, match="windows"):
        d.ddim_sample_loop(w, (2, 263, 1, 196), model_kwargs=kw_ob, skip_timesteps=44)
    d.window = None
    with pytest.raises(ValueError, match="at most 16"):
        d.ddim_sample_loop(w, (2, 263, 1, 196), model_kwargs={"y": dict(kw_ob["y"], obstacles=torch.zeros(2, 17, 3))},
                           skip_timesteps=44)
    # MDM_UNET at bf16x3 and bf16: the reconstruction-guidance refusal, message unchanged
    m, wu, sd, xo, kf, y, c, g = TG.setup(2, seed=25)
    add_obstacles(y, 2, TG.L, True, 1.0, 0, seed=12)
    y["reconstruction_guidance"] = False
    for precision in (C.PRECISION_BF16X3, C.PRECISION_BF16):
        du = C.create_gaussian_diffusion(timestep_respacing="ddim50")
        du.precision, du.joint_space = precision, space
        with pytest.raises(RuntimeError, match="transformer"):
            du.ddim_sample_loop(wu, (2, TG.D, 1, TG.L), model_kwargs={"y": y}, skip_timesteps=48)


def test_c_abi_refusals():
    """cmdi_sample and cmdi_obstacle_seed refuse what the engine cannot run, with their messages"""
    w, x_obs, _, _, kw_ob, space = obstacle_case()
    eng = C.resolve_model(w)[0].engine_for(DEV, max_batch=2, precision=C.PRECISION_BF16X3, nframes=196)
    eng.set_schedule(C.create_gaussian_diffusion(timestep_respacing="ddim50").betas, list(range(50)))
    mean, std = space.mean.to(DEV), space.std.to(DEV)
    base = dict(skip_timesteps=48, x_T=torch.zeros(2, 263, 1, 196, device=DEV), joint_mean=mean, joint_std=std,
                joint_abs3d=True, obstacle_guidance=True, obstacle_coef=[1.0] * 50, obstacle_joints=1)
    for kw, match in ((dict(obstacles=torch.zeros(2, 17, 3, device=DEV)), "n_obstacles"),
                      (dict(obstacles=torch.zeros(2, 1, 3, device=DEV), obstacle_joints=0), "obstacle_joints"),
                      (dict(obstacles=torch.zeros(2, 1, 3, device=DEV), obstacle_joints=1 << 22), "obstacle_joints"),
                      (dict(obstacles=torch.zeros(2, 1, 3, device=DEV), joint_mean=None), "joint_mean")):
        with pytest.raises(RuntimeError, match=match):
            eng.sample(2, C.capi.SAMPLER_DDIM, **dict(base, **kw))
    x0 = torch.zeros(2, 263, 1, 196, device=DEV)
    for kw in (dict(obstacles=torch.zeros(2, 17, 3, device=DEV)), dict(obstacles=torch.zeros(2, 1, 3, device=DEV),
                                                                        obstacle_joints=0)):
        with pytest.raises(RuntimeError, match="cmdi_obstacle_seed"):
            obstacle_seed(x0, mean, std, True, **kw)
    with pytest.raises(RuntimeError, match="cmdi_obstacle_seed"):   # foot contact needs the 263 features
        obstacle_seed(x0[:, :100], mean[:100], std[:100], True, torch.zeros(2, 1, 3, device=DEV), foot_contact=True)

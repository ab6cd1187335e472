"""GPU: RePaint resampling (repaint_sample_loop[_progressive]) behind the public API, against
  (1) tests/golden/repaint.* -- the UNMODIFIED reference's p_sample driven along the walk (oracle/make_golden_repaint.py)
      -- and
  (2) oracle/repaint_oracle.py run in the test,
at rtol 1e-3 / atol 1e-4 (bf16x3); PRECISION_BF16 and the fp16 UNet with the A/F gates of test_gpu_bf16.py and
test_gpu_unet_guidance.py; jump_n_sample = 1 against the engine's own p_sample_loop in every noise mode, bit for bit;
the bit-for-bit properties (generator == fused loop, chunked calls, graph replay == direct launches, sharding, merged
evaluation jobs), torch's generator offset, launches per op and the errors.
"""
from ctypes import byref

import pytest
import torch

import condmdi_b200 as C
import test_gpu_bf16 as TB
import test_gpu_dpm_solver as TD
import test_gpu_unet_guidance as TG
from oracle import condmdi_oracle as O
from oracle import repaint_oracle as R
from oracle.golden_io import load_golden

pytestmark = pytest.mark.gpu
B, D, L = 2, 263, 196
SHAPE = (B, D, 1, L)
DEV = "cuda:0"
REPAINT = C.capi.SAMPLER_REPAINT
close = TD.close


@pytest.fixture(scope="module")
def gold(golden_dir):
    return load_golden(golden_dir, "repaint")


@pytest.fixture(scope="module")
def gi():
    return O.golden_inputs()


@pytest.fixture(scope="module")
def plain():
    return TD._model(False)


@pytest.fixture(scope="module")
def texty(gi):
    return TD._model(True, gi)


def n_ops(respacing, skip, j, r):
    return len(R.build_walk(O.make_tables(respacing).num_timesteps - 1 - skip, j, r))


def cycled(gi, n):
    """golden_inputs()'s 8 draws cycled to x_T + n per-op draws (the fixtures' tapes)"""
    return gi["tape"][torch.arange(n + 1) % 8]


def spaced(respacing, tape=None):
    d = C.create_gaussian_diffusion(timestep_respacing=respacing)
    if tape is not None:
        d.noise_tape = tape.to(DEV)
    return d


def config(gold, name):
    skip, j, r = (int(v) for v in gold[f"{name}.config"])
    return skip, j, r


# ------------------------------------------------------------------------------------------------
# transformer and UNet xl, bf16x3: the fixtures
# ------------------------------------------------------------------------------------------------
def test_golden_transformer(plain, texty, gi, gold):
    skip, j, r = config(gold, "no_cond")
    got = spaced("ddim50", cycled(gi, n_ops("ddim50", skip, j, r))).repaint_sample_loop(
        plain[0], SHAPE, model_kwargs={"y": {}}, jump_length=j, jump_n_sample=r)
    assert got.shape == SHAPE and got.is_cuda
    assert close(got, gold["no_cond.ref"], f"no_cond ddim50 whole walk, j {j}, r {r}")
    w = C.ClassifierFreeSampleModel(texty[0])
    x_obs = gi["x_obs"].to(DEV)
    for name, guided in (("cfg_impute", False), ("guided", True)):
        skip, j, r = config(gold, name)
        got = spaced("ddim50", cycled(gi, n_ops("ddim50", skip, j, r))).repaint_sample_loop(
            w, SHAPE, model_kwargs=TD._ykw(gi, guided), skip_timesteps=skip, init_image=x_obs, jump_length=j, jump_n_sample=r)
        assert close(got, gold[f"{name}.ref"], f"{name}: CFG 2.5 + imputation{' + guidance w=20' if guided else ''}, "
                                               f"last {50 - skip} steps, j {j}, r {r}")


def test_golden_unet_xl_keyframes(gi, gold):
    m, _ = TD._unet_xl(gi)
    w = C.ClassifierFreeSampleModel(m)
    xo, kf = gi["x_obs"].to(DEV), gi["kf_mask"].to(DEV)
    kw = {"y": {"text": ["a", "b"], "text_scale": gi["text_scale"].to(DEV), "mask": gi["y_mask"].to(DEV), "lengths": gi["lengths"]},
          "obs_x0": xo, "obs_mask": kf}
    skip, j, r = config(gold, "unet")
    got = spaced("ddim50", cycled(gi, n_ops("ddim50", skip, j, r))).repaint_sample_loop(
        w, SHAPE, model_kwargs=kw, skip_timesteps=skip, init_image=xo, jump_length=j, jump_n_sample=r)
    assert close(got, gold["unet.ref"], f"keyframe-conditioned MDM_UNET xl, CFG, last {50 - skip} steps, j {j}, r {r}")
    # reconstruction guidance on a bf16x3 MDM_UNET keeps its existing refusal
    kw2 = {"y": dict(kw["y"], reconstruction_guidance=True, reconstruction_weight=20.0, gradient_schedule=None,
                     diffusion_steps=1000, stop_recguidance_at=0, inpainted_motion=xo, inpainting_mask=kf),
           "obs_x0": xo, "obs_mask": kf}
    with pytest.raises(RuntimeError, match="transformer"):
        spaced("ddim50", cycled(gi, 20)).repaint_sample_loop(w, SHAPE, model_kwargs=kw2, skip_timesteps=46, jump_length=2,
                                                            jump_n_sample=2)


# ------------------------------------------------------------------------------------------------
# against the oracle run here
# ------------------------------------------------------------------------------------------------
def test_ddim20_whole_walks_vs_oracle(plain, texty, gi):
    tab = O.make_tables("ddim20")
    j, r = 4, 2
    tape = cycled(gi, n_ops("ddim20", 0, j, r))
    got = spaced("ddim20", tape).repaint_sample_loop(plain[0], SHAPE, model_kwargs={"y": {}}, jump_length=j, jump_n_sample=r)
    want = R.repaint_sample_loop(plain[1], tab, SHAPE, O.Conditioning(), tape, j, r)
    assert close(got, want, f"ddim20 no_cond, j {j}, r {r}")
    w = C.ClassifierFreeSampleModel(texty[0])
    got = spaced("ddim20", tape).repaint_sample_loop(w, SHAPE, model_kwargs=TD._ykw(gi, False), jump_length=j,
                                                     jump_n_sample=r)
    want = R.repaint_sample_loop(texty[1], tab, SHAPE, TD._cfg_cond(gi, False), tape, j, r)
    assert close(got, want, f"ddim20 cfg + imputation, j {j}, r {r}")


def test_b64_transformer_cfg_imputation_tail_vs_oracle(texty):
    m, sd = texty
    Bf, skip, j, r = 64, 44, 2, 3
    g = torch.Generator().manual_seed(33)
    tape = torch.randn(1 + n_ops("ddim50", skip, j, r), Bf, D, 1, L, generator=g)
    x_obs = torch.randn(Bf, D, 1, L, generator=g)
    cond = torch.randn(Bf, 512, generator=g)
    scale = torch.rand(Bf, generator=g) * 3
    kf = torch.rand(Bf, D, 1, L, generator=g) < 0.2
    table = {str(i): cond[i].to(DEV) for i in range(Bf)}
    old = m.encode_text
    m.encode_text = lambda texts: torch.stack([table[s] for s in texts])
    try:
        y = {"text": [str(i) for i in range(Bf)], "text_scale": scale.to(DEV), "imputate": 1, "stop_imputation_at": 1,
             "replacement_distribution": "conditional", "inpainted_motion": x_obs.to(DEV), "inpainting_mask": kf.to(DEV),
             "mask": torch.ones(Bf, 1, 1, L, dtype=torch.bool, device=DEV)}
        got = spaced("ddim50", tape).repaint_sample_loop(C.ClassifierFreeSampleModel(m), (Bf, D, 1, L), model_kwargs={"y": y},
                                                         skip_timesteps=skip, init_image=x_obs.to(DEV), jump_length=j,
                                                         jump_n_sample=r)
    finally:
        m.encode_text = old
    c = O.Conditioning(cond_emb=cond, cfg=True, text_scale=scale, y_mask=torch.ones(Bf, 1, 1, L, dtype=torch.bool),
                       imputate=True, stop_imputation_at=1, inpainted_motion=x_obs, inpainting_mask=kf)
    want = R.repaint_sample_loop(sd, O.make_tables("ddim50"), (Bf, D, 1, L), c, tape, j, r, skip_timesteps=skip,
                                 init_image=x_obs)
    assert close(got, want, f"B=64 transformer ddim50, CFG + imputation, last {50 - skip} steps, j {j}, r {r}")


def test_b64_unet_xl_cfg_keyframes_tail_vs_oracle():
    Bf, skip, j, r = 64, 46, 2, 2
    m, sd = TG.module()
    w = C.ClassifierFreeSampleModel(m)
    x_obs, _, kf, cond, scale = TG.inputs(Bf, seed=41)
    table = {str(i): cond[i].to(DEV) for i in range(Bf)}
    m.encode_text = lambda texts: torch.stack([table[s] for s in texts])
    g = torch.Generator().manual_seed(43)
    tape = torch.randn(1 + n_ops("ddim50", skip, j, r), Bf, D, 1, L, generator=g)
    kw = {"y": {"text": [str(i) for i in range(Bf)], "text_scale": scale.to(DEV)}, "obs_x0": x_obs.to(DEV), "obs_mask": kf.to(DEV)}
    got = spaced("ddim50", tape).repaint_sample_loop(w, (Bf, D, 1, L), model_kwargs=kw, skip_timesteps=skip,
                                                     init_image=x_obs.to(DEV), jump_length=j, jump_n_sample=r)
    c = O.Conditioning(cond_emb=cond, cfg=True, text_scale=scale, obs_x0=x_obs, obs_mask=kf)
    want = TD._unet_fp32_on_gpu(sd, lambda: R.repaint_sample_loop(sd, O.make_tables("ddim50"), (Bf, D, 1, L), c, tape, j, r,
                                                                  skip_timesteps=skip, init_image=x_obs))
    # The bf16x3 UNet's x0 sits at the parity gate's edge on every pass (test_gpu_dpm_solver.unet_gate: max 1.0e-4 over
    # a B = 2 CFG tail), and the walk makes 6 passes over these 4 steps.  Measured on an H100: max 2.4e-4 over the
    # 3.3M elements at B = 64, mean 1.4e-5 (the mean of the transformer tails); B = 2 (the fixture, 9 passes) stays
    # inside the plain gate at 8.5e-5.  So the maximum is gated at atol 3e-4 and the mean at the transformer's level.
    assert close(got, want, f"B=64 MDM_UNET xl, CFG + keyframe input, last {50 - skip} steps, j {j}, r {r}",
                 rtol=1e-3, atol=3e-4)
    assert (got.cpu() - want).abs().mean() < 2e-5


# ------------------------------------------------------------------------------------------------
# PRECISION_BF16 transformer and fp16 UNet: A/F gates
# ------------------------------------------------------------------------------------------------
def test_bf16_transformer_walk_meets_the_contract(gi):
    m, sd = TB.module(text=False)
    sdd = {k: v.to(DEV) for k, v in sd.items()}
    skip, j, r = 14, 2, 2
    tape = cycled(gi, n_ops("ddim20", skip, j, r))
    d = spaced("ddim20", tape)
    d.precision = TB.BF16
    got = d.repaint_sample_loop(m, SHAPE, model_kwargs={"y": {}}, skip_timesteps=skip, jump_length=j, jump_n_sample=r)
    real = O.mdm_forward
    want = {}
    try:
        for name, q in (("A", TB.bf16r), ("F", TB.exact)):
            def fwd(sd_, x, t, cond_emb=None, uncond=False, num_heads=4, _q=q):
                with torch.no_grad():
                    return TB.mdm_model(_q, sdd, x.to(DEV), t.to(DEV), cond_emb, uncond).float().cpu()
            O.mdm_forward = fwd
            want[name] = R.repaint_sample_loop(sd, O.make_tables("ddim20"), SHAPE, O.Conditioning(), tape, j, r,
                                               skip_timesteps=skip)
    finally:
        O.mdm_forward = real
    TB.gate(got, want["A"], want["F"], f"PRECISION_BF16 ddim20, last {20 - skip} steps, j {j}, r {r}")


def test_fp16_unet_xl_walks_meet_the_gates():
    m, w, sd, x_obs, kf, y, c, g = TG.setup(B, seed=51)
    skip, j, r = 45, 2, 2
    tape = torch.randn(1 + n_ops("ddim50", skip, j, r), B, D, 1, L, generator=g)
    tab = O.make_tables("ddim50")
    kw = {"obs_x0": x_obs.to(DEV), "obs_mask": kf.to(DEV)}

    def run(y_, c_):
        d = spaced("ddim50", tape)
        d.precision = C.PRECISION_FP16
        got = d.repaint_sample_loop(w, SHAPE, model_kwargs=dict(kw, y=y_), skip_timesteps=skip, init_image=x_obs.to(DEV),
                                    jump_length=j, jump_n_sample=r)
        a, f = TG.oracle_loop(sd, lambda: R.repaint_sample_loop(sd, tab, SHAPE, c_, tape, j, r, skip_timesteps=skip,
                                                                init_image=x_obs))
        return got, a, f

    y_plain = {k: v for k, v in y.items() if k in ("text", "text_scale", "mask")}
    c_plain = O.Conditioning(cond_emb=c.cond_emb, cfg=True, text_scale=c.text_scale, y_mask=c.y_mask, obs_x0=c.obs_x0,
                             obs_mask=c.obs_mask)
    # loops are gated at track 1.5, as in test_gpu_unet_fp16.py / test_gpu_unet_guidance.py
    TG.gate(*run(y_plain, c_plain), "fp16 UNet xl, CFG + keyframe input, last 5 steps, j 2, r 2", track=1.5)
    # guidance w = 20 at p >= 2: the jumped stretch 2..1 (from jump point 0) is revisited guided at 2, unguided at 1
    y_g = dict(y, stop_recguidance_at=2)
    c.stop_recguidance_at = 2
    TG.gate(*run(y_g, c), "fp16 UNet xl, CFG + guidance w=20 (stop_recguidance_at=2), last 5 steps, j 2, r 2", track=1.5)


# ------------------------------------------------------------------------------------------------
# jump_n_sample = 1 is the engine's own p_sample_loop, bit for bit, in every noise mode
# ------------------------------------------------------------------------------------------------
def test_one_sample_equals_engine_ddpm_with_a_tape(plain, texty, gi):
    d = spaced("ddim50", cycled(gi, 50))
    ddpm = d.p_sample_loop(plain[0], SHAPE, model_kwargs={"y": {}})
    rp = d.repaint_sample_loop(plain[0], SHAPE, model_kwargs={"y": {}}, jump_length=5, jump_n_sample=1)
    assert torch.equal(rp, ddpm)
    w = C.ClassifierFreeSampleModel(texty[0])
    kw = dict(model_kwargs=TD._ykw(gi, True), skip_timesteps=44, init_image=gi["x_obs"].to(DEV))
    assert torch.equal(d.repaint_sample_loop(w, SHAPE, jump_length=2, jump_n_sample=1, **kw), d.p_sample_loop(w, SHAPE, **kw))


def test_one_sample_equals_engine_ddpm_with_torch_rng(plain):
    d = spaced("ddim50")
    assert d.rng == "torch"
    for skip in (0, 40):
        torch.manual_seed(11)
        ddpm = d.p_sample_loop(plain[0], SHAPE, model_kwargs={"y": {}}, skip_timesteps=skip)
        after_ddpm = torch.cuda.get_rng_state(DEV)
        torch.manual_seed(11)
        rp = d.repaint_sample_loop(plain[0], SHAPE, model_kwargs={"y": {}}, skip_timesteps=skip, jump_length=3,
                                   jump_n_sample=1)
        assert torch.equal(torch.cuda.get_rng_state(DEV), after_ddpm)  # the same generator state consumed
        assert torch.equal(rp, ddpm)


def test_one_sample_equals_engine_ddpm_with_engine_rng(plain):
    d = spaced("ddim50")
    d.rng, d.engine_seed = "engine", 77
    ddpm = d.p_sample_loop(plain[0], SHAPE, model_kwargs={"y": {}})
    rp = d.repaint_sample_loop(plain[0], SHAPE, model_kwargs={"y": {}}, jump_length=5, jump_n_sample=1)
    assert torch.equal(rp, ddpm)
    assert not torch.equal(rp, d.repaint_sample_loop(plain[0], SHAPE, model_kwargs={"y": {}}, jump_length=5, jump_n_sample=2))


def test_engine_rng_first_visits_use_ddpm_streams(plain):
    """with the engine generator, the ops of the descent before the first jump (first visits) draw what p_sample_loop
    draws: a walk whose only jump point is 0 equals p_sample_loop until it arrives there"""
    d = spaced("ddim50")
    d.rng, d.engine_seed = "engine", 78
    m = plain[0]
    gen = d.repaint_sample_loop_progressive(m, SHAPE, model_kwargs={"y": {}}, skip_timesteps=44, jump_length=3,
                                            jump_n_sample=2)
    rp = [o["sample"].clone() for o in gen]
    ddpm = [o["sample"].clone() for o in d.p_sample_loop_progressive(m, SHAPE, model_kwargs={"y": {}}, skip_timesteps=44)]
    assert all(torch.equal(a, b) for a, b in zip(rp[:5], ddpm[:5]))  # denoise ops at 5, 4, 3, 2, 1
    assert len(rp) == 9 and not torch.equal(rp[-1], ddpm[-1])


# ------------------------------------------------------------------------------------------------
# bit-for-bit properties, torch's generator and launches
# ------------------------------------------------------------------------------------------------
def _noise_modes(gi):
    def tape(d):
        d.noise_tape = cycled(gi, 60).to(DEV)

    def torch_rng(d):
        d.rng = "torch"

    def engine_rng(d):
        d.rng, d.engine_seed = "engine", 123
    return {"tape": tape, "torch": torch_rng, "engine": engine_rng}


@pytest.mark.parametrize("mode", ["tape", "torch", "engine"])
def test_progressive_equals_fused_in_every_noise_mode(plain, gi, mode):
    m, _ = plain
    d = spaced("ddim50")
    _noise_modes(gi)[mode](d)
    skip, j, r = 40, 4, 3  # jump points 4 and 0: 26 denoise ops, 16 undo ops
    walk = R.build_walk(9, j, r)
    torch.manual_seed(21)
    outs = [{k: (v.clone() if torch.is_tensor(v) else v) for k, v in o.items()} for o in
            d.repaint_sample_loop_progressive(m, SHAPE, model_kwargs={"y": {}}, skip_timesteps=skip, jump_length=j,
                                              jump_n_sample=r)]
    after_gen = torch.cuda.get_rng_state(DEV)
    assert [o["t"] for o in outs] == [p for k, p in walk if k == R.DENOISE]
    assert all(set(o) == {"sample", "pred_xstart", "t"} for o in outs)
    torch.manual_seed(21)
    fused = d.repaint_sample_loop(m, SHAPE, model_kwargs={"y": {}}, skip_timesteps=skip, jump_length=j, jump_n_sample=r)
    assert torch.equal(torch.cuda.get_rng_state(DEV), after_gen)
    assert torch.equal(outs[-1]["sample"], fused)
    assert torch.equal(outs[-1]["sample"], outs[-1]["pred_xstart"])  # step 0 returns x0
    if mode == "torch":
        # an early stop after k denoise ops leaves torch's generator moved by x_T and the draws of the ops run so far
        inc = C.diffusion.aten_launch_policy(B * D * L, torch.device(DEV))[1]
        for k in (5, 6, 12):
            torch.manual_seed(21)
            off0 = C.diffusion._cuda_rng_state(DEV)[1]
            gen = d.repaint_sample_loop_progressive(m, SHAPE, model_kwargs={"y": {}}, skip_timesteps=skip, jump_length=j,
                                                    jump_n_sample=r)
            for i, o in zip(range(k), gen):
                assert torch.equal(o["sample"], outs[i]["sample"])
            ops = [i for i, (kind, _) in enumerate(walk) if kind == R.DENOISE][k - 1] + 1
            assert C.diffusion._cuda_rng_state(DEV)[1] == off0 + (1 + ops) * inc


def test_torch_generator_moves_by_x_T_and_one_draw_per_op(plain):
    m, _ = plain
    d = spaced("ddim50")
    inc = C.diffusion.aten_launch_policy(B * D * L, torch.device(DEV))[1]
    for skip, j, r in ((40, 4, 3), (0, 5, 3), (46, 10, 4)):
        torch.manual_seed(5)
        off0 = C.diffusion._cuda_rng_state(DEV)[1]
        d.repaint_sample_loop(m, SHAPE, model_kwargs={"y": {}}, skip_timesteps=skip, jump_length=j, jump_n_sample=r)
        assert C.diffusion._cuda_rng_state(DEV)[1] == off0 + (1 + n_ops("ddim50", skip, j, r)) * inc, (skip, j, r)


def test_fused_chunks_and_resume_with_a_tape(plain, gi):
    """the native calls directly: num_steps counts denoise ops, a call runs the undo ops before each of them, and a
    walk in chunks (each resuming from the position reached) equals the whole walk"""
    m, _ = plain
    skip, j, r = 40, 4, 3
    walk = R.build_walk(9, j, r)
    tape = cycled(gi, len(walk)).to(DEV)
    d = spaced("ddim50", tape)
    fused = d.repaint_sample_loop(m, SHAPE, model_kwargs={"y": {}}, skip_timesteps=skip, jump_length=j, jump_n_sample=r)
    eng = m.engine_for(torch.device(DEV), max_batch=B)
    denoise_at = [i for i, (k, _) in enumerate(walk) if k == R.DENOISE]
    common = dict(sampler=REPAINT, repaint_jump_length=j, repaint_jump_n_sample=r)
    state, done = eng.sample(B, skip_timesteps=skip, num_steps=7, x_T=tape[0], init_image=torch.zeros(SHAPE, device=DEV),
                             noise_tape=tape[1:], **common)["sample"], 7
    for chunk in (1, 5, 13):
        d0 = denoise_at[done - 1] + 1
        kind, p = walk[d0]
        pos = p - 1 if kind == R.UNDO else p
        state = eng.sample(B, skip_timesteps=49 - pos, num_steps=chunk, x_T=state, resume=True, noise_tape=tape[1 + d0:],
                           **common)["sample"]
        done += chunk
    assert done == len(denoise_at) and torch.equal(state, fused)
    with pytest.raises(RuntimeError, match="does not continue the running history"):  # the walk has ended
        eng.sample(B, skip_timesteps=49, resume=True, x_T=state, noise_tape=tape[1:], **common)
    # 7 denoise ops (9, 8, 7, 6, 5, then 8, 7 after the undo run from jump point 4) leave the walk at position 6
    eng.sample(B, skip_timesteps=skip, num_steps=7, x_T=tape[0], noise_tape=tape[1:], **common)
    for bad in (dict(skip_timesteps=44), dict(repaint_jump_n_sample=2), dict(repaint_jump_length=3),
                dict(sampler=C.capi.SAMPLER_DPM_SOLVER_SDE, dpm_order=1)):
        kw = dict(common, skip_timesteps=49 - 6, **{"x_T": tape[0], "resume": True, "noise_tape": tape[1:]})
        kw.update(bad)
        with pytest.raises(RuntimeError, match="does not continue the running history"):
            eng.sample(B, **kw)
    eng.sample(B, **dict(common, skip_timesteps=49 - 6, x_T=tape[0], resume=True, noise_tape=tape[1:]))  # the right one


@pytest.mark.parametrize("mode", ["tape", "torch", "engine"])
def test_graph_replay_equals_direct_launches(texty, gi, mode):
    w = C.ClassifierFreeSampleModel(texty[0])
    d = spaced("ddim50")
    _noise_modes(gi)[mode](d)
    # guidance w = 20 at p >= 2: the stretch 3..1 jumped from 0 is revisited guided and unguided
    kw = dict(model_kwargs=TD._ykw(gi, True), skip_timesteps=44, init_image=gi["x_obs"].to(DEV), jump_length=3,
              jump_n_sample=3)
    torch.manual_seed(8)
    graphed = d.repaint_sample_loop(w, SHAPE, **kw)
    d.use_graph = False
    torch.manual_seed(8)
    direct = d.repaint_sample_loop(w, SHAPE, **kw)
    assert torch.equal(graphed, direct)


def test_launches_per_denoise_and_undo_op(plain, gi):
    m, _ = plain
    eng = m.engine_for(torch.device(DEV), max_batch=B)
    d = spaced("ddim50")
    d.rng = "engine"
    x_T = gi["tape"][0].to(DEV)

    def launches(fn, skip, **kw):
        n0 = eng.launch_count
        fn(m, SHAPE, noise=x_T, model_kwargs={"y": {}}, skip_timesteps=skip, **kw)
        torch.cuda.synchronize()
        return eng.launch_count - n0

    per_step = launches(d.p_sample_loop, 40) - launches(d.p_sample_loop, 41)
    assert per_step > 1
    base = launches(d.repaint_sample_loop, 40, jump_length=3, jump_n_sample=1)
    assert base == launches(d.p_sample_loop, 40) + 1  # the one launch that sets the walk's two counters
    for j, r in ((3, 2), (3, 4), (4, 3), (9, 2)):
        n_den, n_undo = R.op_counts(9, j, r)
        got = launches(d.repaint_sample_loop, 40, jump_length=j, jump_n_sample=r)
        print(f"j {j} r {r}: {n_den} denoise + {n_undo} undo ops, {got} launches (DDPM step: {per_step})")
        assert got - base == (n_den - 10) * per_step + n_undo * 1


# ------------------------------------------------------------------------------------------------
# batching and sharding
# ------------------------------------------------------------------------------------------------
def test_engine_rng_shards_reproduce_the_unsharded_batch_including_x_T(plain):
    m, _ = plain
    d = spaced("ddim50")
    d.rng, d.engine_seed = "engine", 1234
    kw = dict(model_kwargs={"y": {}}, skip_timesteps=44, jump_length=2, jump_n_sample=3)
    full = d.repaint_sample_loop(m, (4, D, 1, L), **kw).clone()
    parts = []
    for lo in (0, 2):
        d.sample_offset = lo
        parts.append(d.repaint_sample_loop(m, (2, D, 1, L), **kw).clone())
    d.sample_offset = 0
    assert torch.equal(full, torch.cat(parts))
    assert not torch.equal(parts[0], parts[1])
    d.engine_seed = None
    torch.manual_seed(3)
    a = C.sharded_sample(d, m, (4, D, 1, L), {"y": {}}, sampler="repaint_sample_loop", skip_timesteps=44, jump_length=2,
                         jump_n_sample=3).clone()
    torch.manual_seed(3)
    b = C.sharded_sample(d, m, (4, D, 1, L), {"y": {}}, sampler="repaint_sample_loop", skip_timesteps=44, jump_length=2,
                         jump_n_sample=3).clone()
    assert torch.equal(a, b) and d.engine_seed is None and d.rng == "engine"


def test_eval_loop_jobs_merged_equal_unmerged(texty, gi):
    m, _ = texty
    w = C.ClassifierFreeSampleModel(m)
    d = spaced("ddim50")
    conds = [torch.randn(B, 512, generator=torch.Generator().manual_seed(60 + i)).to(DEV) for i in range(3)]
    x_obs, kf = gi["x_obs"].to(DEV), gi["kf_mask"].to(DEV)

    def y_of(i):
        return {"text": [f"job{i}a", f"job{i}b"], "text_scale": gi["text_scale"].to(DEV), "mask": gi["y_mask"].to(DEV),
                "lengths": gi["lengths"], "imputate": 1, "stop_imputation_at": 1, "replacement_distribution": "conditional",
                "inpainted_motion": x_obs + 0.1 * i, "inpainting_mask": kf}

    table = {f"job{i}{s}": conds[i][k] for i in range(3) for k, s in enumerate("ab")}
    old = m.encode_text
    m.encode_text = lambda texts: torch.stack([table[t] for t in texts])
    try:
        jobs = C.build_jobs([((B, D, 1, L), {"y": y_of(i)}) for i in range(3)], seed=10, mm_idxs=[2], mm_num_repeats=2)
        run = dict(sampler="repaint_sample_loop", seed=5, skip_timesteps=45, jump_length=2, jump_n_sample=2)
        one = C.run_eval_jobs(d, w, jobs, merge=1, **run)
        two = C.run_eval_jobs(d, w, jobs, merge=2, **run)
        four = C.run_eval_jobs(d, w, jobs, merge=4, **run)
        for i in range(4):
            assert one[i].shape == (B, D, 1, L) and torch.equal(one[i], two[i]) and torch.equal(one[i], four[i])
        assert not torch.equal(one[2], one[3])
    finally:
        m.encode_text = old


# ------------------------------------------------------------------------------------------------
# refusals
# ------------------------------------------------------------------------------------------------
def test_c_abi_field_errors(plain, gi):
    m, _ = plain
    eng = m.engine_for(torch.device(DEV), max_batch=B)
    eng.set_schedule(spaced("ddim50").betas, spaced("ddim50").timestep_map)
    x_T = gi["tape"][0].to(DEV)
    zeros = torch.zeros(SHAPE, device=DEV)
    ok = dict(repaint_jump_length=2, repaint_jump_n_sample=2)
    cases = [
        (dict(repaint_jump_length=0, repaint_jump_n_sample=2), "repaint_jump_length 0 must be >= 1"),
        (dict(repaint_jump_length=2, repaint_jump_n_sample=0), "repaint_jump_n_sample 0 must be >= 1"),
        (dict(repaint_jump_length=1, repaint_jump_n_sample=1 << 30), "at most 2\\^28"),
        (dict(ok, eta=0.5), "eta"),
        (dict(ok, dump_steps=[1]), "dump_xstart"),
        (dict(ok, resume=True, init_image=zeros), "init_image"),
    ]
    for kw, msg in cases:
        with pytest.raises(RuntimeError, match=msg):
            eng.sample(B, sampler=REPAINT, skip_timesteps=45, x_T=x_T, **kw)
    out = torch.empty(SHAPE, device=DEV)
    for field in ("plms_order", "dpm_order", "unipc_order", "unipc_variant", "unipc_corrector"):
        a = C.capi.SampleArgs(B, REPAINT, 0.0, 45, 0, 0, None, x_T.data_ptr())
        a.repaint_jump_length, a.repaint_jump_n_sample = 2, 2
        setattr(a, field, 1)
        assert eng.lib.cmdi_sample(eng._h, byref(a), out.data_ptr(), None) != 0
        assert field.encode() in eng.lib.cmdi_last_error()
    for field in ("repaint_jump_length", "repaint_jump_n_sample"):
        a = C.capi.SampleArgs(B, C.capi.SAMPLER_DDPM, 0.0, 45, 0, 0, None, x_T.data_ptr())
        setattr(a, field, 1)
        assert eng.lib.cmdi_sample(eng._h, byref(a), out.data_ptr(), None) != 0
        assert field.encode() in eng.lib.cmdi_last_error()

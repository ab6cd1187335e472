"""GPU: the SDE-DPM-Solver++ sampler (dpm_solver_sde_sample_loop[_progressive]) behind the public API, against
  (1) tests/golden/dpm_solver_sde.* -- order 1: the UNMODIFIED reference's p_sample_loop on the same noise tape; order 2:
      the CPU restatement (oracle/make_golden_dpm_solver_sde.py) -- and
  (2) oracle/dpm_solver_sde_oracle.py run in the test,
at rtol 1e-3 / atol 1e-4 (bf16x3); PRECISION_BF16 and the fp16 UNet with the A/F gates of test_gpu_bf16.py and
test_gpu_unet_guidance.py; order 1 against the engine's own p_sample_loop in every noise mode; the bit-for-bit properties
(generator == fused loop, graph replay == direct launches, sharding, merged evaluation jobs), launches per step and the
errors.
"""
import pytest
import torch

import condmdi_b200 as C
import test_gpu_bf16 as TB
import test_gpu_dpm_solver as TD
import test_gpu_unet_guidance as TG
from oracle import condmdi_oracle as O
from oracle import dpm_solver_sde_oracle as S
from oracle.golden_io import load_golden

pytestmark = pytest.mark.gpu
B, D, L = 2, 263, 196
SHAPE = (B, D, 1, L)
DEV = "cuda:0"
SDE = C.capi.SAMPLER_DPM_SOLVER_SDE
close = TD.close
# order 1 against the engine's p_sample_loop on the same noise: only the fp32 rounding of the folded coefficients (A, B0
# against posterior_mean_coef2 / coef1, Cn against exp(0.5 * log variance)) differs, by an ulp of the state per step.
# In fp32 (the CPU restatement against the reference) that stays at 1.7e-6 over a whole ddim50 loop.  On the engine a
# state differing in the last bit is split into different bf16x3 planes, so the next pass differs at the denoiser's own
# error level, and the gap grows to what the engine's DDPM shows against the reference: measured on an H100, 2.5e-5 to
# 3.0e-5 over whole ddim50 loops (tape, torch and engine noise) against 3.2e-5 for engine vs reference.
ORDER1_TOL = dict(rtol=0.0, atol=5e-5)


@pytest.fixture(scope="module")
def gold(golden_dir):
    return load_golden(golden_dir, "dpm_solver_sde")


@pytest.fixture(scope="module")
def gi():
    return O.golden_inputs()


@pytest.fixture(scope="module")
def plain():
    return TD._model(False)


@pytest.fixture(scope="module")
def texty(gi):
    return TD._model(True, gi)


def cycled(gi, n):
    """golden_inputs()'s 8 draws cycled to x_T + n per-step draws (the fixtures' tape at n = 50)"""
    return gi["tape"][torch.arange(n + 1) % 8]


def spaced(respacing, tape=None):
    d = C.create_gaussian_diffusion(timestep_respacing=respacing)
    if tape is not None:
        d.noise_tape = tape.to(DEV)
    return d


def unet_gate(respacing, skip, order):
    """test_gpu_dpm_solver.unet_gate for this sampler's table: atol scales by the largest sum_j |B_j| of the run over
    order 1's"""
    tab = O.make_tables(respacing)
    t0 = tab.num_timesteps - 1 - skip

    def weight(o):
        return abs(S.coefficient_table(tab, t0, o)[1:t0 + 1, 1:3]).sum(1).max()
    return dict(rtol=1e-3, atol=1e-4 * max(1.0, weight(order) / weight(1)))


# ------------------------------------------------------------------------------------------------
# transformer and UNet xl, bf16x3: the fixtures (order 1 = the reference's p_sample_loop)
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("order", [1, 2])
def test_golden_transformer(plain, texty, gi, gold, order):
    want = {1: "ddpm_ref", 2: "o2"}[order]
    tape = cycled(gi, 50)
    got = spaced("ddim50", tape).dpm_solver_sde_sample_loop(plain[0], SHAPE, model_kwargs={"y": {}}, order=order)
    assert got.shape == SHAPE and got.is_cuda
    assert close(got, gold[f"no_cond.{want}"], f"no_cond ddim50 whole loop, order {order}")
    w = C.ClassifierFreeSampleModel(texty[0])
    x_obs = gi["x_obs"].to(DEV)
    got = spaced("ddim50", tape).dpm_solver_sde_sample_loop(w, SHAPE, model_kwargs=TD._ykw(gi, False), skip_timesteps=45,
                                                            init_image=x_obs, order=order)
    assert close(got, gold[f"cfg_impute.{want}"], f"cfg 2.5 + imputation, last 5 steps, order {order}")
    # guidance w = 20 at s = 3, 2, none at s = 1, 0 (stop_recguidance_at = 2 inside the loop)
    got = spaced("ddim50", tape).dpm_solver_sde_sample_loop(w, SHAPE, model_kwargs=TD._ykw(gi, True), skip_timesteps=46,
                                                            init_image=x_obs, order=order)
    assert close(got, gold[f"guided.{want}"], f"cfg + imputation + guidance w=20, last 4 steps, order {order}")


@pytest.mark.parametrize("order", [1, 2])
def test_golden_unet_xl_keyframes(gi, gold, order):
    m, _ = TD._unet_xl(gi)
    w = C.ClassifierFreeSampleModel(m)
    xo, kf = gi["x_obs"].to(DEV), gi["kf_mask"].to(DEV)
    kw = {"y": {"text": ["a", "b"], "text_scale": gi["text_scale"].to(DEV), "mask": gi["y_mask"].to(DEV), "lengths": gi["lengths"]},
          "obs_x0": xo, "obs_mask": kf}
    got = spaced("ddim50", cycled(gi, 50)).dpm_solver_sde_sample_loop(w, SHAPE, model_kwargs=kw, skip_timesteps=45,
                                                                      init_image=xo, order=order)
    want = {1: "ddpm_ref", 2: "o2"}[order]
    assert close(got, gold[f"unet.{want}"], f"keyframe-conditioned MDM_UNET xl, CFG, last 5 steps, order {order}",
                 **unet_gate("ddim50", 45, order))
    # reconstruction guidance on a bf16x3 MDM_UNET keeps its existing refusal
    kw2 = {"y": dict(kw["y"], reconstruction_guidance=True, reconstruction_weight=20.0, gradient_schedule=None,
                     diffusion_steps=1000, stop_recguidance_at=0, inpainted_motion=xo, inpainting_mask=kf),
           "obs_x0": xo, "obs_mask": kf}
    with pytest.raises(RuntimeError, match="transformer"):
        spaced("ddim50", cycled(gi, 50)).dpm_solver_sde_sample_loop(w, SHAPE, model_kwargs=kw2, skip_timesteps=48, order=order)


# ------------------------------------------------------------------------------------------------
# against the oracle run here
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("order", [1, 2])
def test_ddim20_whole_loops_vs_oracle(plain, texty, gi, order):
    tab = O.make_tables("ddim20")
    tape = cycled(gi, 20)
    got = spaced("ddim20", tape).dpm_solver_sde_sample_loop(plain[0], SHAPE, model_kwargs={"y": {}}, order=order)
    want = S.dpm_solver_sde_sample_loop(plain[1], tab, SHAPE, O.Conditioning(), tape, order)
    assert close(got, want, f"ddim20 no_cond, order {order}")
    w = C.ClassifierFreeSampleModel(texty[0])
    got = spaced("ddim20", tape).dpm_solver_sde_sample_loop(w, SHAPE, model_kwargs=TD._ykw(gi, False), order=order)
    want = S.dpm_solver_sde_sample_loop(texty[1], tab, SHAPE, TD._cfg_cond(gi, False), tape, order)
    assert close(got, want, f"ddim20 cfg + imputation, order {order}")


def test_b64_transformer_cfg_imputation_tail_order2_vs_oracle(texty):
    m, sd = texty
    Bf = 64
    g = torch.Generator().manual_seed(33)
    tape = torch.randn(6, Bf, D, 1, L, generator=g)
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
        got = spaced("ddim50", tape).dpm_solver_sde_sample_loop(C.ClassifierFreeSampleModel(m), (Bf, D, 1, L),
                                                                model_kwargs={"y": y}, skip_timesteps=45,
                                                                init_image=x_obs.to(DEV), order=2)
    finally:
        m.encode_text = old
    c = O.Conditioning(cond_emb=cond, cfg=True, text_scale=scale, y_mask=torch.ones(Bf, 1, 1, L, dtype=torch.bool),
                       imputate=True, stop_imputation_at=1, inpainted_motion=x_obs, inpainting_mask=kf)
    want = S.dpm_solver_sde_sample_loop(sd, O.make_tables("ddim50"), (Bf, D, 1, L), c, tape, 2, skip_timesteps=45,
                                        init_image=x_obs)
    assert close(got, want, "B=64 transformer ddim50, CFG + imputation, order 2, last 5 steps")


def test_b64_unet_xl_cfg_keyframes_tail_vs_oracle():
    Bf = 64
    m, sd = TG.module()
    w = C.ClassifierFreeSampleModel(m)
    x_obs, _, kf, cond, scale = TG.inputs(Bf, seed=41)
    table = {str(i): cond[i].to(DEV) for i in range(Bf)}
    m.encode_text = lambda texts: torch.stack([table[s] for s in texts])
    g = torch.Generator().manual_seed(43)
    tape = torch.randn(5, Bf, D, 1, L, generator=g)
    kw = {"y": {"text": [str(i) for i in range(Bf)], "text_scale": scale.to(DEV)}, "obs_x0": x_obs.to(DEV), "obs_mask": kf.to(DEV)}
    got = spaced("ddim50", tape).dpm_solver_sde_sample_loop(w, (Bf, D, 1, L), model_kwargs=kw, skip_timesteps=46,
                                                            init_image=x_obs.to(DEV), order=2)
    c = O.Conditioning(cond_emb=cond, cfg=True, text_scale=scale, obs_x0=x_obs, obs_mask=kf)
    want = TD._unet_fp32_on_gpu(sd, lambda: S.dpm_solver_sde_sample_loop(sd, O.make_tables("ddim50"), (Bf, D, 1, L), c, tape,
                                                                         2, skip_timesteps=46, init_image=x_obs))
    assert close(got, want, "B=64 MDM_UNET xl, CFG + keyframe input, order 2, last 4 steps", **unet_gate("ddim50", 46, 2))


# ------------------------------------------------------------------------------------------------
# PRECISION_BF16 transformer and fp16 UNet: A/F gates
# ------------------------------------------------------------------------------------------------
def test_bf16_transformer_loop_meets_the_contract(gi):
    m, sd = TB.module(text=False)
    sdd = {k: v.to(DEV) for k, v in sd.items()}
    d = spaced("ddim20", gi["tape"])
    d.precision = TB.BF16
    got = d.dpm_solver_sde_sample_loop(m, SHAPE, model_kwargs={"y": {}}, skip_timesteps=14, order=2)
    real = O.mdm_forward
    want = {}
    try:
        for name, q in (("A", TB.bf16r), ("F", TB.exact)):
            def fwd(sd_, x, t, cond_emb=None, uncond=False, num_heads=4, _q=q):
                with torch.no_grad():
                    return TB.mdm_model(_q, sdd, x.to(DEV), t.to(DEV), cond_emb, uncond).float().cpu()
            O.mdm_forward = fwd
            want[name] = S.dpm_solver_sde_sample_loop(sd, O.make_tables("ddim20"), SHAPE, O.Conditioning(), gi["tape"], 2,
                                                      skip_timesteps=14)
    finally:
        O.mdm_forward = real
    TB.gate(got, want["A"], want["F"], "PRECISION_BF16 ddim20, order 2, last 6 steps")


def test_fp16_unet_xl_loops_meet_the_gates():
    m, w, sd, x_obs, kf, y, c, g = TG.setup(B, seed=51)
    tape = torch.randn(6, B, D, 1, L, generator=g)
    tab = O.make_tables("ddim50")
    kw = {"obs_x0": x_obs.to(DEV), "obs_mask": kf.to(DEV)}

    def run(y_, c_, order):
        d = spaced("ddim50", tape)
        d.precision = C.PRECISION_FP16
        got = d.dpm_solver_sde_sample_loop(w, SHAPE, model_kwargs=dict(kw, y=y_), skip_timesteps=45,
                                           init_image=x_obs.to(DEV), order=order)
        a, f = TG.oracle_loop(sd, lambda: S.dpm_solver_sde_sample_loop(sd, tab, SHAPE, c_, tape, order, skip_timesteps=45,
                                                                       init_image=x_obs))
        return got, a, f

    y_plain = {k: v for k, v in y.items() if k in ("text", "text_scale", "mask")}
    c_plain = O.Conditioning(cond_emb=c.cond_emb, cfg=True, text_scale=c.text_scale, y_mask=c.y_mask, obs_x0=c.obs_x0,
                             obs_mask=c.obs_mask)
    # loops are gated at track 1.5, as in test_gpu_unet_fp16.py / test_gpu_unet_guidance.py
    TG.gate(*run(y_plain, c_plain, 2), "fp16 UNet xl, CFG + keyframe input, order 2, last 5 steps", track=1.5)
    # guidance w = 20 at s = 4, 3, 2, not at 1, 0
    y_g = dict(y, stop_recguidance_at=2)
    c.stop_recguidance_at = 2
    TG.gate(*run(y_g, c, 2), "fp16 UNet xl, CFG + guidance w=20 (stop_recguidance_at=2), order 2, last 5 steps", track=1.5)


# ------------------------------------------------------------------------------------------------
# order 1 is the engine's own p_sample_loop, in every noise mode
# ------------------------------------------------------------------------------------------------
def test_order1_equals_engine_ddpm_with_a_tape(plain, texty, gi):
    d = spaced("ddim50", cycled(gi, 50))
    ddpm = d.p_sample_loop(plain[0], SHAPE, model_kwargs={"y": {}})
    sde = d.dpm_solver_sde_sample_loop(plain[0], SHAPE, model_kwargs={"y": {}}, order=1)
    assert close(sde, ddpm, "ddim50 whole loop, tape: order 1 vs the engine's p_sample_loop", **ORDER1_TOL)
    w = C.ClassifierFreeSampleModel(texty[0])
    kw = dict(model_kwargs=TD._ykw(gi, True), skip_timesteps=44, init_image=gi["x_obs"].to(DEV))
    ddpm = d.p_sample_loop(w, SHAPE, **kw)
    sde = d.dpm_solver_sde_sample_loop(w, SHAPE, order=1, **kw)
    # guidance w = 20 gives the largest x0 and the largest pass-to-pass sensitivity: measured 8.8e-5 here, where the
    # engine's guided tail is 7.1e-5 from the reference (test_golden_transformer); the parity gate
    assert close(sde, ddpm, "ddim50 guided tail, tape: order 1 vs the engine's p_sample_loop", **TD.GATE)


def test_order1_equals_engine_ddpm_with_torch_rng(plain):
    d = spaced("ddim50")
    assert d.rng == "torch"
    for skip in (0, 40):
        torch.manual_seed(11)
        ddpm = d.p_sample_loop(plain[0], SHAPE, model_kwargs={"y": {}}, skip_timesteps=skip)
        after_ddpm = torch.cuda.get_rng_state(DEV)
        torch.manual_seed(11)
        sde = d.dpm_solver_sde_sample_loop(plain[0], SHAPE, model_kwargs={"y": {}}, skip_timesteps=skip, order=1)
        assert torch.equal(torch.cuda.get_rng_state(DEV), after_ddpm)  # the same generator state consumed
        assert close(sde, ddpm, f"ddim50 skip {skip}, rng=torch: order 1 vs the engine's p_sample_loop", **ORDER1_TOL)


def test_order1_equals_engine_ddpm_with_engine_rng(plain):
    d = spaced("ddim50")
    d.rng, d.engine_seed = "engine", 77
    ddpm = d.p_sample_loop(plain[0], SHAPE, model_kwargs={"y": {}})
    sde = d.dpm_solver_sde_sample_loop(plain[0], SHAPE, model_kwargs={"y": {}}, order=1)
    assert close(sde, ddpm, "ddim50 whole loop, rng=engine: order 1 vs the engine's p_sample_loop", **ORDER1_TOL)
    assert not torch.equal(sde, d.dpm_solver_sde_sample_loop(plain[0], SHAPE, model_kwargs={"y": {}}, order=2))


# ------------------------------------------------------------------------------------------------
# bit-for-bit properties and launches
# ------------------------------------------------------------------------------------------------
def _noise_modes(gi):
    """(name, diffusion configurator) for the three noise sources"""
    def tape(d):
        d.noise_tape = cycled(gi, 50).to(DEV)

    def torch_rng(d):
        d.rng = "torch"

    def engine_rng(d):
        d.rng, d.engine_seed = "engine", 123
    return [("tape", tape), ("torch", torch_rng), ("engine", engine_rng)]


@pytest.mark.parametrize("order", [1, 2])
@pytest.mark.parametrize("mode", ["tape", "torch", "engine"])
def test_progressive_equals_fused_in_every_noise_mode(plain, gi, mode, order):
    m, _ = plain
    d = spaced("ddim50")
    dict(_noise_modes(gi))[mode](d)
    skip = 40
    torch.manual_seed(21)
    outs = [{k: v.clone() for k, v in o.items()} for o in
            d.dpm_solver_sde_sample_loop_progressive(m, SHAPE, model_kwargs={"y": {}}, skip_timesteps=skip, order=order)]
    after_gen = torch.cuda.get_rng_state(DEV)
    assert len(outs) == 10 and all(set(o) == {"sample", "pred_xstart"} for o in outs)
    torch.manual_seed(21)
    fused = d.dpm_solver_sde_sample_loop(m, SHAPE, model_kwargs={"y": {}}, skip_timesteps=skip, order=order)
    assert torch.equal(torch.cuda.get_rng_state(DEV), after_gen)
    assert torch.equal(outs[-1]["sample"], fused)
    assert torch.equal(outs[-1]["sample"], outs[-1]["pred_xstart"])  # the last step returns x0
    # an early stop leaves torch's generator where p_sample_loop_progressive leaves it
    torch.manual_seed(21)
    gen = d.dpm_solver_sde_sample_loop_progressive(m, SHAPE, model_kwargs={"y": {}}, skip_timesteps=skip, order=order)
    for k, o in zip(range(3), gen):
        assert torch.equal(o["sample"], outs[k]["sample"])
    stop_sde = torch.cuda.get_rng_state(DEV)
    torch.manual_seed(21)
    for _, _o in zip(range(3), d.p_sample_loop_progressive(m, SHAPE, model_kwargs={"y": {}}, skip_timesteps=skip)):
        pass
    assert torch.equal(stop_sde, torch.cuda.get_rng_state(DEV))


@pytest.mark.parametrize("order", [1, 2])
def test_fused_chunks_and_resume_with_a_tape(plain, gi, order):
    """the native calls directly: a prefix of the loop equals the generator's step, and a loop in two chunks (the second
    resumes the x0 history, its draws numbered from its own first step) equals the whole loop"""
    m, _ = plain
    tape = cycled(gi, 50).to(DEV)
    d = spaced("ddim50", tape)
    skip = 40
    outs = [o["sample"].clone() for o in
            d.dpm_solver_sde_sample_loop_progressive(m, SHAPE, model_kwargs={"y": {}}, skip_timesteps=skip, order=order)]
    fused = d.dpm_solver_sde_sample_loop(m, SHAPE, model_kwargs={"y": {}}, skip_timesteps=skip, order=order)
    eng = m.engine_for(torch.device(DEV), max_batch=B)
    zeros = torch.zeros(SHAPE, device=DEV)
    common = dict(sampler=SDE, dpm_order=order, x_T=tape[0], init_image=zeros)
    for k in (0, 1, 4):
        res = eng.sample(B, skip_timesteps=skip, num_steps=k + 1, noise_tape=tape[1:], **common)
        assert torch.equal(res["sample"], outs[k])
    part = eng.sample(B, skip_timesteps=skip, num_steps=4, noise_tape=tape[1:], **common)["sample"]
    rest = eng.sample(B, sampler=SDE, dpm_order=order, skip_timesteps=skip + 4, resume=True, x_T=part,
                      noise_tape=tape[5:])["sample"]
    assert torch.equal(rest, fused)
    with pytest.raises(RuntimeError, match="does not continue the running history"):
        eng.sample(B, sampler=SDE, dpm_order=order, skip_timesteps=skip + 4, resume=True, x_T=part, noise_tape=tape[5:])
    # DPM-Solver++ (ODE) cannot resume an SDE history, nor the other order
    part = eng.sample(B, skip_timesteps=skip, num_steps=4, noise_tape=tape[1:], **common)["sample"]
    with pytest.raises(RuntimeError, match="does not continue the running history"):
        eng.sample(B, sampler=C.capi.SAMPLER_DPM_SOLVER, dpm_order=order, skip_timesteps=skip + 4, resume=True, x_T=part)
    part = eng.sample(B, skip_timesteps=skip, num_steps=4, noise_tape=tape[1:], **common)["sample"]
    with pytest.raises(RuntimeError, match="does not continue the running history"):
        eng.sample(B, sampler=SDE, dpm_order=3 - order, skip_timesteps=skip + 4, resume=True, x_T=part, noise_tape=tape[5:])


@pytest.mark.parametrize("mode", ["tape", "torch", "engine"])
def test_graph_replay_equals_direct_launches(texty, gi, mode):
    w = C.ClassifierFreeSampleModel(texty[0])
    d = spaced("ddim50")
    dict(_noise_modes(gi))[mode](d)
    kw = dict(model_kwargs=TD._ykw(gi, True), skip_timesteps=44, init_image=gi["x_obs"].to(DEV), order=2)
    torch.manual_seed(8)
    graphed = d.dpm_solver_sde_sample_loop(w, SHAPE, **kw)
    d.use_graph = False
    torch.manual_seed(8)
    direct = d.dpm_solver_sde_sample_loop(w, SHAPE, **kw)
    assert torch.equal(graphed, direct)


def test_launches_per_step_equal_ddpm(plain, gi):
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

    ddpm = {s: launches(d.p_sample_loop, s) for s in (40, 41)}
    for order in (1, 2):
        sde = {s: launches(d.dpm_solver_sde_sample_loop, s, order=order) for s in (40, 41)}
        print(f"order {order}: DDPM {ddpm}, SDE-DPM-Solver++ {sde}")
        assert ddpm[40] - ddpm[41] > 0 and sde[40] - sde[41] == ddpm[40] - ddpm[41]
        assert sde[40] == ddpm[40]


# ------------------------------------------------------------------------------------------------
# batching and sharding
# ------------------------------------------------------------------------------------------------
def test_engine_rng_shards_reproduce_the_unsharded_batch_including_x_T(plain):
    m, _ = plain
    d = spaced("ddim50")
    d.rng, d.engine_seed = "engine", 1234
    full = d.dpm_solver_sde_sample_loop(m, (4, D, 1, L), model_kwargs={"y": {}}, skip_timesteps=46).clone()
    parts = []
    for lo in (0, 2):
        d.sample_offset = lo
        parts.append(d.dpm_solver_sde_sample_loop(m, (2, D, 1, L), model_kwargs={"y": {}}, skip_timesteps=46).clone())
    d.sample_offset = 0
    assert torch.equal(full, torch.cat(parts))
    assert not torch.equal(parts[0], parts[1])
    d.engine_seed = None
    torch.manual_seed(3)
    a = C.sharded_sample(d, m, (4, D, 1, L), {"y": {}}, sampler="dpm_solver_sde_sample_loop", skip_timesteps=46).clone()
    torch.manual_seed(3)
    b = C.sharded_sample(d, m, (4, D, 1, L), {"y": {}}, sampler="dpm_solver_sde_sample_loop", skip_timesteps=46).clone()
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
        run = dict(sampler="dpm_solver_sde_sample_loop", seed=5, skip_timesteps=45)
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
    cases = [
        (dict(dpm_order=0), "dpm_order 0 outside"),
        (dict(dpm_order=3), "dpm_order 3 outside"),
        (dict(dpm_order=2, eta=0.5), "eta"),
        (dict(dpm_order=2, dump_steps=[1]), "dump_xstart"),
        (dict(dpm_order=2, resume=True, init_image=zeros), "init_image"),
    ]
    for kw, msg in cases:
        with pytest.raises(RuntimeError, match=msg):
            eng.sample(B, sampler=SDE, skip_timesteps=45, x_T=x_T, **kw)
    from ctypes import byref
    out = torch.empty(SHAPE, device=DEV)
    for field in ("plms_order", "unipc_order", "unipc_variant", "unipc_corrector"):
        a = C.capi.SampleArgs(B, SDE, 0.0, 45, 0, 0, None, x_T.data_ptr())
        a.dpm_order = 2
        setattr(a, field, 1)
        assert eng.lib.cmdi_sample(eng._h, byref(a), out.data_ptr(), None) != 0
        assert field.encode() in eng.lib.cmdi_last_error()
    a = C.capi.SampleArgs(B, C.capi.SAMPLER_DDPM, 0.0, 45, 0, 0, None, x_T.data_ptr())
    a.dpm_order = 1
    assert eng.lib.cmdi_sample(eng._h, byref(a), out.data_ptr(), None) != 0
    assert b"dpm_order" in eng.lib.cmdi_last_error()

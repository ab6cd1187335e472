"""GPU: the UniPC sampler (unipc_sample_loop[_progressive]) behind the public API, against
  (1) tests/golden/unipc.* -- order 1 without the corrector: the UNMODIFIED reference's ddim_sample_loop at eta = 0; every
      other order, variant and corrector setting: the CPU restatement (oracle/make_golden_unipc.py) -- and
  (2) oracle/unipc_oracle.py run in the test,
at rtol 1e-3 / atol 1e-4 (bf16x3); PRECISION_BF16 and the fp16 UNet with the A/F gates of test_gpu_bf16.py and
test_gpu_unet_guidance.py; order 1 without the corrector against the engine's DPM-Solver++ order 1, bit for bit; and the
bit-for-bit properties (generator == fused loop, graph replay == direct launches, launches per step, the noise contract)
and the errors.
"""
import pytest
import torch

import condmdi_b200 as C
import test_gpu_bf16 as TB
import test_gpu_unet_guidance as TG
from oracle import condmdi_oracle as O
from oracle import unipc_oracle as U
from oracle.golden_io import load_golden
from test_gpu_dpm_solver import _cfg_cond, _unet_fp32_on_gpu, _unet_xl, _ykw, close, spaced

pytestmark = pytest.mark.gpu
B, D, L = 2, 263, 196
SHAPE = (B, D, 1, L)
DEV = "cuda:0"
UNIPC = C.capi.SAMPLER_UNIPC
# every stored run: key -> (order, variant, corrector)
KEYS = {"p1": (1, "bh2", False)}
for _v in U.VARIANTS:
    KEYS.update({f"p{o}_{_v}": (o, _v, False) for o in (2, 3)})
    KEYS.update({f"c{o}_{_v}": (o, _v, True) for o in (1, 2, 3)})


@pytest.fixture(scope="module")
def gold(golden_dir):
    return load_golden(golden_dir, "unipc")


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


def x0_weight(tab, t0, order, variant, corrector):
    """The largest weight one step puts on the x0 errors of the run: sum_j |B_j| of the predictor plus |A| sum_j |C_j|
    of the correction it starts from (the correction's x0 errors reach x_{s-1} through A)."""
    t = U.coefficient_table(tab, t0, order, variant, corrector)[1:t0 + 1]
    return (abs(t[:, 1:4]).sum(1) + abs(t[:, 0]) * abs(t[:, 5:9]).sum(1)).max()


def weighted_gate(respacing, skip, order, variant, corrector):
    """The gate for the bf16x3 tails, derived as test_gpu_dpm_solver.py derives its UNet gate: a step weights each x0
    error by x0_weight instead of DDIM's |B0|, and the largest weight of a ddim50 tail is that of the step into s = 0
    (bh2 orders 2 / 3: 4.5x order 1's, as DPM-Solver++'s 3.80 / 0.85; bh1: 8.8-8.9x, since B_h = hh weights the
    history differences more).  atol scales by the ratio of the run's largest such weight to order 1's without the
    corrector; there the gate is the plain one.  The UNet's x0 already sits at the plain gate's edge at order 1, and the
    transformer's CFG + imputation tails reach 1.4e-4 to 1.6e-4 under bh1."""
    tab = O.make_tables(respacing)
    t0 = tab.num_timesteps - 1 - skip
    ratio = x0_weight(tab, t0, order, variant, corrector) / x0_weight(tab, t0, 1, "bh2", False)
    return dict(rtol=1e-3, atol=1e-4 * max(1.0, ratio))


def run(d, model, key, **kw):
    order, variant, corrector = KEYS[key]
    return d.unipc_sample_loop(model, SHAPE, order=order, variant=variant, corrector=corrector, **kw)


# ------------------------------------------------------------------------------------------------
# transformer and UNet xl, bf16x3: the fixtures (p1 = the reference's DDIM)
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("key", list(KEYS))
def test_golden_transformer(plain, texty, gi, gold, key):
    got = run(spaced("ddim50", gi), plain[0], key, model_kwargs={"y": {}})
    assert got.shape == SHAPE and got.is_cuda
    assert close(got, gold[f"no_cond.{key}"], f"no_cond ddim50 whole loop, {key}")
    if key == "p1":
        assert close(got, gold["no_cond.ddim_ref"], "no_cond ddim50 whole loop, p1 vs the reference's DDIM")
    w = C.ClassifierFreeSampleModel(texty[0])
    x_obs = gi["x_obs"].to(DEV)
    got = run(spaced("ddim50", gi), w, key, model_kwargs=_ykw(gi, False), skip_timesteps=45, init_image=x_obs)
    assert close(got, gold[f"cfg_impute.{key}"], f"cfg 2.5 + imputation, last 5 steps, {key}",
                 **weighted_gate("ddim50", 45, *KEYS[key]))
    # guidance w = 20 at s = 3, 2, none at s = 1, 0 (stop_recguidance_at = 2 inside the loop)
    got = run(spaced("ddim50", gi), w, key, model_kwargs=_ykw(gi, True), skip_timesteps=46, init_image=x_obs)
    assert close(got, gold[f"guided.{key}"], f"cfg + imputation + guidance w=20, last 4 steps, {key}",
                 **weighted_gate("ddim50", 46, *KEYS[key]))
    if key == "p1":
        assert close(got, gold["guided.ddim_ref"], "guided, p1 vs the reference's DDIM")


@pytest.mark.parametrize("key", list(KEYS))
def test_golden_unet_xl_keyframes(gi, gold, key):
    m, _ = _unet_xl(gi)
    w = C.ClassifierFreeSampleModel(m)
    xo, kf = gi["x_obs"].to(DEV), gi["kf_mask"].to(DEV)
    kw = {"y": {"text": ["a", "b"], "text_scale": gi["text_scale"].to(DEV), "mask": gi["y_mask"].to(DEV), "lengths": gi["lengths"]},
          "obs_x0": xo, "obs_mask": kf}
    got = run(spaced("ddim50", gi), w, key, model_kwargs=kw, skip_timesteps=45, init_image=xo)
    assert close(got, gold[f"unet.{key}"], f"keyframe-conditioned MDM_UNET xl, CFG, last 5 steps, {key}",
                 **weighted_gate("ddim50", 45, *KEYS[key]))
    # reconstruction guidance on a bf16x3 MDM_UNET keeps its existing refusal
    kw2 = {"y": dict(kw["y"], reconstruction_guidance=True, reconstruction_weight=20.0, gradient_schedule=None,
                     diffusion_steps=1000, stop_recguidance_at=0, inpainted_motion=xo, inpainting_mask=kf),
           "obs_x0": xo, "obs_mask": kf}
    with pytest.raises(RuntimeError, match="transformer"):
        run(spaced("ddim50", gi), w, key, model_kwargs=kw2, skip_timesteps=48)


# ------------------------------------------------------------------------------------------------
# against the oracle run here
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("order", [1, 2, 3])
def test_ddim20_whole_loops_vs_oracle(plain, texty, gi, order):
    tab = O.make_tables("ddim20")
    for variant, corrector in (("bh2", True), ("bh1", True), ("bh2", False)):
        kw = dict(order=order, variant=variant, corrector=corrector)
        got = spaced("ddim20", gi).unipc_sample_loop(plain[0], SHAPE, model_kwargs={"y": {}}, **kw)
        want = U.unipc_sample_loop(plain[1], tab, SHAPE, O.Conditioning(), gi["tape"], order, variant, corrector)
        assert close(got, want, f"ddim20 no_cond, {kw}")
    w = C.ClassifierFreeSampleModel(texty[0])
    got = spaced("ddim20", gi).unipc_sample_loop(w, SHAPE, model_kwargs=_ykw(gi, False), order=order)
    want = U.unipc_sample_loop(texty[1], tab, SHAPE, _cfg_cond(gi, False), gi["tape"], order)
    assert close(got, want, f"ddim20 cfg + imputation, order {order}, bh2 + corrector")


def test_b64_transformer_tail_vs_oracle(plain):
    m, sd = plain
    Bf = 64
    g = torch.Generator().manual_seed(31)
    tape = torch.randn(1, Bf, D, 1, L, generator=g)
    init = torch.randn(Bf, D, 1, L, generator=g)
    d = spaced("ddim50")
    d.noise_tape = tape.to(DEV)
    for order, variant in ((2, "bh2"), (3, "bh1")):
        got = d.unipc_sample_loop(m, (Bf, D, 1, L), model_kwargs={"y": {}}, skip_timesteps=44, init_image=init.to(DEV),
                                  order=order, variant=variant)
        want = U.unipc_sample_loop(sd, O.make_tables("ddim50"), (Bf, D, 1, L), O.Conditioning(), tape, order, variant,
                                   skip_timesteps=44, init_image=init)
        assert close(got, want, f"B=64 transformer ddim50, order {order} {variant} + corrector, last 6 steps")


def test_b64_unet_xl_cfg_keyframes_tail_vs_oracle():
    Bf = 64
    m, sd = TG.module()
    w = C.ClassifierFreeSampleModel(m)
    x_obs, _, kf, cond, scale = TG.inputs(Bf, seed=41)
    table = {str(i): cond[i].to(DEV) for i in range(Bf)}
    m.encode_text = lambda texts: torch.stack([table[s] for s in texts])
    g = torch.Generator().manual_seed(42)
    tape = torch.randn(1, Bf, D, 1, L, generator=g)
    d = spaced("ddim50")
    d.noise_tape = tape.to(DEV)
    kw = {"y": {"text": [str(i) for i in range(Bf)], "text_scale": scale.to(DEV)}, "obs_x0": x_obs.to(DEV), "obs_mask": kf.to(DEV)}
    got = d.unipc_sample_loop(w, (Bf, D, 1, L), model_kwargs=kw, skip_timesteps=46, init_image=x_obs.to(DEV), order=3)
    c = O.Conditioning(cond_emb=cond, cfg=True, text_scale=scale, obs_x0=x_obs, obs_mask=kf)
    want = _unet_fp32_on_gpu(sd, lambda: U.unipc_sample_loop(sd, O.make_tables("ddim50"), (Bf, D, 1, L), c, tape, 3,
                                                             skip_timesteps=46, init_image=x_obs))
    assert close(got, want, "B=64 MDM_UNET xl, CFG + keyframe input, order 3 bh2 + corrector, last 4 steps",
                 **weighted_gate("ddim50", 46, 3, "bh2", True))


# ------------------------------------------------------------------------------------------------
# PRECISION_BF16 transformer and fp16 UNet: A/F gates
# ------------------------------------------------------------------------------------------------
def test_bf16_transformer_loop_meets_the_contract(gi):
    m, sd = TB.module(text=False)
    sdd = {k: v.to(DEV) for k, v in sd.items()}
    d = spaced("ddim20", gi)
    d.precision = TB.BF16
    got = d.unipc_sample_loop(m, SHAPE, model_kwargs={"y": {}}, skip_timesteps=14, order=2)
    real = O.mdm_forward
    want = {}
    try:
        for name, q in (("A", TB.bf16r), ("F", TB.exact)):
            def fwd(sd_, x, t, cond_emb=None, uncond=False, num_heads=4, _q=q):
                with torch.no_grad():
                    return TB.mdm_model(_q, sdd, x.to(DEV), t.to(DEV), cond_emb, uncond).float().cpu()
            O.mdm_forward = fwd
            want[name] = U.unipc_sample_loop(sd, O.make_tables("ddim20"), SHAPE, O.Conditioning(), gi["tape"], 2,
                                             skip_timesteps=14)
    finally:
        O.mdm_forward = real
    TB.gate(got, want["A"], want["F"], "PRECISION_BF16 ddim20, order 2 bh2 + corrector, last 6 steps")


def test_fp16_unet_xl_loops_meet_the_gates():
    m, w, sd, x_obs, kf, y, c, g = TG.setup(B, seed=51)
    tape = torch.randn(1, B, D, 1, L, generator=g)
    tab = O.make_tables("ddim50")
    kw = {"obs_x0": x_obs.to(DEV), "obs_mask": kf.to(DEV)}

    def run_(y_, c_, order):
        d = spaced("ddim50")
        d.precision = C.PRECISION_FP16
        d.noise_tape = tape.to(DEV)
        got = d.unipc_sample_loop(w, SHAPE, model_kwargs=dict(kw, y=y_), skip_timesteps=45, init_image=x_obs.to(DEV),
                                  order=order)
        a, f = TG.oracle_loop(sd, lambda: U.unipc_sample_loop(sd, tab, SHAPE, c_, tape, order, skip_timesteps=45,
                                                              init_image=x_obs))
        return got, a, f

    y_plain = {k: v for k, v in y.items() if k in ("text", "text_scale", "mask")}
    c_plain = O.Conditioning(cond_emb=c.cond_emb, cfg=True, text_scale=c.text_scale, y_mask=c.y_mask, obs_x0=c.obs_x0,
                             obs_mask=c.obs_mask)
    # loops are gated at track 1.5, as in test_gpu_unet_fp16.py / test_gpu_unet_guidance.py
    TG.gate(*run_(y_plain, c_plain, 3), "fp16 UNet xl, CFG + keyframe input, order 3 + corrector, last 5 steps", track=1.5)
    # guidance w = 20 at s = 4, 3, 2, not at 1, 0
    y_g = dict(y, stop_recguidance_at=2)
    c.stop_recguidance_at = 2
    TG.gate(*run_(y_g, c, 2), "fp16 UNet xl, CFG + guidance w=20 (stop_recguidance_at=2), order 2 + corrector, last 5 steps",
            track=1.5)


# ------------------------------------------------------------------------------------------------
# the engine's DPM-Solver++ and DDIM, and bit-for-bit properties
# ------------------------------------------------------------------------------------------------
def test_order1_without_corrector_equals_engine_dpm_solver_order1(plain, texty, gi):
    """the same float64 rows (A, B0), the same fp32 arithmetic: bit for bit"""
    x_T = gi["tape"][0].to(DEV)
    d = spaced("ddim20")
    for variant in U.VARIANTS:
        dpm = d.dpm_solver_sample_loop(plain[0], SHAPE, noise=x_T, model_kwargs={"y": {}}, order=1)
        uni = d.unipc_sample_loop(plain[0], SHAPE, noise=x_T, model_kwargs={"y": {}}, order=1, variant=variant,
                                  corrector=False)
        assert torch.equal(uni, dpm)
        w = C.ClassifierFreeSampleModel(texty[0])
        dpm = d.dpm_solver_sample_loop(w, SHAPE, noise=x_T, model_kwargs=_ykw(gi, True), skip_timesteps=15, order=1)
        uni = d.unipc_sample_loop(w, SHAPE, noise=x_T, model_kwargs=_ykw(gi, True), skip_timesteps=15, order=1,
                                  variant=variant, corrector=False)
        assert torch.equal(uni, dpm)
        ddim = d.ddim_sample_loop(w, SHAPE, noise=x_T, model_kwargs=_ykw(gi, True), skip_timesteps=15)
        assert close(uni, ddim, "ddim20 guided tail, UniP order 1 vs the engine's DDIM")


@pytest.mark.parametrize("order,variant,corrector", [(1, "bh2", True), (2, "bh1", True), (3, "bh2", True), (3, "bh2", False)])
def test_progressive_equals_fused_and_resume(plain, gi, order, variant, corrector):
    m, _ = plain
    d = spaced("ddim50", gi)
    skip = 40  # 10 steps: the ramp, steady steps and the two lowered final steps
    args = dict(order=order, variant=variant, corrector=corrector)
    outs = [{k: v.clone() for k, v in o.items()} for o in
            d.unipc_sample_loop_progressive(m, SHAPE, model_kwargs={"y": {}}, skip_timesteps=skip, **args)]
    assert len(outs) == 10 and all(set(o) == {"sample", "pred_xstart"} for o in outs)
    fused = d.unipc_sample_loop(m, SHAPE, model_kwargs={"y": {}}, skip_timesteps=skip, **args)
    assert torch.equal(outs[-1]["sample"], fused)
    assert torch.equal(outs[-1]["sample"], outs[-1]["pred_xstart"])  # the last step returns x0
    want = U.unipc_sample_loop(plain[1], O.make_tables("ddim50"), SHAPE, O.Conditioning(), gi["tape"], order, variant,
                               corrector, skip_timesteps=skip, return_all=True)
    for k in (0, 4, 9):  # "sample" is the uncorrected state the next pass evaluates, "pred_xstart" this pass's x0
        assert close(outs[k]["sample"], want[k]["sample"], f"generator step {k} sample")
        assert close(outs[k]["pred_xstart"], want[k]["pred_xstart"], f"generator step {k} pred_xstart")
    eng = m.engine_for(torch.device(DEV), max_batch=B)
    x_T = gi["tape"][0].to(DEV)
    zeros = torch.zeros(SHAPE, device=DEV)
    uk = dict(unipc_order=order, unipc_variant=C.capi.UNIPC_BH1 if variant == "bh1" else C.capi.UNIPC_BH2,
              unipc_corrector=corrector)
    for k in (0, 1, 2, 5):
        res = eng.sample(B, sampler=UNIPC, skip_timesteps=skip, num_steps=k + 1, x_T=x_T, init_image=zeros,
                         want_pred_xstart=True, **uk)
        assert torch.equal(res["sample"], outs[k]["sample"]) and torch.equal(res["pred_xstart"], outs[k]["pred_xstart"])
    # a loop in two chunks: the second call resumes the x0 history and corrected state of the first
    part = eng.sample(B, sampler=UNIPC, skip_timesteps=skip, num_steps=4, x_T=x_T, init_image=zeros, **uk)["sample"]
    rest = eng.sample(B, sampler=UNIPC, skip_timesteps=skip + 4, resume=True, x_T=part, **uk)["sample"]
    assert torch.equal(rest, fused)
    with pytest.raises(RuntimeError, match="does not continue the running history"):
        eng.sample(B, sampler=UNIPC, skip_timesteps=skip + 4, resume=True, x_T=part, **uk)
    # a resume must continue the same variant and corrector setting
    eng.sample(B, sampler=UNIPC, skip_timesteps=skip, num_steps=4, x_T=x_T, init_image=zeros, **uk)
    for change in (dict(unipc_corrector=not corrector),
                   dict(unipc_variant=C.capi.UNIPC_BH2 if variant == "bh1" else C.capi.UNIPC_BH1)):
        with pytest.raises(RuntimeError, match="does not continue the running history"):
            eng.sample(B, sampler=UNIPC, skip_timesteps=skip + 4, resume=True, x_T=part, **dict(uk, **change))


def test_graph_replay_equals_direct_launches(texty, gi):
    w = C.ClassifierFreeSampleModel(texty[0])
    d = spaced("ddim50", gi)
    kw = dict(model_kwargs=_ykw(gi, True), skip_timesteps=44, init_image=gi["x_obs"].to(DEV), order=3)
    graphed = d.unipc_sample_loop(w, SHAPE, **kw)
    d.use_graph = False
    direct = d.unipc_sample_loop(w, SHAPE, **kw)
    assert torch.equal(graphed, direct)


def test_launches_per_step_equal_ddim(plain, gi):
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

    ddim = {s: launches(d.ddim_sample_loop, s) for s in (40, 41)}
    for order in (1, 2, 3):
        for corrector in (False, True):
            uni = {s: launches(d.unipc_sample_loop, s, order=order, corrector=corrector) for s in (40, 41)}
            print(f"order {order} corrector {corrector}: DDIM {ddim}, UniPC {uni}")
            assert ddim[40] - ddim[41] > 0 and uni[40] - uni[41] == ddim[40] - ddim[41]
            assert uni[40] == ddim[40]


def test_torch_rng_draws_x_T_only_and_tape_gives_x_T_only(plain, gi):
    m, _ = plain
    d = spaced("ddim50")
    assert d.rng == "torch" and d.noise_tape is None
    torch.manual_seed(5)
    got = d.unipc_sample_loop(m, SHAPE, model_kwargs={"y": {}}, skip_timesteps=45)
    after = torch.cuda.get_rng_state(DEV)
    torch.manual_seed(5)
    x_T = torch.randn(*SHAPE, device=DEV)
    assert torch.equal(torch.cuda.get_rng_state(DEV), after)  # the generator moved by exactly one randn(*shape)
    assert torch.equal(d.unipc_sample_loop(m, SHAPE, noise=x_T, model_kwargs={"y": {}}, skip_timesteps=45), got)
    torch.manual_seed(5)
    outs = [o["sample"] for o in d.unipc_sample_loop_progressive(m, SHAPE, model_kwargs={"y": {}}, skip_timesteps=45)]
    assert torch.equal(torch.cuda.get_rng_state(DEV), after) and torch.equal(outs[-1], got)
    # a tape contributes tape[0] only
    tape = gi["tape"].to(DEV)
    d.noise_tape = tape
    with_tape = d.unipc_sample_loop(m, SHAPE, model_kwargs={"y": {}}, skip_timesteps=45, order=3)
    d.noise_tape = torch.cat([tape[:1], 100 * tape[1:]])
    assert torch.equal(d.unipc_sample_loop(m, SHAPE, model_kwargs={"y": {}}, skip_timesteps=45, order=3), with_tape)
    d.noise_tape = None
    assert torch.equal(d.unipc_sample_loop(m, SHAPE, noise=tape[0], model_kwargs={"y": {}}, skip_timesteps=45, order=3),
                       with_tape)


def test_c_abi_field_errors(plain, gi):
    m, _ = plain
    eng = m.engine_for(torch.device(DEV), max_batch=B)
    eng.set_schedule(spaced("ddim50").betas, spaced("ddim50").timestep_map)
    x_T = gi["tape"][0].to(DEV)
    zeros = torch.zeros(SHAPE, device=DEV)
    tape = gi["tape"].to(DEV)
    cases = [
        (dict(unipc_order=0), "unipc_order 0 outside"),
        (dict(unipc_order=4), "unipc_order 4 outside"),
        (dict(unipc_variant=3), "unipc_variant 3"),
        (dict(unipc_variant=0), "unipc_variant 0"),
        (dict(eta=0.5), "eta"),
        (dict(noise_tape=tape), "noise_tape"),
        (dict(dump_steps=[1]), "dump_xstart"),
        (dict(resume=True, init_image=zeros), "init_image"),
    ]
    for kw, msg in cases:
        with pytest.raises(RuntimeError, match=msg):
            eng.sample(B, sampler=UNIPC, skip_timesteps=45, x_T=x_T, **kw)
    from ctypes import byref
    out = torch.empty(SHAPE, device=DEV)

    def args(sampler, **fields):
        a = C.capi.SampleArgs(B, sampler, 0.0, 45, 0, 0, None, x_T.data_ptr())
        for k, v in fields.items():
            setattr(a, k, v)
        return a
    good = dict(unipc_order=2, unipc_variant=C.capi.UNIPC_BH2, unipc_corrector=1)
    for sampler, fields, name in [
        (UNIPC, dict(good, plms_order=2), b"plms_order"),
        (UNIPC, dict(good, dpm_order=2), b"dpm_order"),
        (UNIPC, dict(good, unipc_corrector=2), b"unipc_corrector"),
        (C.capi.SAMPLER_DDIM, dict(unipc_order=2), b"unipc_order"),
        (C.capi.SAMPLER_DPM_SOLVER, dict(dpm_order=2, unipc_variant=2), b"unipc_variant"),
        (C.capi.SAMPLER_DDIM, dict(unipc_corrector=1), b"unipc_corrector"),
    ]:
        assert eng.lib.cmdi_sample(eng._h, byref(args(sampler, **fields)), out.data_ptr(), None) != 0, (sampler, fields)
        assert name in eng.lib.cmdi_last_error(), (name, eng.lib.cmdi_last_error())
    assert eng.lib.cmdi_sample(eng._h, byref(args(UNIPC, **good)), out.data_ptr(), None) == 0

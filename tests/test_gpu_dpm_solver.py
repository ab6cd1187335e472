"""GPU: the DPM-Solver++ sampler (dpm_solver_sample_loop[_progressive]) behind the public API, against
  (1) tests/golden/dpm_solver.* -- order 1: the UNMODIFIED reference's ddim_sample_loop at eta = 0; orders 2 / 3: the CPU
      restatement (oracle/make_golden_dpm_solver.py) -- and
  (2) oracle/dpm_solver_oracle.py run in the test,
at rtol 1e-3 / atol 1e-4 (bf16x3); PRECISION_BF16 and the fp16 UNet with the A/F gates of test_gpu_bf16.py and
test_gpu_unet_guidance.py; order 1 against the engine's own DDIM; and the bit-for-bit properties (generator == fused loop,
graph replay == direct launches, launches per step, the noise contract) and the errors.
"""
import pytest
import torch

import condmdi_b200 as C
import test_gpu_bf16 as TB
import test_gpu_unet_guidance as TG
from oracle import condmdi_oracle as O
from oracle import dpm_solver_oracle as S
from oracle.golden_io import load_golden

pytestmark = pytest.mark.gpu
GATE = dict(rtol=1e-3, atol=1e-4)
B, D, L = 2, 263, 196
SHAPE = (B, D, 1, L)
DEV = "cuda:0"
DPM = C.capi.SAMPLER_DPM_SOLVER


@pytest.fixture(scope="module")
def gold(golden_dir):
    return load_golden(golden_dir, "dpm_solver")


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


def close(a, b, what="", **tol):
    tol = tol or GATE
    a, b = torch.as_tensor(a).cpu().float(), torch.as_tensor(b).cpu().float()
    err = (a - b).abs()
    print(f"[{what}] max_abs={err.max():.3e} mean_abs={err.mean():.3e}")
    return torch.allclose(a, b, **tol)


def unet_gate(respacing, skip, order):
    """The gate for bf16x3 MDM_UNET runs.  The UNet's x0 already sits at the parity gate's edge at order 1 (max 1.0e-4
    over a CFG tail, inside rtol 1e-3 / atol 1e-4 only through rtol), and orders 2 / 3 weight each step's x0 error by
    sum_j |B_j| instead of DDIM's |B0| (3.80 against 0.85 at s = 1 of a ddim50 tail).  atol scales by the ratio of the
    largest such weight of the run to order 1's; at order 1 the gate is the plain one."""
    tab = O.make_tables(respacing)
    t0 = tab.num_timesteps - 1 - skip

    def weight(o):
        return abs(S.coefficient_table(tab, t0, o)[1:t0 + 1, 1:]).sum(1).max()
    return dict(rtol=1e-3, atol=1e-4 * max(1.0, weight(order) / weight(1)))


def spaced(respacing, gi=None):
    d = C.create_gaussian_diffusion(timestep_respacing=respacing)
    if gi is not None:
        d.noise_tape = gi["tape"].to(DEV)  # DPM-Solver++ reads tape[0] (x_T) only
    return d


def _ykw(gi, guided):
    y = {"text": ["a", "b"], "text_scale": gi["text_scale"].to(DEV), "mask": gi["y_mask"].to(DEV), "lengths": gi["lengths"],
         "imputate": 1, "stop_imputation_at": 1, "replacement_distribution": "conditional",
         "inpainted_motion": gi["x_obs"].to(DEV), "inpainting_mask": gi["kf_mask"].to(DEV)}
    if guided:
        y.update(reconstruction_guidance=True, reconstruction_weight=20.0, gradient_schedule=None, diffusion_steps=1000,
                 stop_recguidance_at=2)
    return {"y": y}


def _cfg_cond(gi, guided):
    kw = dict(cond_emb=gi["cond"], cfg=True, text_scale=gi["text_scale"], y_mask=gi["y_mask"], imputate=True,
              stop_imputation_at=1, inpainted_motion=gi["x_obs"], inpainting_mask=gi["kf_mask"])
    if guided:
        kw.update(reconstruction_guidance=True, reconstruction_weight=20.0, stop_recguidance_at=2)
    return O.Conditioning(**kw)


def _unet_xl(gi):
    sd = O.random_unet_state_dict(seed=11, text=True)
    m = C.MDM_UNET(keyframe_conditioned=True, cond_mode="text", cond_mask_prob=0.1)
    assert not any(m.load_state_dict(sd, strict=False))
    m = m.to(DEV)
    table = {"a": gi["cond"][0].to(DEV), "b": gi["cond"][1].to(DEV)}
    m.encode_text = lambda texts: torch.stack([table[t] for t in texts])
    return m, sd


# ------------------------------------------------------------------------------------------------
# transformer and UNet xl, bf16x3: the fixtures (order 1 = the reference's DDIM)
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("order", [1, 2, 3])
def test_golden_transformer(plain, texty, gi, gold, order):
    want = {1: "ddim_ref", 2: "o2", 3: "o3"}[order]
    got = spaced("ddim50", gi).dpm_solver_sample_loop(plain[0], SHAPE, model_kwargs={"y": {}}, order=order)
    assert got.shape == SHAPE and got.is_cuda
    assert close(got, gold[f"no_cond.{want}"], f"no_cond ddim50 whole loop, order {order}")
    w = C.ClassifierFreeSampleModel(texty[0])
    x_obs = gi["x_obs"].to(DEV)
    got = spaced("ddim50", gi).dpm_solver_sample_loop(w, SHAPE, model_kwargs=_ykw(gi, False), skip_timesteps=45,
                                                      init_image=x_obs, order=order)
    assert close(got, gold[f"cfg_impute.{want}"], f"cfg 2.5 + imputation, last 5 steps, order {order}")
    # guidance w = 20 at s = 3, 2, none at s = 1, 0 (stop_recguidance_at = 2 inside the loop)
    got = spaced("ddim50", gi).dpm_solver_sample_loop(w, SHAPE, model_kwargs=_ykw(gi, True), skip_timesteps=46,
                                                      init_image=x_obs, order=order)
    assert close(got, gold[f"guided.{want}"], f"cfg + imputation + guidance w=20, last 4 steps, order {order}")


@pytest.mark.parametrize("order", [1, 2, 3])
def test_golden_unet_xl_keyframes(gi, gold, order):
    m, _ = _unet_xl(gi)
    w = C.ClassifierFreeSampleModel(m)
    xo, kf = gi["x_obs"].to(DEV), gi["kf_mask"].to(DEV)
    kw = {"y": {"text": ["a", "b"], "text_scale": gi["text_scale"].to(DEV), "mask": gi["y_mask"].to(DEV), "lengths": gi["lengths"]},
          "obs_x0": xo, "obs_mask": kf}
    got = spaced("ddim50", gi).dpm_solver_sample_loop(w, SHAPE, model_kwargs=kw, skip_timesteps=45, init_image=xo, order=order)
    want = {1: "ddim_ref", 2: "o2", 3: "o3"}[order]
    assert close(got, gold[f"unet.{want}"], f"keyframe-conditioned MDM_UNET xl, CFG, last 5 steps, order {order}",
                 **unet_gate("ddim50", 45, order))
    # reconstruction guidance on a bf16x3 MDM_UNET keeps its existing refusal
    kw2 = {"y": dict(kw["y"], reconstruction_guidance=True, reconstruction_weight=20.0, gradient_schedule=None,
                     diffusion_steps=1000, stop_recguidance_at=0, inpainted_motion=xo, inpainting_mask=kf),
           "obs_x0": xo, "obs_mask": kf}
    with pytest.raises(RuntimeError, match="transformer"):
        spaced("ddim50", gi).dpm_solver_sample_loop(w, SHAPE, model_kwargs=kw2, skip_timesteps=48, order=order)


# ------------------------------------------------------------------------------------------------
# against the oracle run here
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("order", [1, 2, 3])
def test_ddim20_whole_loops_vs_oracle(plain, texty, gi, order):
    tab = O.make_tables("ddim20")
    got = spaced("ddim20", gi).dpm_solver_sample_loop(plain[0], SHAPE, model_kwargs={"y": {}}, order=order)
    want = S.dpm_solver_sample_loop(plain[1], tab, SHAPE, O.Conditioning(), gi["tape"], order)
    assert close(got, want, f"ddim20 no_cond, order {order}")
    w = C.ClassifierFreeSampleModel(texty[0])
    got = spaced("ddim20", gi).dpm_solver_sample_loop(w, SHAPE, model_kwargs=_ykw(gi, False), order=order)
    want = S.dpm_solver_sample_loop(texty[1], tab, SHAPE, _cfg_cond(gi, False), gi["tape"], order)
    assert close(got, want, f"ddim20 cfg + imputation, order {order}")


def test_b64_transformer_tail_order2_vs_oracle(plain):
    m, sd = plain
    Bf = 64
    g = torch.Generator().manual_seed(31)
    tape = torch.randn(1, Bf, D, 1, L, generator=g)
    init = torch.randn(Bf, D, 1, L, generator=g)
    d = spaced("ddim50")
    d.noise_tape = tape.to(DEV)
    got = d.dpm_solver_sample_loop(m, (Bf, D, 1, L), model_kwargs={"y": {}}, skip_timesteps=45, init_image=init.to(DEV), order=2)
    want = S.dpm_solver_sample_loop(sd, O.make_tables("ddim50"), (Bf, D, 1, L), O.Conditioning(), tape, 2, skip_timesteps=45,
                                    init_image=init)
    assert close(got, want, "B=64 transformer ddim50, order 2, last 5 steps")


def _unet_fp32_on_gpu(sd, run):
    """run() with the oracle's UNet evaluated on the GPU in exact fp32 (the CPU restatement at B = 64 would take minutes)"""
    sdd = {k: v.to(DEV) for k, v in sd.items()}

    def gpu_forward(sd_, x, t, cond_emb=None, uncond=False, obs_x0=None, obs_mask=None):
        dev = lambda v: None if v is None else v.to(DEV)  # noqa: E731
        with TG.exact_fp32(), torch.no_grad():
            return TG.UNET_FORWARD(sdd, dev(x), dev(t), dev(cond_emb), uncond, dev(obs_x0), dev(obs_mask)).float().cpu()
    try:
        O.unet_forward = gpu_forward
        return run()
    finally:
        O.unet_forward = TG.UNET_FORWARD


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
    got = d.dpm_solver_sample_loop(w, (Bf, D, 1, L), model_kwargs=kw, skip_timesteps=46, init_image=x_obs.to(DEV), order=3)
    c = O.Conditioning(cond_emb=cond, cfg=True, text_scale=scale, obs_x0=x_obs, obs_mask=kf)
    want = _unet_fp32_on_gpu(sd, lambda: S.dpm_solver_sample_loop(sd, O.make_tables("ddim50"), (Bf, D, 1, L), c, tape, 3,
                                                                  skip_timesteps=46, init_image=x_obs))
    assert close(got, want, "B=64 MDM_UNET xl, CFG + keyframe input, order 3, last 4 steps", **unet_gate("ddim50", 46, 3))


# ------------------------------------------------------------------------------------------------
# PRECISION_BF16 transformer and fp16 UNet: A/F gates
# ------------------------------------------------------------------------------------------------
def test_bf16_transformer_loop_meets_the_contract(gi):
    m, sd = TB.module(text=False)
    sdd = {k: v.to(DEV) for k, v in sd.items()}
    d = spaced("ddim20", gi)
    d.precision = TB.BF16
    got = d.dpm_solver_sample_loop(m, SHAPE, model_kwargs={"y": {}}, skip_timesteps=14, order=2)
    real = O.mdm_forward
    want = {}
    try:
        for name, q in (("A", TB.bf16r), ("F", TB.exact)):
            def fwd(sd_, x, t, cond_emb=None, uncond=False, num_heads=4, _q=q):
                with torch.no_grad():
                    return TB.mdm_model(_q, sdd, x.to(DEV), t.to(DEV), cond_emb, uncond).float().cpu()
            O.mdm_forward = fwd
            want[name] = S.dpm_solver_sample_loop(sd, O.make_tables("ddim20"), SHAPE, O.Conditioning(), gi["tape"], 2,
                                                  skip_timesteps=14)
    finally:
        O.mdm_forward = real
    TB.gate(got, want["A"], want["F"], "PRECISION_BF16 ddim20, order 2, last 6 steps")


def test_fp16_unet_xl_loops_meet_the_gates():
    m, w, sd, x_obs, kf, y, c, g = TG.setup(B, seed=51)
    tape = torch.randn(1, B, D, 1, L, generator=g)
    tab = O.make_tables("ddim50")
    kw = {"obs_x0": x_obs.to(DEV), "obs_mask": kf.to(DEV)}

    def run(y_, c_, order):
        d = spaced("ddim50")
        d.precision = C.PRECISION_FP16
        d.noise_tape = tape.to(DEV)
        got = d.dpm_solver_sample_loop(w, SHAPE, model_kwargs=dict(kw, y=y_), skip_timesteps=45, init_image=x_obs.to(DEV),
                                       order=order)
        a, f = TG.oracle_loop(sd, lambda: S.dpm_solver_sample_loop(sd, tab, SHAPE, c_, tape, order, skip_timesteps=45,
                                                                   init_image=x_obs))
        return got, a, f

    y_plain = {k: v for k, v in y.items() if k in ("text", "text_scale", "mask")}
    c_plain = O.Conditioning(cond_emb=c.cond_emb, cfg=True, text_scale=c.text_scale, y_mask=c.y_mask, obs_x0=c.obs_x0,
                             obs_mask=c.obs_mask)
    # loops are gated at track 1.5, as in test_gpu_unet_fp16.py / test_gpu_unet_guidance.py
    TG.gate(*run(y_plain, c_plain, 3), "fp16 UNet xl, CFG + keyframe input, order 3, last 5 steps", track=1.5)
    # guidance w = 20 at s = 4, 3, 2, not at 1, 0
    y_g = dict(y, stop_recguidance_at=2)
    c.stop_recguidance_at = 2
    TG.gate(*run(y_g, c, 2), "fp16 UNet xl, CFG + guidance w=20 (stop_recguidance_at=2), order 2, last 5 steps", track=1.5)


# ------------------------------------------------------------------------------------------------
# the engine's own DDIM, and bit-for-bit properties
# ------------------------------------------------------------------------------------------------
def test_order1_equals_engine_ddim(plain, texty, gi):
    x_T = gi["tape"][0].to(DEV)
    d = spaced("ddim20")
    ddim = d.ddim_sample_loop(plain[0], SHAPE, noise=x_T, model_kwargs={"y": {}})
    dpm = d.dpm_solver_sample_loop(plain[0], SHAPE, noise=x_T, model_kwargs={"y": {}}, order=1)
    assert close(dpm, ddim, "ddim20 order 1 vs the engine's DDIM")
    w = C.ClassifierFreeSampleModel(texty[0])
    ddim = d.ddim_sample_loop(w, SHAPE, noise=x_T, model_kwargs=_ykw(gi, True), skip_timesteps=15)
    dpm = d.dpm_solver_sample_loop(w, SHAPE, noise=x_T, model_kwargs=_ykw(gi, True), skip_timesteps=15, order=1)
    assert close(dpm, ddim, "ddim20 guided tail, order 1 vs the engine's DDIM")


@pytest.mark.parametrize("order", [1, 2, 3])
def test_progressive_equals_fused_and_resume(plain, gi, order):
    m, _ = plain
    d = spaced("ddim50", gi)
    skip = 40  # 10 steps: the ramp, steady steps and the two lowered final steps
    outs = [{k: v.clone() for k, v in o.items()} for o in
            d.dpm_solver_sample_loop_progressive(m, SHAPE, model_kwargs={"y": {}}, skip_timesteps=skip, order=order)]
    assert len(outs) == 10 and all(set(o) == {"sample", "pred_xstart"} for o in outs)
    fused = d.dpm_solver_sample_loop(m, SHAPE, model_kwargs={"y": {}}, skip_timesteps=skip, order=order)
    assert torch.equal(outs[-1]["sample"], fused)
    assert torch.equal(outs[-1]["sample"], outs[-1]["pred_xstart"])  # the last step returns x0
    eng = m.engine_for(torch.device(DEV), max_batch=B)
    x_T = gi["tape"][0].to(DEV)
    zeros = torch.zeros(SHAPE, device=DEV)
    for k in (0, 1, 2, 5):
        res = eng.sample(B, sampler=DPM, skip_timesteps=skip, num_steps=k + 1, x_T=x_T, init_image=zeros, dpm_order=order,
                         want_pred_xstart=True)
        assert torch.equal(res["sample"], outs[k]["sample"]) and torch.equal(res["pred_xstart"], outs[k]["pred_xstart"])
    # a loop in two chunks: the second call resumes the x0 history of the first
    part = eng.sample(B, sampler=DPM, skip_timesteps=skip, num_steps=4, x_T=x_T, init_image=zeros, dpm_order=order)["sample"]
    rest = eng.sample(B, sampler=DPM, skip_timesteps=skip + 4, resume=True, x_T=part, dpm_order=order)["sample"]
    assert torch.equal(rest, fused)
    with pytest.raises(RuntimeError, match="does not continue the running history"):
        eng.sample(B, sampler=DPM, skip_timesteps=skip + 4, resume=True, x_T=part, dpm_order=order)


def test_graph_replay_equals_direct_launches(texty, gi):
    w = C.ClassifierFreeSampleModel(texty[0])
    d = spaced("ddim50", gi)
    kw = dict(model_kwargs=_ykw(gi, True), skip_timesteps=44, init_image=gi["x_obs"].to(DEV), order=3)
    graphed = d.dpm_solver_sample_loop(w, SHAPE, **kw)
    d.use_graph = False
    direct = d.dpm_solver_sample_loop(w, SHAPE, **kw)
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
        dpm = {s: launches(d.dpm_solver_sample_loop, s, order=order) for s in (40, 41)}
        print(f"order {order}: DDIM {ddim}, DPM-Solver++ {dpm}")
        assert ddim[40] - ddim[41] > 0 and dpm[40] - dpm[41] == ddim[40] - ddim[41]
        assert dpm[40] == ddim[40]


def test_torch_rng_draws_x_T_only_and_tape_gives_x_T_only(plain, gi):
    m, _ = plain
    d = spaced("ddim50")
    assert d.rng == "torch" and d.noise_tape is None
    torch.manual_seed(5)
    got = d.dpm_solver_sample_loop(m, SHAPE, model_kwargs={"y": {}}, skip_timesteps=45)
    after = torch.cuda.get_rng_state(DEV)
    torch.manual_seed(5)
    x_T = torch.randn(*SHAPE, device=DEV)
    assert torch.equal(torch.cuda.get_rng_state(DEV), after)  # the generator moved by exactly one randn(*shape)
    assert torch.equal(d.dpm_solver_sample_loop(m, SHAPE, noise=x_T, model_kwargs={"y": {}}, skip_timesteps=45), got)
    torch.manual_seed(5)
    outs = [o["sample"] for o in d.dpm_solver_sample_loop_progressive(m, SHAPE, model_kwargs={"y": {}}, skip_timesteps=45)]
    assert torch.equal(torch.cuda.get_rng_state(DEV), after) and torch.equal(outs[-1], got)
    # a tape contributes tape[0] only
    tape = gi["tape"].to(DEV)
    d.noise_tape = tape
    with_tape = d.dpm_solver_sample_loop(m, SHAPE, model_kwargs={"y": {}}, skip_timesteps=45, order=2)
    d.noise_tape = torch.cat([tape[:1], 100 * tape[1:]])
    assert torch.equal(d.dpm_solver_sample_loop(m, SHAPE, model_kwargs={"y": {}}, skip_timesteps=45, order=2), with_tape)
    d.noise_tape = None
    assert torch.equal(d.dpm_solver_sample_loop(m, SHAPE, noise=tape[0], model_kwargs={"y": {}}, skip_timesteps=45, order=2),
                       with_tape)


def test_c_abi_field_errors(plain, gi):
    m, _ = plain
    eng = m.engine_for(torch.device(DEV), max_batch=B)
    eng.set_schedule(spaced("ddim50").betas, spaced("ddim50").timestep_map)
    x_T = gi["tape"][0].to(DEV)
    zeros = torch.zeros(SHAPE, device=DEV)
    tape = gi["tape"].to(DEV)
    cases = [
        (dict(dpm_order=0), "dpm_order 0 outside"),
        (dict(dpm_order=4), "dpm_order 4 outside"),
        (dict(dpm_order=2, eta=0.5), "eta"),
        (dict(dpm_order=2, noise_tape=tape), "noise_tape"),
        (dict(dpm_order=2, dump_steps=[1]), "dump_xstart"),
        (dict(dpm_order=2, resume=True, init_image=zeros), "init_image"),
    ]
    for kw, msg in cases:
        with pytest.raises(RuntimeError, match=msg):
            eng.sample(B, sampler=DPM, skip_timesteps=45, x_T=x_T, **kw)
    from ctypes import byref
    a = C.capi.SampleArgs(B, DPM, 0.0, 45, 0, 0, None, x_T.data_ptr())
    a.dpm_order, a.plms_order = 2, 2
    out = torch.empty(SHAPE, device=DEV)
    assert eng.lib.cmdi_sample(eng._h, byref(a), out.data_ptr(), None) != 0
    assert b"plms_order" in eng.lib.cmdi_last_error()
    a.plms_order, a.sampler = 0, C.capi.SAMPLER_DDIM
    assert eng.lib.cmdi_sample(eng._h, byref(a), out.data_ptr(), None) != 0
    assert b"dpm_order" in eng.lib.cmdi_last_error()

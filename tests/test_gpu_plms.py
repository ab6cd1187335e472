"""GPU: the PLMS sampler (plms_sample_loop / plms_sample_loop_progressive, gaussian_diffusion.py:1589-1804) behind the public
API, against
  (1) tests/golden/plms.* -- outputs of the UNMODIFIED reference (oracle/make_golden_plms.py), and
  (2) the CPU oracle at B = 64,
at rtol 1e-3 / atol 1e-4; the progressive generator against the fused loop bit for bit; the noise contract; errors; and the
launch accounting.
"""
import pytest
import torch

import condmdi_b200 as C
from oracle import condmdi_oracle as O
from oracle import plms_oracle as P
from oracle.golden_io import load_golden

pytestmark = pytest.mark.gpu
GATE = dict(rtol=1e-3, atol=1e-4)
B, D, L = 2, 263, 196
SHAPE = (B, D, 1, L)
DEV = "cuda:0"


@pytest.fixture(scope="module")
def gold(golden_dir):
    return load_golden(golden_dir, "plms")


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


def ddim50(gi):
    d = C.create_gaussian_diffusion(timestep_respacing="ddim50")
    d.noise_tape = gi["tape"].to(DEV)  # PLMS reads tape[0] (x_T) only
    return d


def first(gen, n):
    outs = []
    for k, o in enumerate(gen):
        outs.append({"sample": o["sample"].clone(), "pred_xstart": o["pred_xstart"].clone(), "old_eps": [e.clone() for e in o["old_eps"]]})
        if k + 1 == n:
            break
    return outs


# ------------------------------------------------------------------------------------------------
# the reference's own outputs
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("order,ks", [(2, (0, 1, 2)), (4, (3,))])
def test_plms_ddim50_vs_reference_golden(plain, gi, gold, order, ks):
    m, _ = plain
    d = ddim50(gi)
    outs = first(d.plms_sample_loop_progressive(m, SHAPE, model_kwargs={"y": {}}, order=order), max(ks) + 1)
    for k in ks:
        assert close(outs[k]["sample"], gold[f"o{order}.sample_k{k}"], f"order {order} after k={k}")
        assert len(outs[k]["old_eps"]) == min(k + 1, order - 1)
    got = d.plms_sample_loop(m, SHAPE, model_kwargs={"y": {}}, clip_denoised=False, order=order)
    assert got.shape == SHAPE and got.is_cuda
    assert close(got, gold[f"o{order}.final"], f"order {order} whole loop")


def _ykw(gi, guided):
    y = {"text": ["a", "b"], "text_scale": gi["text_scale"].to(DEV), "mask": gi["y_mask"].to(DEV), "lengths": gi["lengths"],
         "imputate": 1, "stop_imputation_at": 1, "replacement_distribution": "conditional",
         "inpainted_motion": gi["x_obs"].to(DEV), "inpainting_mask": gi["kf_mask"].to(DEV)}
    if guided:
        y.update(reconstruction_guidance=True, reconstruction_weight=20.0, gradient_schedule=None, diffusion_steps=1000,
                 stop_recguidance_at=0)
    return {"y": y}


def test_plms_cfg_imputation_vs_reference_golden(texty, gi, gold):
    m, _ = texty
    w = C.ClassifierFreeSampleModel(m)
    got = ddim50(gi).plms_sample_loop(w, SHAPE, model_kwargs=_ykw(gi, False), skip_timesteps=45, init_image=gi["x_obs"].to(DEV))
    assert close(got, gold["cfg_impute.final"], "cfg 2.5 + imputation, last 5 steps")


def test_plms_reconstruction_guidance_vs_reference_golden(texty, gi, gold):
    """the first step runs two guided evaluations, the second one at t - 1"""
    m, _ = texty
    w = C.ClassifierFreeSampleModel(m)
    outs = first(ddim50(gi).plms_sample_loop_progressive(w, SHAPE, model_kwargs=_ykw(gi, True)), 2)
    assert close(outs[1]["sample"], gold["recon.sample_k1"], "cfg + imputation + guidance w=20, 2 steps")


def test_plms_one_step_at_t0_vs_reference_golden(plain, gi, gold):
    m, _ = plain
    outs = list(ddim50(gi).plms_sample_loop_progressive(m, SHAPE, model_kwargs={"y": {}}, skip_timesteps=49,
                                                         init_image=gi["x_obs"].to(DEV)))
    assert len(outs) == 1 and len(outs[0]["old_eps"]) == 1
    assert torch.equal(outs[0]["sample"], outs[0]["pred_xstart"])
    assert close(outs[0]["sample"], gold["t0.sample"], "one step at t = 0")
    got = ddim50(gi).plms_sample_loop(m, SHAPE, model_kwargs={"y": {}}, skip_timesteps=49, init_image=gi["x_obs"].to(DEV))
    assert torch.equal(got, outs[0]["sample"])


def test_plms_unet_xl_order3_vs_reference_golden(gi, gold):
    sd = O.random_unet_state_dict(seed=11, text=True)
    m = C.MDM_UNET(keyframe_conditioned=True, cond_mode="text", cond_mask_prob=0.1)
    assert not any(m.load_state_dict(sd, strict=False))
    m = m.to(DEV)
    table = {"a": gi["cond"][0].to(DEV), "b": gi["cond"][1].to(DEV)}
    m.encode_text = lambda texts: torch.stack([table[t] for t in texts])
    w = C.ClassifierFreeSampleModel(m)
    xo, kf = gi["x_obs"].to(DEV), gi["kf_mask"].to(DEV)
    kw = {"y": {"text": ["a", "b"], "text_scale": gi["text_scale"].to(DEV), "mask": gi["y_mask"].to(DEV), "lengths": gi["lengths"]},
          "obs_x0": xo, "obs_mask": kf}
    got = ddim50(gi).plms_sample_loop(w, SHAPE, model_kwargs=kw, skip_timesteps=45, init_image=xo, order=3)
    assert close(got, gold["unet.final"], "keyframe-conditioned MDM_UNET xl, CFG, order 3, last 5 steps")
    # reconstruction guidance needs the denoiser's input-VJP, which exists for the transformer only
    kw2 = {"y": dict(kw["y"], reconstruction_guidance=True, reconstruction_weight=20.0, gradient_schedule=None, diffusion_steps=1000,
                     stop_recguidance_at=0, inpainted_motion=xo, inpainting_mask=kf), "obs_x0": xo, "obs_mask": kf}
    with pytest.raises(RuntimeError, match="transformer"):
        ddim50(gi).plms_sample_loop(w, SHAPE, model_kwargs=kw2, skip_timesteps=48)


# ------------------------------------------------------------------------------------------------
# B = 64 against the oracle
# ------------------------------------------------------------------------------------------------
def test_plms_b64_transformer_tail_vs_oracle(plain):
    m, sd = plain
    Bf = 64
    g = torch.Generator().manual_seed(21)
    tape = torch.randn(1, Bf, D, 1, L, generator=g)
    init = torch.randn(Bf, D, 1, L, generator=g)
    d = C.create_gaussian_diffusion(timestep_respacing="ddim50")
    d.noise_tape = tape.to(DEV)
    got = d.plms_sample_loop(m, (Bf, D, 1, L), model_kwargs={"y": {}}, skip_timesteps=46, init_image=init.to(DEV), order=2)
    want = P.plms_sample_loop(sd, O.make_tables("ddim50"), (Bf, D, 1, L), O.Conditioning(), tape, skip_timesteps=46,
                              init_image=init, order=2)
    assert close(got, want, "B=64 transformer, order 2, last 4 steps")


def test_plms_b64_unet_tail_with_imputation_vs_oracle():
    Bf = 64
    g = torch.Generator().manual_seed(22)
    sd = O.random_unet_state_dict(seed=5, mults=(1, 1))
    m = C.MDM_UNET(dim_mults=(1, 1), keyframe_conditioned=True)
    m.load_state_dict(sd, strict=False)
    m = m.to(DEV)
    x_obs = torch.randn(Bf, D, 1, L, generator=g)
    lengths = torch.randint(20, 197, (Bf,), generator=g)
    kf = C.get_keyframes_mask(x_obs, lengths, "benchmark_sparse", trans_length=5)
    y_mask = (torch.arange(L)[None] < lengths[:, None]).view(Bf, 1, 1, L)
    tape = torch.randn(1, Bf, D, 1, L, generator=g)
    d = C.create_gaussian_diffusion(timestep_respacing="ddim50")
    d.noise_tape = tape.to(DEV)
    y = {"mask": y_mask.to(DEV), "imputate": 1, "stop_imputation_at": 1, "replacement_distribution": "conditional",
         "inpainted_motion": x_obs.to(DEV), "inpainting_mask": kf.to(DEV)}
    got = d.plms_sample_loop(m, (Bf, D, 1, L), model_kwargs={"y": y, "obs_x0": x_obs.to(DEV), "obs_mask": kf.to(DEV)},
                             skip_timesteps=45, init_image=x_obs.to(DEV), order=3)
    c = O.Conditioning(y_mask=y_mask, imputate=True, stop_imputation_at=1, inpainted_motion=x_obs, inpainting_mask=kf, obs_x0=x_obs,
                       obs_mask=kf)
    want = P.plms_sample_loop(sd, O.make_tables("ddim50"), (Bf, D, 1, L), c, tape, skip_timesteps=45, init_image=x_obs, order=3)
    assert close(got, want, "B=64 2-level UNet, keyframe input + imputation, order 3, last 5 steps")


# ------------------------------------------------------------------------------------------------
# progressive == fused, noise, launches
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("order", [2, 3, 4])
def test_plms_progressive_equals_fused_bit_for_bit(plain, gi, order):
    m, sd = plain
    d = ddim50(gi)
    skip = 38  # 12 steps: the first step, the ramp and steady Adams-Bashforth steps, down to t = 0
    outs = first(d.plms_sample_loop_progressive(m, SHAPE, model_kwargs={"y": {}}, skip_timesteps=skip, order=order), 12)
    assert len(outs) == 12
    fused = d.plms_sample_loop(m, SHAPE, model_kwargs={"y": {}}, skip_timesteps=skip, order=order)
    assert torch.equal(outs[-1]["sample"], fused)
    # the history after k + 1 steps of one fused call equals the history the generator yielded at step k
    eng = m.engine_for(torch.device(DEV), max_batch=B)
    x_T = gi["tape"][0].to(DEV)
    for k in (0, 1, 2, 3, 11):
        res = eng.sample(B, sampler=C.capi.SAMPLER_PLMS, skip_timesteps=skip, num_steps=k + 1, x_T=x_T,
                         init_image=torch.zeros(SHAPE, device=DEV), plms_order=order, want_pred_xstart=True, want_old_eps=True)
        assert torch.equal(res["sample"], outs[k]["sample"]) and torch.equal(res["pred_xstart"], outs[k]["pred_xstart"])
        assert len(res["old_eps"]) == len(outs[k]["old_eps"]) == min(k + 1, order - 1)
        for a, b in zip(res["old_eps"], outs[k]["old_eps"]):
            assert torch.equal(a, b)
    # ... and the old_eps values are the reference's (the oracle restates them; eps carries 1 / sqrt(1/abar - 1))
    want = P.plms_sample_loop(sd, O.make_tables("ddim50"), SHAPE, O.Conditioning(), gi["tape"], skip_timesteps=skip,
                              return_all=True, max_steps=4, order=order)
    for k in range(4):
        assert close(outs[k]["sample"], want[k]["sample"], f"order {order} k={k}")
        for a, b in zip(outs[k]["old_eps"], want[k]["old_eps"]):
            assert close(a, b, f"order {order} k={k} old_eps", rtol=1e-3, atol=1e-3)


def test_plms_torch_rng_draws_x_T_only(plain):
    m, _ = plain
    d = C.create_gaussian_diffusion(timestep_respacing="ddim50")
    assert d.rng == "torch" and d.noise_tape is None
    torch.manual_seed(5)
    got = d.plms_sample_loop(m, SHAPE, model_kwargs={"y": {}}, skip_timesteps=46)
    after = torch.cuda.get_rng_state(DEV)
    torch.manual_seed(5)
    x_T = torch.randn(*SHAPE, device=DEV)
    assert torch.equal(torch.cuda.get_rng_state(DEV), after)  # the generator moved by exactly one randn(*shape)
    assert torch.equal(d.plms_sample_loop(m, SHAPE, noise=x_T, model_kwargs={"y": {}}, skip_timesteps=46), got)
    torch.manual_seed(5)
    gen = d.plms_sample_loop_progressive(m, SHAPE, model_kwargs={"y": {}}, skip_timesteps=46)
    outs = [o["sample"] for o in gen]
    assert torch.equal(torch.cuda.get_rng_state(DEV), after) and torch.equal(outs[-1], got)
    # rng="engine": x_T keyed by global sample index -> a half batch at sample_offset 1 reproduces sample 1
    d.rng, d.engine_seed = "engine", 1234
    full = d.plms_sample_loop(m, SHAPE, model_kwargs={"y": {}}, skip_timesteps=46)
    d.sample_offset = 1
    half = d.plms_sample_loop(m, (1, D, 1, L), model_kwargs={"y": {}}, skip_timesteps=46)
    assert close(half[0], full[1], "sharding-independent x_T")


def test_plms_through_sharded_sample(plain):
    """distributed.sharded_sample dispatches by name: PLMS with its order keyword, keyed by global sample index"""
    m, _ = plain
    d = C.create_gaussian_diffusion(timestep_respacing="ddim50")
    d.engine_seed = 99
    got = C.sharded_sample(d, m, SHAPE, model_kwargs={"y": {}}, sampler="plms_sample_loop", order=3, skip_timesteps=45)
    assert d.rng == "torch" and d.sample_offset == 0  # restored
    d.rng = "engine"
    want = d.plms_sample_loop(m, SHAPE, model_kwargs={"y": {}}, order=3, skip_timesteps=45)
    assert torch.equal(got, want)


def test_plms_launch_accounting(plain, gi):
    """One PLMS call costs what a DDIM call of the same length costs plus one evaluation (the first step's second one) --
    measured on the engine's own count of the kernels it launched"""
    m, _ = plain
    eng = m.engine_for(torch.device(DEV), max_batch=B)
    d = ddim50(gi)
    x_T = gi["tape"][0].to(DEV)

    def launches(fn, skip, **kw):
        n0 = eng.launch_count
        fn(m, SHAPE, noise=x_T, model_kwargs={"y": {}}, skip_timesteps=skip, **kw)
        torch.cuda.synchronize()
        return eng.launch_count - n0

    ddim = {s: launches(d.ddim_sample_loop, s) for s in (40, 41)}
    plms = {s: launches(d.plms_sample_loop, s, order=3) for s in (40, 41)}
    per_step = ddim[40] - ddim[41]
    assert per_step > 0 and plms[40] - plms[41] == per_step
    assert plms[40] == ddim[40] + per_step
    # the generator: the same work in one call per step, plus the old_eps copies (min(k + 1, order - 1) per yield)
    n0 = eng.launch_count
    list(d.plms_sample_loop_progressive(m, SHAPE, noise=x_T, model_kwargs={"y": {}}, skip_timesteps=45, order=3))
    n_prog = eng.launch_count - n0
    n_fused = launches(d.plms_sample_loop, 45, order=3)
    setup = n_fused - 6 * per_step  # 5 steps + the extra evaluation
    # every generator call also copies out pred_xstart (+1); the 4 resuming calls skip the q_sample of init_image (-1)
    assert n_prog == 5 * setup + 5 - 4 + 6 * per_step + sum(min(k + 1, 2) for k in range(5))

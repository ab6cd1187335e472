"""GPU: the engine at the model geometries the reference builds besides HumanML3D's 263 features x 196 frames
(utils/model_util.py:62-76: 251 for KIT, 67 with drop_redundant, 764 for AMASS; sample/gmd/generate.py:110-112 asks for
fewer frames), where the input projection's K, the output head's N, the token <-> frame row maps, the UNet's padding to
224 frames and the step kernel's noise paths all run with other tile and padding arithmetic than at 263 x 196.

Expected values: tests/golden/geometries.* (outputs of the UNMODIFIED reference, oracle/make_golden_geometries.py) and the
CPU oracle on the same inputs.  Gate: rtol 1e-3 / atol 1e-4 unless a test states otherwise.
"""
import ctypes

import pytest
import torch

import condmdi_b200 as C
from oracle import condmdi_oracle as O
from oracle import make_golden_geometries as G
from oracle import plms_oracle as P
from oracle.golden_io import load_golden
from test_gpu_unet_fp16 import engine_forward as fp16_engine_forward
from test_gpu_unet_fp16 import gate as fp16_gate
from test_gpu_unet_fp16 import oracle as fp16_oracle
from test_gpu_unet_fp16 import to_dev

pytestmark = pytest.mark.gpu
GATE = dict(rtol=1e-3, atol=1e-4)
DEV = "cuda:0"
TEXTS = ["a", "b", "c", "d"]


@pytest.fixture(scope="module")
def gold(golden_dir):
    return load_golden(golden_dir, "geometries")


def close(a, b, what, **tol):
    tol = tol or GATE
    a, b = torch.as_tensor(a).cpu().double(), torch.as_tensor(b).cpu().double()
    err = (a - b).abs()
    viol = (err > tol["atol"] + tol["rtol"] * b.abs()).double().mean().item()
    print(f"[{what}] max_abs={err.max():.3e} mean_abs={err.mean():.3e} gate violations={viol:.2e}")
    return a.shape == b.shape and torch.allclose(a, b, **tol)


def with_text(m, cond):
    """encode_text of the synthetic text embeddings: text i -> cond[i]."""
    table = {s: cond[i].to(DEV) for i, s in enumerate(TEXTS[:len(cond)])}
    m.encode_text = lambda texts: torch.stack([table[s] for s in texts])
    return m


def transformer(D, text, seed=7, layers=8):
    sd = O.random_state_dict(seed=seed, feats=D, text=text, layers=layers)
    m = C.MDM(njoints=D, num_layers=layers, cond_mode="text" if text else "no_cond", cond_mask_prob=0.1)
    missing, unexpected = m.load_state_dict(sd, strict=False)
    assert not missing and not unexpected
    return m.to(DEV), sd


def unet(D, mults, kf=True, seed=11, dataset="humanml"):
    sd = O.random_unet_state_dict(seed=seed, mults=mults, feats=D, keyframe_conditioned=kf)
    m = C.MDM_UNET(njoints=D, dim_mults=mults, keyframe_conditioned=kf, dataset=dataset)
    missing, unexpected = m.load_state_dict(sd, strict=False)
    assert not missing and not unexpected
    return m.to(DEV), sd


def fixture_model(name, gi):
    c = G.CASES[name]
    if c["kind"] == "mdm":
        m, sd = transformer(c["D"], c["text"])
        if c["text"]:
            with_text(m, gi["cond"])
        return m, sd
    return unet(c["D"], c["mults"], dataset=c["dataset"])


def tail_kwargs(name, gi):
    """model_kwargs of the fixture tails (oracle/make_golden_geometries.py::reference_outputs)."""
    c, B = G.CASES[name], gi["x"].shape[0]
    xo, mask = gi["x_obs"].to(DEV), gi["mask"].to(DEV)
    y = {"mask": gi["y_mask"].to(DEV), "lengths": gi["lengths"], "imputate": 1, "stop_imputation_at": 1,
         "replacement_distribution": "conditional", "inpainted_motion": xo, "inpainting_mask": mask}
    kw = {"y": y}
    if c["kind"] == "unet":
        kw.update(obs_x0=xo, obs_mask=mask)
    elif c["text"]:
        y.update(text=TEXTS[:B], text_scale=gi["text_scale"].to(DEV))
    return kw


# ------------------------------------------------------------------------------------------------
# transformer: one denoiser evaluation
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("D,L", [(251, 120), (67, 57), (764, 207), (263, 1), (263, 121), (263, 207)])
def test_transformer_forward_plain_uncond_cfg(D, L):
    """B = 3 on an engine built for 4: per-sample timesteps for the text and unconditional passes, one shared timestep
    for the batch-doubled CFG pass (6 sequences of L + 1 tokens)."""
    m, sd = transformer(D, text=True)
    eng = m.engine_for(DEV, max_batch=4, nframes=L)
    g = torch.Generator().manual_seed(D * 1000 + L)
    x = torch.randn(3, D, 1, L, generator=g)
    cond = torch.randn(3, 512, generator=g)
    scale = torch.tensor([2.5, 0.7, 1.3])
    with_text(m, cond)
    t = torch.tensor([999, 37, 500])
    y = {"text": TEXTS[:3]}
    got = m(x.to(DEV), t.to(DEV), y=y)
    assert got.shape == (3, D, 1, L) and m.engine_for(DEV, max_batch=3, nframes=L) is eng
    assert close(got, O.mdm_forward(sd, x, t, cond), f"{D}x{L} text")
    got = m(x.to(DEV), t.to(DEV), y=dict(y, uncond=True))
    assert close(got, O.mdm_forward(sd, x, t, cond, uncond=True), f"{D}x{L} uncond")
    t = torch.full((3,), 500)
    got = C.ClassifierFreeSampleModel(m)(x.to(DEV), t.to(DEV), y=dict(y, text_scale=scale.to(DEV)))
    assert close(got, O.cfg_forward(sd, x, t, cond, scale), f"{D}x{L} cfg")


@pytest.mark.parametrize("name", [n for n, c in G.CASES.items() if c["kind"] == "mdm"])
def test_transformer_forward_and_ddpm_tail_vs_reference_golden(gold, name):
    gi = G.case_inputs(name)
    m, _ = fixture_model(name, gi)
    c = G.CASES[name]
    x, t = gi["x"].to(DEV), gi["t"].to(DEV)
    y = {"text": TEXTS[:2]} if c["text"] else {}
    assert close(m(x, t, y=y), G.fixture(gold, f"{name}.fwd"), f"{name} forward vs reference")
    if c["text"]:
        got = C.ClassifierFreeSampleModel(m)(x, t, y=dict(y, text_scale=gi["text_scale"].to(DEV)))
        assert close(got, G.fixture(gold, f"{name}.fwd_cfg"), f"{name} cfg forward vs reference")
    d = C.create_gaussian_diffusion()
    d.noise_tape = gi["tape"].to(DEV)
    model = C.ClassifierFreeSampleModel(m) if c["text"] else m
    got = d.p_sample_loop(model, tuple(x.shape), model_kwargs=tail_kwargs(name, gi), skip_timesteps=G.SKIP,
                          init_image=gi["x_obs"].to(DEV))
    assert close(got, G.fixture(gold, f"{name}.tail"), f"{name} ddpm tail (t = 3..0, imputation) vs reference")


# ------------------------------------------------------------------------------------------------
# transformer: sampling loops
# ------------------------------------------------------------------------------------------------
def edit_case(D, L, seed):
    """Text model, seeded inputs, ~20 % observed (whole frames and single features), lengths shorter than L."""
    m, sd = transformer(D, text=True)
    g = torch.Generator().manual_seed(seed)
    B = 2
    x_obs = torch.randn(B, D, 1, L, generator=g)
    cond = torch.randn(B, 512, generator=g)
    mask = G.random_obs_mask(g, B, D, L)
    lengths = torch.tensor([L - 3, (2 * L) // 3])
    y_mask = (torch.arange(L)[None] < lengths[:, None]).view(B, 1, 1, L)
    scale = torch.tensor([2.5, 0.7])
    tape = torch.randn(6, B, D, 1, L, generator=g)
    with_text(m, cond)
    y = {"text": TEXTS[:B], "text_scale": scale.to(DEV), "mask": y_mask.to(DEV), "lengths": lengths, "imputate": 1,
         "stop_imputation_at": 1, "replacement_distribution": "conditional", "inpainted_motion": x_obs.to(DEV),
         "inpainting_mask": mask.to(DEV)}
    c = O.Conditioning(cond_emb=cond, cfg=True, text_scale=scale, y_mask=y_mask, imputate=True, stop_imputation_at=1,
                       inpainted_motion=x_obs, inpainting_mask=mask)
    return m, sd, x_obs, tape, y, c


@pytest.mark.parametrize("D,L", [(251, 120), (67, 57)])
def test_ddim50_tail_cfg_imputation_vs_oracle(D, L):
    m, sd, x_obs, tape, y, c = edit_case(D, L, seed=D + L)
    tape = tape[torch.arange(51) % 6]
    d = C.create_gaussian_diffusion(timestep_respacing="ddim50")
    d.noise_tape = tape.to(DEV)
    got = d.ddim_sample_loop(C.ClassifierFreeSampleModel(m), (2, D, 1, L), model_kwargs={"y": y}, skip_timesteps=40,
                             init_image=x_obs.to(DEV))
    want = O.sample_loop(sd, O.make_tables("ddim50"), (2, D, 1, L), c, tape, "ddim", skip_timesteps=40, init_image=x_obs)
    assert close(got, want, f"{D}x{L} ddim50 tail t = 9..0, cfg + imputation")


def test_reconstruction_guided_steps_at_kit_geometry():
    """10 guided steps (w = 20) from t = 49 at 251 x 120: the input-VJP (backward.cu, attention_bwd_tc.cu) at S = 121 and
    K = D_pad = 256, in the contracting regime test_guided_50_step_tail_vs_reference_golden holds to the gate."""
    D, L = 251, 120
    m, sd, x_obs, tape, y, c = edit_case(D, L, seed=99)
    tape = tape[torch.arange(51) % 6]
    y = dict(y, reconstruction_guidance=True, reconstruction_weight=20.0, gradient_schedule=None, diffusion_steps=1000,
             stop_recguidance_at=0)
    c.reconstruction_guidance, c.reconstruction_weight = True, 20.0
    d = C.create_gaussian_diffusion()
    d.noise_tape = tape.to(DEV)
    outs = []
    for k, o in enumerate(d.p_sample_loop_progressive(C.ClassifierFreeSampleModel(m), (2, D, 1, L), model_kwargs={"y": y},
                                                      skip_timesteps=950, init_image=x_obs.to(DEV))):
        outs.append(o["sample"].clone())
        if k == 9:
            break
    want = O.sample_loop(sd, O.make_tables(""), (2, D, 1, L), c, tape, "ddpm", skip_timesteps=950, init_image=x_obs,
                         max_steps=10)
    assert close(outs[-1], want, "251x120 guided steps t = 49..40")


def test_plms_order2_at_drop_redundant_geometry():
    D, L = 67, 57
    m, sd, x_obs, tape, y, c = edit_case(D, L, seed=5)
    d = C.create_gaussian_diffusion(timestep_respacing="ddim50")
    d.noise_tape = tape.to(DEV)
    got = d.plms_sample_loop(C.ClassifierFreeSampleModel(m), (2, D, 1, L), model_kwargs={"y": y}, skip_timesteps=40,
                             init_image=x_obs.to(DEV), order=2)
    want = P.plms_sample_loop(sd, O.make_tables("ddim50"), (2, D, 1, L), c, tape, order=2, skip_timesteps=40, init_image=x_obs)
    assert close(got, want, "67x57 plms order 2, t = 9..0, cfg + imputation")


# ------------------------------------------------------------------------------------------------
# MDM_UNET, bf16x3
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", [n for n, c in G.CASES.items() if c["kind"] == "unet"])
def test_unet_forward_and_ddpm_tail_vs_reference_golden(gold, name):
    gi = G.case_inputs(name)
    m, _ = fixture_model(name, gi)
    x, xo, mask = gi["x"].to(DEV), gi["x_obs"].to(DEV), gi["mask"].to(DEV)
    got = m(x, gi["t"].to(DEV), y={}, obs_x0=xo, obs_mask=mask)
    assert close(got, G.fixture(gold, f"{name}.fwd"), f"{name} forward vs reference")
    d = C.create_gaussian_diffusion()
    d.noise_tape = gi["tape"].to(DEV)
    got = d.p_sample_loop(m, tuple(x.shape), model_kwargs=tail_kwargs(name, gi), skip_timesteps=G.SKIP, init_image=xo)
    assert close(got, G.fixture(gold, f"{name}.tail"), f"{name} ddpm tail (t = 3..0, keyframes + imputation) vs reference")


def test_unet_amass_ddim_tail_imputation_vs_oracle():
    name = "unet.764x120"
    gi = G.case_inputs(name)
    m, sd = fixture_model(name, gi)
    D, L = G.CASES[name]["D"], G.CASES[name]["L"]
    tape = gi["tape"][torch.arange(51) % len(gi["tape"])]
    d = C.create_gaussian_diffusion(timestep_respacing="ddim50")
    d.noise_tape = tape.to(DEV)
    got = d.ddim_sample_loop(m, (2, D, 1, L), model_kwargs=tail_kwargs(name, gi), skip_timesteps=45, init_image=gi["x_obs"].to(DEV))
    want = O.sample_loop(sd, O.make_tables("ddim50"), (2, D, 1, L), G.case_conditioning(name, gi), tape, "ddim",
                         skip_timesteps=45, init_image=gi["x_obs"])
    assert close(got, want, "unet 764x120 ddim50 tail t = 4..0, keyframes + imputation")


def test_unet_unconditioned_kit_geometry():
    """A 2-level UNet without keyframe input conditioning at 251 x 196 (KIT): forward at per-sample timesteps and a DDPM
    tail against the oracle."""
    D, L = 251, 196
    m, sd = unet(D, (1, 1), kf=False, seed=3)
    g = torch.Generator().manual_seed(251)
    x = torch.randn(2, D, 1, L, generator=g)
    tape = torch.randn(5, 2, D, 1, L, generator=g)
    t = torch.tensor([999, 37])
    assert close(m(x.to(DEV), t.to(DEV), y={}), O.unet_forward(sd, x, t), "unet 251x196 no keyframes, forward")
    d = C.create_gaussian_diffusion()
    d.noise_tape = tape.to(DEV)
    got = d.p_sample_loop(m, (2, D, 1, L), model_kwargs={"y": {}}, skip_timesteps=G.SKIP, init_image=x.to(DEV))
    want = O.sample_loop(sd, O.make_tables(""), (2, D, 1, L), O.Conditioning(), tape, "ddpm", skip_timesteps=G.SKIP, init_image=x)
    assert close(got, want, "unet 251x196 no keyframes, ddpm tail")


# ------------------------------------------------------------------------------------------------
# MDM_UNET, fp16 autocast precision: the gate of tests/test_gpu_unet_fp16.py
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["unet.263x120", "unet.764x120"])
def test_fp16_unet_forward(name):
    gi = G.case_inputs(name)
    m, sd = fixture_model(name, gi)
    x, t, xo, kf = gi["x"], gi["t"], gi["x_obs"], gi["mask"]
    got = fp16_engine_forward(m, x, t, xo=xo, kf=kf)
    sdd = to_dev(sd)
    fp16_gate(got, fp16_oracle(sdd, x, t, xo=xo, kf=kf), fp16_oracle(sdd, x, t, xo=xo, kf=kf, autocast=False), f"fp16 {name}")


# ------------------------------------------------------------------------------------------------
# the step kernel's noise: engine generator (quad path when L % 4 == 0, scalar path otherwise) and torch's stream
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("D,L", [(251, 57), (263, 196)])
def test_engine_noise_is_the_counter_based_stream(D, L):
    """A DDPM step at t = 998 (sigma ~ 1): the noise recovered in float64 from (x_t, pred_xstart, x_{t-1}) is
    cmdi_test_normal(seed, stream_id = t + 1, sample_offset) over the D * L elements of each sample."""
    m, _ = transformer(D, text=False, layers=2)
    d = C.create_gaussian_diffusion()
    d.rng, d.engine_seed = "engine", 4321
    outs = []
    for k, o in enumerate(d.p_sample_loop_progressive(m, (2, D, 1, L), model_kwargs={"y": {}})):
        outs.append({key: v.clone() for key, v in o.items()})
        if k == 1:
            break
    t = 998
    f32 = lambda a: float(torch.tensor(a[t]).float())  # noqa: E731  (the fp32 table entries the step uses)
    c1, c2 = f32(d.posterior_mean_coef1), f32(d.posterior_mean_coef2)
    sigma = float(torch.exp(0.5 * torch.tensor(d.posterior_log_variance_clipped[t]).float()))
    assert sigma > 0.5
    x_t, x_next, x0 = outs[0]["sample"].double(), outs[1]["sample"].double(), outs[1]["pred_xstart"].double()
    noise = (x_next - c1 * x0 - c2 * x_t) / sigma
    want = torch.empty(2, D * L, device=DEV)
    lib = C.capi.load()
    C.capi.check(lib.cmdi_test_normal(ctypes.c_void_p(want.data_ptr()), 2, D * L, 4321, t + 1, 0, None))
    torch.cuda.synchronize()
    err = (noise.reshape(2, -1) - want.double()).abs()
    print(f"[{D}x{L} engine noise at t={t}] max_abs={err.max():.3e} mean_abs={err.mean():.3e}")
    assert err.max() < 1e-4


def test_engine_rng_shards_reproduce_the_unsharded_batch_at_251x57():
    m, _ = transformer(251, text=False, layers=2)
    shape = (4, 251, 1, 57)
    d = C.create_gaussian_diffusion(timestep_respacing="ddim50")
    d.rng, d.engine_seed = "engine", 1234
    full = d.ddim_sample_loop(m, shape, model_kwargs={"y": {}}, skip_timesteps=46, eta=1.0).clone()
    parts = []
    for lo in (0, 2):
        d.sample_offset = lo
        parts.append(d.ddim_sample_loop(m, (2,) + shape[1:], model_kwargs={"y": {}}, skip_timesteps=46, eta=1.0).clone())
    d.sample_offset = 0
    assert torch.equal(full, torch.cat(parts))
    assert not torch.equal(parts[0], parts[1])


def test_torch_stream_noise_when_numel_is_not_a_multiple_of_4():
    """rng='torch' at 251 x 57 (B * D * L = 28614): the loop draws what randn(*shape) and one randn_like per step draw."""
    from condmdi_b200.diffusion import _cuda_rng_state
    m, _ = transformer(251, text=False, layers=2)
    shape, skip = (2, 251, 1, 57), 995
    assert (2 * 251 * 57) % 4 != 0
    d = C.create_gaussian_diffusion()
    assert d.rng == "torch"
    torch.manual_seed(17)
    tape = torch.stack([torch.randn(*shape, device=DEV) for _ in range(1 + 1000 - skip)])
    state_after = _cuda_rng_state(torch.device(DEV))
    d.noise_tape = tape
    want = d.p_sample_loop(m, shape, model_kwargs={"y": {}}, skip_timesteps=skip)
    d.noise_tape = None
    torch.manual_seed(17)
    got = d.p_sample_loop(m, shape, model_kwargs={"y": {}}, skip_timesteps=skip)
    assert torch.equal(got, want)
    assert _cuda_rng_state(torch.device(DEV)) == state_after
    torch.manual_seed(17)
    last = None
    for last in d.p_sample_loop_progressive(m, shape, model_kwargs={"y": {}}, skip_timesteps=skip):
        pass
    assert torch.equal(last["sample"], want)


# ------------------------------------------------------------------------------------------------
# limits
# ------------------------------------------------------------------------------------------------
def test_unet_at_224_frames_builds_and_keeps_its_shape():
    m, _ = unet(263, (1, 1))
    x = torch.randn(2, 263, 1, 224, device=DEV)
    mask = torch.zeros(2, 263, 1, 224, dtype=torch.bool, device=DEV)
    out = m(x, torch.tensor([10, 10], device=DEV), y={}, obs_x0=x, obs_mask=mask)
    assert out.shape == (2, 263, 1, 224) and torch.isfinite(out).all()


@pytest.mark.parametrize("arch,D,L,match", [("mdm", 263, 208, r"nframes <= 207"), ("unet", 263, 225, r"nframes <= 224"),
                                            ("mdm", 4, 60, r"njoints >= 8"), ("unet", 4, 60, r"njoints >= 8")])
def test_unsupported_geometries_are_refused_at_creation(arch, D, L, match):
    """The reference's traj_only models (njoints = 4) and sequences past the engine's limits: an error that names the
    limit, never numbers."""
    m = C.MDM(njoints=D, num_layers=2) if arch == "mdm" else C.MDM_UNET(njoints=D, dim_mults=(1, 1))
    m = m.to(DEV)
    x = torch.randn(2, D, 1, L, device=DEV)
    with pytest.raises(RuntimeError, match=match):
        m(x, torch.tensor([10, 10], device=DEV), y={})

"""GPU: loop-level parity where round 1 had none (VERDICT r01, "Parity gaps"):

  * whole DDIM-100 loop (BASELINE configs[4]) against the reference's own output          (tests/golden/chains.npz)
  * the last 50 steps (t = 49..0) of configs[2] (CFG + imputation) and configs[3] (CFG + imputation + reconstruction
    guidance w = 20) against the reference -- the regime where sqrt(alpha_bar_t) ~ 1 and guidance acts at full strength
  * B = 64 (the BASELINE shape) loops against the CPU oracle: DDIM-50 (configs[0] sampler at the configs[4] batch), a
    20-step DDPM tail (configs[1]) and a CFG + imputation tail (configs[2])
  * the drop-in boundary exercised on this box: a denoiser assembled from STOCK torch.nn modules under the reference's
    state-dict keys, wrapped by a class named like the reference's CFG wrapper, and a diffusion object carrying the
    reference's attributes, pushed through `accelerate()` / `resolve_model`

Gate: rtol 1e-3 / atol 1e-4 (BASELINE north_star) unless a test states otherwise and why.
"""
import os

import numpy as np
import pytest
import torch

import condmdi_b200 as C
from oracle import condmdi_oracle as O
from oracle.golden_io import load_golden

pytestmark = pytest.mark.gpu
GATE = dict(rtol=1e-3, atol=1e-4)
B, D, L = 2, 263, 196
DEV = "cuda:0"


@pytest.fixture(scope="module")
def chains(golden_dir):
    return load_golden(golden_dir, "chains")


@pytest.fixture(scope="module")
def gi():
    return O.golden_inputs()


def _model(text, seed=7):
    sd = O.random_state_dict(seed=seed, text=text)
    m = C.MDM(cond_mode="text" if text else "no_cond", cond_mask_prob=0.1)
    missing, unexpected = m.load_state_dict(sd, strict=False)
    assert not missing and not unexpected
    return m.cuda(), sd


@pytest.fixture(scope="module")
def plain():
    return _model(False)


@pytest.fixture(scope="module")
def texty(gi):
    m, sd = _model(True)
    m.encode_text = lambda texts: gi["cond"].to(DEV)
    return m, sd


def report(a, b, what=""):
    a, b = torch.as_tensor(a).cpu().double(), torch.as_tensor(b).cpu().double()
    err = (a - b).abs()
    viol = (err > GATE["atol"] + GATE["rtol"] * b.abs()).double().mean().item()
    print(f"[{what}] max_abs={err.max():.3e} mean_abs={err.mean():.3e} gate violations={viol:.2e}")
    return err.max().item(), err.mean().item(), viol


def close(a, b, what="", **tol):
    tol = tol or GATE
    report(a, b, what)
    return torch.allclose(torch.as_tensor(a).cpu().float(), torch.as_tensor(b).cpu().float(), **tol)


def _edit_kwargs(gi, guided):
    x_obs, kf = gi["x_obs"].to(DEV), gi["kf_mask"].to(DEV)
    y = {"text": ["a", "b"], "text_scale": gi["text_scale"].to(DEV), "mask": gi["y_mask"].to(DEV), "lengths": gi["lengths"],
         "imputate": 1, "stop_imputation_at": 1, "replacement_distribution": "conditional", "inpainted_motion": x_obs,
         "inpainting_mask": kf}
    if guided:
        y.update(reconstruction_guidance=True, reconstruction_weight=20.0, gradient_schedule=None, diffusion_steps=1000,
                 stop_recguidance_at=0)
    return y, x_obs


# ------------------------------------------------------------------------------------------------
# reference fixtures, B = 2
# ------------------------------------------------------------------------------------------------
def test_ddim100_full_loop_vs_reference_golden(plain, gi, chains):
    """configs[4]'s sampler: `ddim_sample_loop` over the 'ddim100' respacing, all 100 steps including t = 0."""
    m, _ = plain
    d = C.create_gaussian_diffusion(timestep_respacing="ddim100")
    assert d.num_timesteps == 100 and d.timestep_map[:3] == [0, 10, 20]
    d.noise_tape = gi["tape"][torch.arange(101) % 8].to(DEV)
    got = d.ddim_sample_loop(m, (B, D, 1, L), model_kwargs={"y": {}}, clip_denoised=False)
    assert close(got, chains["ddim100.sample"], "ddim100 vs reference")


def test_cfg_imputation_50_step_tail_vs_reference_golden(texty, gi, chains):
    """configs[2]: CFG 2.5 + sparse-keyframe imputation, t = 49 .. 0 (skip_timesteps = 950, init_image = x_obs)."""
    m, _ = texty
    w = C.ClassifierFreeSampleModel(m)
    d = C.create_gaussian_diffusion()
    d.noise_tape = gi["tape"][torch.arange(51) % 8].to(DEV)
    y, x_obs = _edit_kwargs(gi, guided=False)
    got = d.p_sample_loop(w, (B, D, 1, L), model_kwargs={"y": y}, skip_timesteps=950, init_image=x_obs, clip_denoised=False)
    assert close(got, chains["cfg_impute50.sample"], "cfg+imputation 50-step tail vs reference")


def test_guided_50_step_tail_vs_reference_golden(texty, gi, chains):
    """configs[3]: CFG + imputation + reconstruction guidance (w = 20), t = 49 .. 0.

    oracle/make_golden.py::golden_chains measured what this chain is: contracting down to t ~ 10 (two fp32 implementations
    6e-6 apart after 40 steps), EXPANDING below t ~ 8 (x0_tilde = x0_hat - 10 * grad with coef1 -> 1: rounding differences
    grow ~2.5x per step; the reference ends 1.9e-3 from the float64 chain, the fp32 oracle 3.5e-3, 2e-3 from each other).
    So: (a) the state after t = 10 is held to the gate; (b) inside the expanding regime single steps restarted from the
    REFERENCE's own states are held to the gate; (c) the end state is held to the float64 chain within a stated multiple
    of the reference's own distance from it."""
    m, _ = texty
    w = C.ClassifierFreeSampleModel(m)
    d = C.create_gaussian_diffusion()
    tape = gi["tape"][torch.arange(51) % 8].to(DEV)
    d.noise_tape = tape
    y, x_obs = _edit_kwargs(gi, guided=True)
    outs = [o["sample"].clone() for o in
            d.p_sample_loop_progressive(w, (B, D, 1, L), model_kwargs={"y": y}, skip_timesteps=950, init_image=x_obs)]
    assert len(outs) == 50
    # (a) 40 guided steps, t = 49 .. 10
    assert close(outs[39], chains["recon50.sample_k39"], "guided chain after t=10")
    # the fused loop (one native call, graph replay) equals the per-step generator bit for bit
    fused = d.p_sample_loop(w, (B, D, 1, L), model_kwargs={"y": y}, skip_timesteps=950, init_image=x_obs)
    assert torch.equal(fused, outs[-1])
    # (b) single guided steps from the reference's states: k -> k+1 means the step at t = 49 - (k + 1)
    eng = m.engine_for(torch.device(DEV), max_batch=B)
    tt = torch.arange(d.num_timesteps)
    coef = (torch.from_numpy(C.get_gradient_schedule(None, 1000))[tt].float() * 20.0 *
            torch.from_numpy(d.sqrt_alphas_cumprod)[tt].float() / 2).numpy()
    for k in (44, 47, 48):
        state = torch.from_numpy(chains[f"recon50.sample_k{k}"]).to(DEV)
        res = eng.sample(B, x_T=state, resume=True, skip_timesteps=950 + k + 1, num_steps=1, noise_tape=tape[1 + k + 1:],
                         cond_emb=gi["cond"].to(DEV), cfg=True, text_scale=gi["text_scale"].to(DEV),
                         y_mask=gi["y_mask"].to(DEV).reshape(B, -1), imputate=True, stop_imputation_at=1,
                         inpainted_motion=x_obs, inpainting_mask=gi["kf_mask"].to(DEV), recon_guidance=True,
                         stop_recguidance_at=0, recon_coef=coef)
        want = chains[f"recon50.sample_k{k + 1}"]
        mx, _, viol = report(res["sample"], want, f"guided single step t={49 - (k + 1)} from the reference's state")
        if k < 47:
            assert viol == 0.0
        else:
            # t = 1 and t = 0 carry the largest guidance coefficient (w * sqrt(alpha_bar_t) / 2 ~ 10) on top of the CFG
            # scale: the bf16x3 products' 2^-17 relative error, amplified 25x, leaves a few elements in 1e5 outside the
            # gate (measured on H100: t = 1: 1, t = 0: 2 of 103 096 elements, max |err| 2.8e-4 where |x| reaches 20).
            # Documented in DESIGN.md.
            assert viol <= 2e-4 and mx <= 2e-3
    # (c) the end of the chain against the float64 chain
    ref_max, ref_mean = chains["recon50.ref_err_vs_f64"]
    got_max, got_mean, _ = report(outs[-1], chains["recon50.f64_final"], "guided chain end vs float64 chain")
    print(f"reference (fp32) vs float64 chain: max {ref_max:.3e} mean {ref_mean:.3e}; engine/reference: max x{got_max / ref_max:.1f} mean x{got_mean / ref_mean:.1f}")
    # bf16x3 products carry ~2^-17 relative error against fp32's 2^-24: one to two orders of magnitude more per step,
    # amplified by the same expanding map.  Measured on H100: engine 9.7e-2 max / 5.3e-4 mean from the float64 chain
    # where the reference's own fp32 run is 1.9e-3 / 3.8e-5 from it (x51 / x14).
    # The end of a w = 20 guided chain is not a quantity any finite-precision implementation reproduces; what is pinned
    # is (a), (b) and this ratio.
    assert got_max <= 100 * ref_max and got_mean <= 50 * ref_mean


# ------------------------------------------------------------------------------------------------
# BASELINE batch (B = 64) loops against the CPU oracle (tens of seconds of CPU each)
# ------------------------------------------------------------------------------------------------
def _big_inputs(n_tape):
    g = torch.Generator().manual_seed(77)
    tape = torch.randn(n_tape, 64, D, 1, L, generator=g)
    return tape


def test_b64_ddim50_full_loop_vs_oracle(plain):
    m, sd = plain
    tape = _big_inputs(9)
    tape = tape[torch.arange(51) % 9]
    d = C.create_gaussian_diffusion(timestep_respacing="ddim50")
    d.noise_tape = tape.to(DEV)
    got = d.ddim_sample_loop(m, (64, D, 1, L), model_kwargs={"y": {}})
    want = O.sample_loop(sd, O.make_tables("ddim50"), (64, D, 1, L), O.Conditioning(), tape, "ddim")
    assert close(got, want, "B=64 ddim50 vs oracle")


def test_b64_ddpm_20_step_tail_vs_oracle(plain):
    """configs[1] at its own batch: the last 20 ancestral steps (t = 19 .. 0) of the 1000-step schedule."""
    m, sd = plain
    tape = _big_inputs(9)
    tape = tape[torch.arange(21) % 9]
    x0 = torch.randn(64, D, 1, L, generator=torch.Generator().manual_seed(5))
    d = C.create_gaussian_diffusion()
    d.noise_tape = tape.to(DEV)
    got = d.p_sample_loop(m, (64, D, 1, L), model_kwargs={"y": {}}, skip_timesteps=980, init_image=x0.to(DEV))
    want = O.sample_loop(sd, O.make_tables(""), (64, D, 1, L), O.Conditioning(), tape, "ddpm", skip_timesteps=980, init_image=x0)
    assert close(got, want, "B=64 ddpm 20-step tail vs oracle")


def test_b64_cfg_imputation_tail_vs_oracle(texty):
    """configs[2] at B = 64: CFG 2.5 + benchmark_sparse imputation with ragged lengths, t = 9 .. 0."""
    m, sd = texty
    Bf = 64
    g = torch.Generator().manual_seed(4)
    cond = torch.randn(Bf, 512, generator=g)
    x_obs = torch.randn(Bf, D, 1, L, generator=g)
    lengths = torch.randint(20, 197, (Bf,), generator=g)
    kf = C.get_keyframes_mask(x_obs, lengths, "benchmark_sparse", trans_length=5)
    y_mask = (torch.arange(L)[None] < lengths[:, None]).view(Bf, 1, 1, L)
    scale = torch.full((Bf,), 2.5)
    tape = _big_inputs(9)[torch.arange(11) % 9]
    enc = m.encode_text
    m.encode_text = lambda texts: cond.to(DEV)
    try:
        d = C.create_gaussian_diffusion()
        d.noise_tape = tape.to(DEV)
        y = {"text": [""] * Bf, "text_scale": scale.to(DEV), "mask": y_mask.to(DEV), "imputate": 1, "stop_imputation_at": 1,
             "replacement_distribution": "conditional", "inpainted_motion": x_obs.to(DEV), "inpainting_mask": kf.to(DEV)}
        got = d.p_sample_loop(C.ClassifierFreeSampleModel(m), (Bf, D, 1, L), model_kwargs={"y": y}, skip_timesteps=990,
                              init_image=x_obs.to(DEV))
    finally:
        m.encode_text = enc
    c = O.Conditioning(cond_emb=cond, cfg=True, text_scale=scale, y_mask=y_mask, imputate=True, stop_imputation_at=1,
                       inpainted_motion=x_obs, inpainting_mask=kf)
    want = O.sample_loop(sd, O.make_tables(""), (Bf, D, 1, L), c, tape, "ddpm", skip_timesteps=990, init_image=x_obs)
    assert close(got, want, "B=64 cfg+imputation tail vs oracle")


# ------------------------------------------------------------------------------------------------
# drop-in under objects this package has never seen (runs on the GPU box: no /root/reference needed)
# ------------------------------------------------------------------------------------------------
def test_drop_in_under_stock_torch_modules(gi):
    from standin import ClassifierFreeSampleModel as StockCFG
    from standin import StockDiffusion, StockMDM

    torch.manual_seed(11)
    stock = StockMDM(text=True)
    with torch.no_grad():  # default init leaves LayerNorm at (1, 0): move it so gamma / beta matter
        for n_, p_ in stock.named_parameters():
            if ".norm" in n_:
                p_.add_(0.1 * torch.randn_like(p_))
    stock = stock.to(DEV).eval()
    cond = gi["cond"].to(DEV)
    stock.text_emb = cond
    ref_keys = set(O.random_state_dict(seed=0, text=True).keys())
    assert set(stock.state_dict().keys()) == ref_keys  # the reference's key set (SURVEY 8 a-W)

    # one denoiser evaluation: the engine (through resolve_model's duck-typing) against stock PyTorch on the same GPU
    inner, is_cfg = C.resolve_model(StockCFG(stock))
    assert is_cfg and inner is stock
    x = gi["x"].to(DEV)
    t = torch.tensor([300, 300], device=DEV)
    eng = inner.engine_for(torch.device(DEV), max_batch=B)
    got = eng.forward(x, 300, cond_emb=cond, cfg=True, text_scale=gi["text_scale"].to(DEV))
    prev = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    try:
        with torch.no_grad():
            want = StockCFG(stock)(x, t, y={"text": ["a", "b"], "text_scale": gi["text_scale"].to(DEV)})
    finally:
        torch.backends.cuda.matmul.allow_tf32 = prev
    assert close(got, want, "engine vs stock nn.TransformerEncoder (eager fp32, same GPU)")

    # the whole loop through accelerate(): a diffusion object carrying the reference's attributes, the stock model in
    # the reference-named CFG wrapper, keyframe imputation on; expected values from the CPU oracle on the same weights
    base = C.create_gaussian_diffusion(timestep_respacing="ddim50")
    fast = C.accelerate(StockDiffusion(base.betas, base.timestep_map))
    assert fast is not base and fast.num_timesteps == 50 and list(fast.timestep_map) == list(base.timestep_map)
    tape = gi["tape"][torch.arange(51) % 8]
    fast.noise_tape = tape.to(DEV)
    x_obs, kf = gi["x_obs"].to(DEV), gi["kf_mask"].to(DEV)
    y = {"text": ["a", "b"], "text_scale": gi["text_scale"].to(DEV), "mask": gi["y_mask"].to(DEV), "imputate": 1,
         "stop_imputation_at": 1, "replacement_distribution": "conditional", "inpainted_motion": x_obs, "inpainting_mask": kf}
    got = fast.ddim_sample_loop(StockCFG(stock), (B, D, 1, L), model_kwargs={"y": y, "obs_x0": x_obs, "obs_mask": kf})
    sd = {k: v.detach().cpu() for k, v in stock.state_dict().items()}
    c = O.Conditioning(cond_emb=gi["cond"], cfg=True, text_scale=gi["text_scale"], y_mask=gi["y_mask"], imputate=True,
                       stop_imputation_at=1, inpainted_motion=gi["x_obs"], inpainting_mask=gi["kf_mask"])
    want = O.sample_loop(sd, O.make_tables("ddim50"), (B, D, 1, L), c, tape, "ddim")
    assert close(got, want, "accelerate(stock diffusion) + stock CFG-wrapped model, ddim50 loop")


# ------------------------------------------------------------------------------------------------
# sharding: x_T belongs to the global sample, not to the rank (ADVICE r01)
# ------------------------------------------------------------------------------------------------
def test_engine_rng_shards_reproduce_the_unsharded_batch_including_x_T(plain):
    """`sharded_sample` runs each rank with rng='engine', sample_offset = first global row, noise=None.  Emulated here on
    one GPU: the two halves of a batch, run as ranks 0 and 1 of a 2-way job would run them, reproduce the 1-way batch."""
    m, _ = plain
    d = C.create_gaussian_diffusion(timestep_respacing="ddim50")
    d.rng, d.engine_seed = "engine", 1234
    full = d.ddim_sample_loop(m, (4, D, 1, L), model_kwargs={"y": {}}, skip_timesteps=46, eta=1.0).clone()
    parts = []
    for lo in (0, 2):
        d.sample_offset = lo
        parts.append(d.ddim_sample_loop(m, (2, D, 1, L), model_kwargs={"y": {}}, skip_timesteps=46, eta=1.0).clone())
    d.sample_offset = 0
    assert torch.equal(full, torch.cat(parts))
    assert not torch.equal(parts[0], parts[1])  # ranks do not repeat each other's samples
    # and through sharded_sample itself at world size 1 (seed drawn from torch's CPU generator)
    d.engine_seed = None
    torch.manual_seed(3)
    a = C.sharded_sample(d, m, (4, D, 1, L), {"y": {}}, sampler="ddim_sample_loop", skip_timesteps=46, eta=1.0).clone()
    torch.manual_seed(3)
    b = C.sharded_sample(d, m, (4, D, 1, L), {"y": {}}, sampler="ddim_sample_loop", skip_timesteps=46, eta=1.0).clone()
    assert torch.equal(a, b) and d.engine_seed is None and d.rng == "engine"


def test_dump_steps_duplicates_and_out_of_range_entries(plain, gi):
    """gaussian_diffusion.py:1208-1213 appends once per matching iteration: duplicates collapse, absent steps vanish."""
    m, _ = plain
    d = C.create_gaussian_diffusion()
    d.noise_tape = gi["tape"].to(DEV)
    dump = d.p_sample_loop(m, (B, D, 1, L), model_kwargs={"y": {}}, skip_timesteps=996, dump_steps=[2, 0, 2, 7, 100])
    ref = list(d.p_sample_loop_progressive(m, (B, D, 1, L), model_kwargs={"y": {}}, skip_timesteps=996))
    assert len(dump) == 2 and torch.equal(dump[0], ref[0]["pred_xstart"]) and torch.equal(dump[1], ref[2]["pred_xstart"])


def test_cfg_wrapper_with_uncond_flag_runs_both_passes_unconditional(texty, gi):
    """cfg_sampler.py:28-33 deep-copies y and sets uncond on the copy: a caller-set y['uncond'] makes both passes uncond."""
    m, sd = texty
    x = gi["x"].to(DEV)
    t = torch.tensor([500, 500], device=DEV)
    w = C.ClassifierFreeSampleModel(m)
    got = w(x, t, y={"text": ["a", "b"], "text_scale": gi["text_scale"].to(DEV), "uncond": True})
    want = m(x, t, y={"text": ["a", "b"], "uncond": True})
    assert close(got, want, "cfg(uncond) == uncond", rtol=1e-6, atol=1e-6)


def test_guidance_imputes_without_reading_replacement_distribution(texty, gi):
    """gaussian_diffusion.py:405-425: the guided branch imputes whenever requires_imputation() holds; the key
    'replacement_distribution' is only read by the un-guided branch (:427-442)."""
    m, sd = texty
    d = C.create_gaussian_diffusion()
    d.noise_tape = gi["tape"].to(DEV)
    y, x_obs = _edit_kwargs(gi, guided=True)
    a = d.p_sample_loop(m, (B, D, 1, L), model_kwargs={"y": y}, skip_timesteps=997, init_image=x_obs)
    y2 = dict(y)
    del y2["replacement_distribution"]
    b = d.p_sample_loop(m, (B, D, 1, L), model_kwargs={"y": y2}, skip_timesteps=997, init_image=x_obs)
    y3 = dict(y, replacement_distribution="marginal")
    c = d.p_sample_loop(m, (B, D, 1, L), model_kwargs={"y": y3}, skip_timesteps=997, init_image=x_obs)
    assert torch.equal(a, b) and torch.equal(a, c)


def test_engine_knobs_are_per_engine_state(monkeypatch, gi):
    """An engine keeps the configuration it was created under; creating another one under different settings does not
    change it (round 1 kept some of these switches in process globals).  CMDI_CHAIN=0 selects the unchained forward path
    (one launch per linear layer + LayerNorm kernels): 59 launches per pass instead of 19."""
    sd = O.random_state_dict(seed=7)
    x = gi["x"].to(DEV)
    want = O.mdm_forward(sd, gi["x"], torch.tensor([41, 41]))

    def make():
        m = C.MDM()
        m.load_state_dict(sd, strict=False)
        return m.cuda()

    monkeypatch.setenv("CMDI_CHAIN", "0")
    m_plain = make()
    e_plain = m_plain.engine_for(torch.device(DEV), max_batch=B)
    monkeypatch.delenv("CMDI_CHAIN")
    m_chain = make()
    e_chain = m_chain.engine_for(torch.device(DEV), max_batch=B)   # created AFTER, under the default settings

    def launches(eng):
        n0 = eng.launch_count
        out = eng.forward(x, 41)
        return eng.launch_count - n0, out

    launches(e_plain), launches(e_chain)   # the first call of an engine also tabulates the timestep embedding
    n_plain, out_plain = launches(e_plain)
    n_chain, out_chain = launches(e_chain)
    n_plain2, _ = launches(e_plain)
    assert n_plain == n_plain2 == 2 + 7 * 8 + 1 + 4 and n_chain == 3 + 2 * 8 + 4
    assert close(out_plain, want, "unchained path vs oracle") and close(out_chain, want, "chained path vs oracle")
    assert not torch.equal(out_plain, out_chain)  # different arithmetic order (LayerNorm folded) -- both within the gate


# ------------------------------------------------------------------------------------------------
# evaluation-loop caller (SURVEY 8f-3) and the generator loops through the step graph
# ------------------------------------------------------------------------------------------------
def test_eval_loop_jobs_on_the_engine(texty, gi):
    """`run_eval_jobs` (the reference's double loop of comp_v6_model_dataset_condmdi.py:190-356 as a job list): merged
    engine batches give bit-identical motions to one call per job, and rng='torch' reproduces a fixseed + direct call."""
    m, _ = texty
    w = C.ClassifierFreeSampleModel(m)
    d = C.create_gaussian_diffusion()
    conds = [torch.randn(B, 512, generator=torch.Generator().manual_seed(40 + i)).to(DEV) for i in range(3)]
    state = {"i": 0}
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
        assert len(jobs) == 4
        one = C.run_eval_jobs(d, w, jobs, seed=5, merge=1, skip_timesteps=996)
        two = C.run_eval_jobs(d, w, jobs, seed=5, merge=2, skip_timesteps=996)
        four = C.run_eval_jobs(d, w, jobs, seed=5, merge=4, skip_timesteps=996)
        for i in range(4):
            assert one[i].shape == (B, D, 1, L) and torch.equal(one[i], two[i]) and torch.equal(one[i], four[i])
        assert not torch.equal(one[2], one[3])        # the two repetitions of the multimodality batch differ (other motions)
        # the reference's own seeding, call by call
        ref_style = C.run_eval_jobs(d, w, jobs, rng="torch", skip_timesteps=996)
        torch.manual_seed(jobs[1].seed_number)
        direct = d.p_sample_loop(w, (B, D, 1, L), clip_denoised=False, model_kwargs=jobs[1].model_kwargs, skip_timesteps=996)
        assert torch.equal(ref_style[1], direct) and d.rng == "torch"
    finally:
        m.encode_text = old
    del state


def test_progressive_loops_replay_the_step_graph(plain):
    """One native call per step (the generator loops): every call replays the same captured step graph -- the first step
    index of a call lives in device memory, so neither skip_timesteps nor the step number re-captures."""
    m, _ = plain
    d = C.create_gaussian_diffusion(timestep_respacing="ddim50")
    d.rng, d.engine_seed = "engine", 77
    eng = m.engine_for(torch.device(DEV), max_batch=B)
    fused = d.ddim_sample_loop(m, (B, D, 1, L), model_kwargs={"y": {}}, skip_timesteps=40, eta=1.0).clone()
    n0 = eng.launch_count
    outs = list(d.ddim_sample_loop_progressive(m, (B, D, 1, L), model_kwargs={"y": {}}, skip_timesteps=40, eta=1.0))
    assert len(outs) == 10 and torch.equal(outs[-1]["sample"], fused)
    other = list(d.ddim_sample_loop_progressive(m, (B, D, 1, L), model_kwargs={"y": {}}, skip_timesteps=45, eta=1.0))
    assert len(other) == 5 and torch.isfinite(other[-1]["sample"]).all()
    assert eng.launch_count > n0

"""GPU: reconstruction guidance on the MDM transformer -- the input-VJP (engine.cu run_backward after the stashing,
unchained guided pass) and guided sampling loops, against fp64 autograd.

  F = tests/test_gpu_bf16.py's fp64 model of MDM on the fp32 weights, differentiated by autograd
  A = the same with both operands of every product of the forward AND of the backward rounded to bf16 (one bf16 MMA per
      product, everything else exact)
  E = the engine: Engine.test_input_vjp, the pass gradients (cond pass first, seeded with s G and G - s G)

Gates per pass gradient, in max and in mean of the absolute difference; every ratio is printed:
  PRECISION_BF16   |E - F| <= 2 |A - F|     (the contract of DESIGN.md section 3)
  bf16x3           |E - F| <= 0.02 |A - F|  bf16x3 products carry ~2^-17 relative error (2^-16 for attention's truncated
                                            split) against bf16's 2^-9; measured on H100: 0.001-0.003 in max, 0.002 in
                                            mean.  One dgrad product run with one MMA, or reading a stale lo plane, moves
                                            the gradient by 0.03 |A - F| in max and 0.07 in mean
                                            (test_gpu_bf16.py::test_bf16x3_vjp_gate_catches_one_dgrad_product_at_one_mma).
Exact zeros that a ratio can average away: a sample whose inpainting mask is empty has a gradient of 0 in every pass;
under CFG a sample with text_scale 0 has a cond-pass gradient of 0, one with text_scale 1 an uncond-pass gradient of 0
((1 - s) G is 0 in fp32).  A row that leaks across sequences or an M-tail row written from the wrong tile breaks them.
"""
import pytest
import torch

import condmdi_b200 as C
import test_gpu_bf16 as TB
import test_gpu_unet_guidance as TG
from oracle import condmdi_oracle as O

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
PRECISIONS = {"bf16x3": C.PRECISION_BF16X3, "bf16": C.PRECISION_BF16}
GATES = {"bf16x3": TB.BF16X3_VJP_GATE, "bf16": 2.0}
TIMESTEPS = (999, 500, 30, 0)
MDM_FORWARD = O.mdm_forward

# name: D, L, B, text model, mode
VJP_CASES = {
    "text": (263, 196, 2, True, "text"),
    "uncond": (263, 196, 2, True, "uncond"),
    "cfg": (263, 196, 2, True, "cfg"),
    "cfg-B64": (263, 196, 64, True, "cfg"),         # 128 sequences, 25 216 rows: the largest attention-backward and dgrad grids
    "no_cond": (263, 196, 2, False, "plain"),
    "text-B3": (263, 196, 3, True, "text"),         # 591 rows: the last M tile is partly tail (and belongs to sample 2)
    "251x120-cfg": (251, 120, 2, True, "cfg"),
    "67x57-cfg": (67, 57, 2, True, "cfg"),
    "263x1-cfg": (263, 1, 2, True, "cfg"),          # S = 2
    "263x207-cfg": (263, 207, 2, True, "cfg"),      # S = 208: every key row of the pad is a token
}


def vjp_case_inputs(D, L, B, seed):
    """x, x_obs, the inpainting mask (sparse keyframes at 263 x 196, Bernoulli elsewhere), text embeddings, per-sample
    scales.  From B = 3 on, the last sample observes nothing; at B = 64 sample 0 has scale 0 and sample 1 scale 1."""
    x, xo, mask, cond, scale = TB.vjp_inputs(B, D, L, seed)
    if (D, L) == (263, 196):
        lengths = torch.randint(40, L + 1, (B,), generator=torch.Generator().manual_seed(seed + 1))
        mask = O.get_keyframes_mask(xo, lengths, "benchmark_sparse", trans_length=5)
    if B >= 3:
        mask[-1] = False
    if B >= 64:
        scale[0], scale[1] = 0.0, 1.0
    return x, xo, mask, cond, scale


def oracle_vjps(sd, x, t, xo, M, **kw):
    """(A, F): the pass gradients of the fp64 model on the GPU with q = bf16r and with q = exact"""
    sdd = {k: v.to(DEV).double() for k, v in sd.items()}
    tt = torch.full((x.shape[0],), int(t))
    return [TB.pass_vjps(lambda z, t_, c, u, q=q: TB.mdm_model(q, sdd, z, t_, c, u), x.to(DEV), tt, xo, M, **kw).cpu()
            for q in (TB.bf16r, TB.exact)]


def check_exact_zeros(got, M, scale, what):
    """got: (passes, B, ...) from the engine"""
    got = got.cpu()
    for b in range(got.shape[1]):
        if not M[b].any():
            assert (got[:, b] == 0).all(), f"{what}: sample {b} observes nothing but has a gradient"
    if got.shape[0] == 2:
        for b in range(got.shape[1]):
            if scale[b] == 0:
                assert (got[0, b] == 0).all(), f"{what}: sample {b} has text_scale 0 but a cond-pass gradient"
            if scale[b] == 1:
                assert (got[1, b] == 0).all(), f"{what}: sample {b} has text_scale 1 but an uncond-pass gradient"


@pytest.mark.parametrize("name", list(VJP_CASES))
def test_input_vjp(name):
    D, L, B, text, mode = VJP_CASES[name]
    m, sd = TB.module(D, text=text)
    x, xo, M, cond, scale = vjp_case_inputs(D, L, B, seed=B * 1000 + D + L)
    kw = {}
    if text:
        kw["cond_emb"] = cond
    if mode == "uncond":
        kw["uncond"] = True
    if mode == "cfg":
        kw["scale"] = scale
    engines = {p: m.engine_for(DEV, max_batch=B, precision=PRECISIONS[p], nframes=L) for p in PRECISIONS}
    failures = []
    for t in TIMESTEPS:
        a, f = oracle_vjps(sd, x, t, xo, M, **kw)
        for p, eng in engines.items():
            got = eng.test_input_vjp(x, t, xo, M, cond_emb=kw.get("cond_emb"), uncond=kw.get("uncond", False),
                                     cfg=mode == "cfg", text_scale=scale if mode == "cfg" else None)
            assert got.shape == a.shape
            check_exact_zeros(got, M, scale, f"{name} {p} t={t}")
            for k, which in enumerate(["cond", "uncond"][: got.shape[0]]):
                what = f"vjp {p} {name} B={B} {D}x{L} t={t} {which} pass"
                e_f = (got[k].cpu().double() - f[k]).abs().max().item()
                print(f"[{what}] max|E-F|={e_f:.3e} max|F|={f[k].abs().max().item():.3e}")
                try:
                    TB.gate(got[k], a[k], f[k], what, c=GATES[p])
                except AssertionError as err:
                    failures.append(str(err))
    assert not failures, failures


@pytest.mark.parametrize("prec", list(PRECISIONS))
def test_input_vjp_does_not_depend_on_the_calls_before_it(prec):
    """Every plane the guided pass and its backward read was written by the same call: a VJP after a chained forward, a
    B = 64 CFG VJP and a guided sampling step equals the first one on that engine and one on a fresh engine, bit for bit."""
    m, sd = TB.module()
    eng = m.engine_for(DEV, max_batch=64, precision=PRECISIONS[prec], nframes=196)
    x1, xo1, M1, cond1, scale1 = vjp_case_inputs(263, 196, 2, seed=1)
    x64, xo64, M64, cond64, scale64 = vjp_case_inputs(263, 196, 64, seed=2)
    vjp1 = lambda e: e.test_input_vjp(x1, 500, xo1, M1, cond_emb=cond1, cfg=True, text_scale=scale1)  # noqa: E731
    first = vjp1(eng)
    eng.forward(x64.to(DEV) * 3, 500, cond_emb=cond64.to(DEV), cfg=True, text_scale=scale64.to(DEV))
    eng.test_input_vjp(x64, 30, xo64, M64, cond_emb=cond64, cfg=True, text_scale=scale64)
    d = C.create_gaussian_diffusion(timestep_respacing="ddim50")
    eng.set_schedule(d.betas, d.timestep_map)
    eng.sample(64, sampler=C.capi.SAMPLER_DDIM, skip_timesteps=40, num_steps=1, seed=5, cond_emb=cond64.to(DEV), cfg=True,
               text_scale=scale64.to(DEV), inpainted_motion=xo64.to(DEV), inpainting_mask=M64.to(DEV), recon_guidance=True,
               stop_recguidance_at=0, recon_coef=[10.0] * d.num_timesteps)
    again = vjp1(eng)
    alone = vjp1(TB.module()[0].engine_for(DEV, max_batch=64, precision=PRECISIONS[prec], nframes=196))
    print(f"[{prec} vjp after other calls] max |diff| = {(again - first).abs().max().item():.3e}, "
          f"fresh engine: {(alone - first).abs().max().item():.3e}")
    assert torch.equal(again, first)
    assert torch.equal(alone, first)


# ---------------------------------------------------------------------------------------------------------------------
# guided loops against the oracle with its model (and so its guidance gradient) evaluated on the GPU
# ---------------------------------------------------------------------------------------------------------------------
def oracle_loop(sd, run, exact_fp32=False):
    """run() (an oracle sampling loop) with O.mdm_forward replaced by a grad-enabled GPU model: [A, F] in fp64, or the
    oracle's own model in exact fp32 (one run)"""
    sdd = {k: v.to(DEV) for k, v in sd.items()}
    dev = lambda v: None if v is None else v.to(DEV)  # noqa: E731
    want = []
    try:
        if exact_fp32:
            O.mdm_forward = lambda sd_, x, t, cond_emb=None, uncond=False, num_heads=4: \
                MDM_FORWARD(sdd, dev(x), dev(t), dev(cond_emb), uncond).cpu()
            with TG.exact_fp32():
                return run()
        for q in (TB.bf16r, TB.exact):
            def fwd(sd_, x, t, cond_emb=None, uncond=False, num_heads=4, _q=q):
                return TB.mdm_model(_q, sdd, dev(x), dev(t), dev(cond_emb), uncond).float().cpu()
            O.mdm_forward = fwd
            want.append(run())
    finally:
        O.mdm_forward = MDM_FORWARD
    return want


def loop_case(B, seed, stop_recguidance_at):
    """the text model with its text table, and the model_kwargs / oracle Conditioning of CFG + imputation + guidance
    (w = 20: the coefficient w sqrt(alpha_bar) / 2 is ~10 at these timesteps) over ragged lengths"""
    m, sd = TB.module()
    x_obs, _, kf, cond, scale = TG.inputs(B, seed)
    g = torch.Generator().manual_seed(seed + 1)
    lengths = torch.randint(40, 197, (B,), generator=g)
    y_mask = (torch.arange(196)[None] < lengths[:, None]).view(B, 1, 1, 196)
    table = {str(i): cond[i].to(DEV) for i in range(B)}
    m.encode_text = lambda texts: torch.stack([table[s] for s in texts])
    y = {"text": [str(i) for i in range(B)], "text_scale": scale.to(DEV), "mask": y_mask.to(DEV), "imputate": 1,
         "stop_imputation_at": 1, "replacement_distribution": "conditional", "inpainted_motion": x_obs.to(DEV),
         "inpainting_mask": kf.to(DEV), "reconstruction_guidance": True, "reconstruction_weight": 20.0,
         "gradient_schedule": None, "diffusion_steps": 1000, "stop_recguidance_at": stop_recguidance_at}
    c = O.Conditioning(cond_emb=cond, cfg=True, text_scale=scale, y_mask=y_mask, imputate=True, stop_imputation_at=1,
                       inpainted_motion=x_obs, inpainting_mask=kf, reconstruction_guidance=True, reconstruction_weight=20.0,
                       stop_recguidance_at=stop_recguidance_at)
    return C.ClassifierFreeSampleModel(m), sd, x_obs, {"y": y}, c, g


def engine_steps(progressive, n):
    """the first n steps of a step generator: sample and pred_xstart of each"""
    out = []
    for o in progressive:
        out.append({"sample": o["sample"].clone(), "pred_xstart": o["pred_xstart"].clone()})
        if len(out) == n:
            break
    return out


def gate_steps(got, a, f, what):
    for k, (e, sa, sf) in enumerate(zip(got, a, f)):
        TB.gate(e["pred_xstart"], sa["pred_xstart"], sf["pred_xstart"], f"{what}: pred_xstart of step {k}")
    TB.gate(got[-1]["sample"], a[-1]["sample"], f[-1]["sample"], f"{what}: final sample")


def test_bf16_ddpm_tail_cfg_imputation_guidance_b2():
    """t = 49 .. 44, every step guided"""
    B, n = 2, 6
    w, sd, x_obs, kw, c, g = loop_case(B, seed=61, stop_recguidance_at=0)
    tape = torch.randn(1 + n, B, 263, 1, 196, generator=g)
    d = C.create_gaussian_diffusion()
    d.precision = TB.BF16
    d.noise_tape = tape.to(DEV)
    got = engine_steps(d.p_sample_loop_progressive(w, (B, 263, 1, 196), model_kwargs=kw, skip_timesteps=950,
                                                   init_image=x_obs.to(DEV)), n)
    a, f = oracle_loop(sd, lambda: O.sample_loop(sd, O.make_tables(""), (B, 263, 1, 196), c, tape, "ddpm", skip_timesteps=950,
                                                init_image=x_obs, max_steps=n, return_all=True))
    gate_steps(got, a, f, "bf16 B=2 ddpm t=49..44, cfg 2.5 + imputation + guidance w=20")


def ddim50_b64_case():
    """ddim50 t = 5 .. 0 at B = 64: guided down to t = 3 (stop_recguidance_at inside the run), then imputation alone"""
    B, n = 64, 6
    w, sd, x_obs, kw, c, g = loop_case(B, seed=62, stop_recguidance_at=3)
    tape = torch.randn(1 + n, B, 263, 1, 196, generator=g)
    run = lambda: O.sample_loop(sd, O.make_tables("ddim50"), (B, 263, 1, 196), c, tape, "ddim", skip_timesteps=44,  # noqa: E731
                                init_image=x_obs, max_steps=n, return_all=True)
    return w, sd, x_obs, kw, tape, run, B, n


def engine_ddim50(precision, w, kw, tape, x_obs, B, n):
    d = C.create_gaussian_diffusion(timestep_respacing="ddim50")
    d.precision = precision
    d.noise_tape = tape.to(DEV)
    return engine_steps(d.ddim_sample_loop_progressive(w, (B, 263, 1, 196), model_kwargs=kw, skip_timesteps=44,
                                                       init_image=x_obs.to(DEV)), n)


def test_bf16_ddim50_tail_cfg_imputation_guidance_b64():
    w, sd, x_obs, kw, tape, run, B, n = ddim50_b64_case()
    got = engine_ddim50(TB.BF16, w, kw, tape, x_obs, B, n)
    a, f = oracle_loop(sd, run)
    gate_steps(got, a, f, "bf16 B=64 ddim50 t=5..0, cfg + imputation + guidance down to t=3")


def test_bf16x3_ddim50_tail_cfg_imputation_guidance_b64():
    """against the oracle with its model in exact fp32 on the GPU, rtol 1e-3 / atol 1e-4 on every step's pred_xstart and
    sample, with no allowance for the guided steps (coefficient ~10): measured on H100, max 8.9e-5, no element outside"""
    w, sd, x_obs, kw, tape, run, B, n = ddim50_b64_case()
    got = engine_ddim50(C.PRECISION_BF16X3, w, kw, tape, x_obs, B, n)
    want = oracle_loop(sd, run, exact_fp32=True)
    failures = []
    for k, (e, r) in enumerate(zip(got, want)):
        for key in ("pred_xstart", "sample"):
            ge, gr = e[key].cpu().double(), r[key].double()
            err = (ge - gr).abs()
            viol = (err > 1e-4 + 1e-3 * gr.abs()).double().mean().item()
            print(f"[bf16x3 B=64 ddim50 step {k} (t={5 - k}) {key}] max_abs={err.max():.3e} mean_abs={err.mean():.3e} "
                  f"gate violations={viol:.2e}")
            if viol > 0:
                failures.append((k, key, err.max().item(), viol))
    assert not failures, failures

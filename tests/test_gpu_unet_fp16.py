"""GPU: the MDM_UNET denoiser at CMDI_PRECISION_FP16 ("autocast"), the arithmetic the reference samples the published
use_fp16 checkpoints with: every conv / linear in fp16 (fp32 accumulation, fp16 result), GroupNorm / AdaGN / Mish and the
residual sums in fp32 (DESIGN.md section 3).

  A = the oracle's unet_forward on CUDA tensors inside torch.autocast("cuda", torch.float16): the reference's own GPU
      arithmetic (oracle/make_golden_unet_autocast.py shows the restatement puts autocast's casts where the reference does)
  F = the same oracle in fp32 (TF32 off)

Gates, in max and in mean of the absolute difference: |engine - A| <= |A - F| on every denoiser pass, and |engine - F| <=
2 |A - F| everywhere -- the engine is as close to the reference's fp16 run as that run is to fp32, and as accurate as it.

Two fp16 runs that round at the same points still part ways: where their fp32 sums differ in the last bit, an fp16 rounding
goes the other way, and the network spreads that.  Measured on H100, |engine - A| is 0.71-0.85 of |A - F| (max) on a pass.
A CFG output (1 - s) u + s c with s = 2.5 weighs two passes whose fp16 errors are largely shared; those shared parts cancel
in A - F more than in engine - A, and there the ratio is 1.02-1.07.  So a CFG forward is checked as its two passes (gated
above) plus the fp32 combine, and the B = 64 loop, whose steps are CFG outputs, against |A - F| with a 1.5x margin
(measured 1.18) besides the accuracy gate.
"""
import ctypes
import contextlib

import pytest
import torch

import condmdi_b200 as C
from oracle import condmdi_oracle as O

pytestmark = pytest.mark.gpu
D, L = 263, 196
DEV = "cuda:0"
FP16 = C.PRECISION_FP16


@contextlib.contextmanager
def exact_fp32():
    saved = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    try:
        yield
    finally:
        torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = saved


UNET_FORWARD = O.unet_forward  # (the loop test swaps the oracle's model function for a GPU one)


def to_dev(sd):
    return {k: v.to(DEV) for k, v in sd.items()}


def oracle(sd_dev, x, t, cond_emb=None, uncond=False, xo=None, kf=None, text_scale=None, autocast=True):
    """unet_forward (with the ClassifierFreeSampleModel combine when text_scale is given) on the GPU, under CUDA autocast or
    in exact fp32."""
    dev = lambda v: None if v is None else v.to(DEV)  # noqa: E731
    x, t, cond_emb, xo, kf = dev(x), dev(t), dev(cond_emb), dev(xo), dev(kf)
    ctx = torch.autocast("cuda", dtype=torch.float16) if autocast else exact_fp32()
    with torch.no_grad(), ctx:
        out = UNET_FORWARD(sd_dev, x, t, cond_emb, uncond, xo, kf)
        if text_scale is not None:
            out_u = UNET_FORWARD(sd_dev, x, t, cond_emb, True, xo, kf)
            out = out_u + (text_scale.to(DEV).view(-1, 1, 1, 1) * (out - out_u))  # cfg_sampler.py:25-35
    return out.float()


def engine_forward(m, x, t, cond_emb=None, uncond=False, xo=None, kf=None, text_scale=None, precision=FP16):
    """One engine call per distinct timestep (Engine.forward takes one)."""
    eng = m.engine_for(DEV, max_batch=x.shape[0], precision=precision, nframes=x.shape[-1])
    out = torch.empty(x.shape, device=DEV)
    for tv in t.unique().tolist():
        idx = (t == tv).nonzero().reshape(-1)
        sub = lambda v: None if v is None else v[idx].to(DEV)  # noqa: E731
        out[idx.to(DEV)] = eng.forward(x[idx].to(DEV), int(tv), cond_emb=sub(cond_emb), uncond=uncond, cfg=text_scale is not None,
                                       text_scale=sub(text_scale), obs_x0=sub(xo), obs_mask=sub(kf))
    return out


def gate(got, a, f, what, track=1.0):
    """|got - A| <= track * |A - F| and |got - F| <= 2 |A - F|, in max and in mean; prints every ratio."""
    got, a, f = got.double().cpu(), a.double().cpu(), f.double().cpu()
    e_a, a_f, e_f = (got - a).abs(), (a - f).abs(), (got - f).abs()
    r = {"max|E-A|/max|A-F|": (e_a.max() / a_f.max()).item(), "mean|E-A|/mean|A-F|": (e_a.mean() / a_f.mean()).item(),
         "max|E-F|/max|A-F|": (e_f.max() / a_f.max()).item(), "mean|E-F|/mean|A-F|": (e_f.mean() / a_f.mean()).item()}
    print(f"[{what}] |A-F| max={a_f.max():.3e} mean={a_f.mean():.3e}  " + "  ".join(f"{k}={v:.3f}" for k, v in r.items()))
    assert a_f.max() > 0
    assert r["max|E-A|/max|A-F|"] <= track and r["mean|E-A|/mean|A-F|"] <= track, what
    assert r["max|E-F|/max|A-F|"] <= 2.0 and r["mean|E-F|/mean|A-F|"] <= 2.0, what


def fp16_valued(t):
    return torch.equal(t, t.half().float())


def xl_module(B, seed=11):
    sd = O.random_unet_state_dict(seed=seed, text=True)
    m = C.MDM_UNET(keyframe_conditioned=True, cond_mode="text", cond_mask_prob=0.1)
    assert not any(m.load_state_dict(sd, strict=False))
    return m.to(DEV), sd


def xl_inputs(B, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, D, 1, L, generator=g)
    xo = torch.randn(B, D, 1, L, generator=g)
    lengths = torch.randint(40, L + 1, (B,), generator=g)
    kf = C.get_keyframes_mask(xo, lengths, "benchmark_sparse", trans_length=5)
    cond = torch.randn(B, 512, generator=g)
    t = torch.tensor([999, 37] * (B // 2))                 # per-sample timesteps
    scale = torch.full((B,), 2.5)
    return x, xo, kf, cond, t, scale


@pytest.mark.parametrize("B", [2, 64])
def test_fp16_unet_xl_forward(B):
    """The xl geometry (dim 512, dim_mults (2,2,2,2), keyframe input conditioning, text): plain, unconditional and CFG."""
    m, sd = xl_module(B)
    sdd = to_dev(sd)
    x, xo, kf, cond, t, scale = xl_inputs(B, seed=B)
    passes = {}
    for what, kw in [("text", {}), ("uncond", {"uncond": True})]:
        passes[what] = got = engine_forward(m, x, t, cond, xo=xo, kf=kf, **kw)
        assert fp16_valued(got)
        a = oracle(sdd, x, t, cond, xo=xo, kf=kf, **kw)
        f = oracle(sdd, x, t, cond, xo=xo, kf=kf, autocast=False, **kw)
        gate(got, a, f, f"xl B={B} {what}")
    # CFG: the batch-doubled pass computes the two passes above, combined in fp32 (cfg_sampler.py:25-35)
    got = engine_forward(m, x, t, cond, xo=xo, kf=kf, text_scale=scale)
    u, c = passes["uncond"], passes["text"]
    assert torch.allclose(got, u + scale.to(DEV).view(-1, 1, 1, 1) * (c - u), rtol=0, atol=1e-5)
    a = oracle(sdd, x, t, cond, xo=xo, kf=kf, text_scale=scale)
    f = oracle(sdd, x, t, cond, xo=xo, kf=kf, text_scale=scale, autocast=False)
    gate(got, a, f, f"xl B={B} cfg 2.5", track=1.5)


@pytest.mark.parametrize("mults,kf_cond", [((1, 1), True), ((1, 1), False), ((1, 1, 1), True), ((1, 1, 1), False)])
def test_fp16_unet_other_geometries(mults, kf_cond):
    """2- and 3-level UNets with and without keyframe input conditioning; unconditional model."""
    sd = O.random_unet_state_dict(seed=3, mults=mults, keyframe_conditioned=kf_cond)
    m = C.MDM_UNET(dim_mults=mults, keyframe_conditioned=kf_cond)
    assert not any(m.load_state_dict(sd, strict=False))
    m = m.to(DEV)
    x, xo, kf, _, t, _ = xl_inputs(2, seed=7)
    if not kf_cond:
        xo = kf = None
    got = engine_forward(m, x, t, xo=xo, kf=kf)
    assert fp16_valued(got)
    sdd = to_dev(sd)
    gate(got, oracle(sdd, x, t, xo=xo, kf=kf), oracle(sdd, x, t, xo=xo, kf=kf, autocast=False), f"unet {mults} kf={kf_cond}")


def test_fp16_unet_b64_ddim_tail_cfg_imputation():
    """B = 64 DDIM tail from a noise tape: keyframe input conditioning, imputation and CFG 2.5, against the oracle's loop
    with its model evaluations run on the GPU under autocast (A) and in fp32 (F)."""
    Bf = 64
    m, sd = xl_module(Bf)
    w = C.ClassifierFreeSampleModel(m)
    x_obs, _, kf, cond, _, scale = xl_inputs(Bf, seed=12)
    g = torch.Generator().manual_seed(13)
    lengths = torch.randint(40, L + 1, (Bf,), generator=g)
    y_mask = (torch.arange(L)[None] < lengths[:, None]).view(Bf, 1, 1, L)
    tape = torch.randn(5, Bf, D, 1, L, generator=g)
    table = {str(i): cond[i].to(DEV) for i in range(Bf)}
    m.encode_text = lambda texts: torch.stack([table[s] for s in texts])
    d = C.create_gaussian_diffusion(timestep_respacing="ddim50")
    d.precision = FP16
    d.noise_tape = tape.to(DEV)
    y = {"text": [str(i) for i in range(Bf)], "text_scale": scale.to(DEV), "mask": y_mask.to(DEV), "imputate": 1,
         "stop_imputation_at": 1, "replacement_distribution": "conditional", "inpainted_motion": x_obs.to(DEV),
         "inpainting_mask": kf.to(DEV)}
    got = d.ddim_sample_loop(w, (Bf, D, 1, L), model_kwargs={"y": y, "obs_x0": x_obs.to(DEV), "obs_mask": kf.to(DEV)},
                             skip_timesteps=46, init_image=x_obs.to(DEV))
    c = O.Conditioning(cond_emb=cond, cfg=True, text_scale=scale, y_mask=y_mask, imputate=True, stop_imputation_at=1,
                       inpainted_motion=x_obs, inpainting_mask=kf, obs_x0=x_obs, obs_mask=kf)
    sdd = to_dev(sd)
    want = {}
    try:
        for name, autocast in (("A", True), ("F", False)):
            def gpu_forward(sd_, x, t, cond_emb=None, uncond=False, obs_x0=None, obs_mask=None, _ac=autocast):
                out = oracle(sdd, x, t, cond_emb, uncond, obs_x0, obs_mask, autocast=_ac)
                return out.cpu()
            O.unet_forward = gpu_forward
            want[name] = O.sample_loop(sd, O.make_tables("ddim50"), (Bf, D, 1, L), c, tape, "ddim", skip_timesteps=46,
                                       init_image=x_obs)
    finally:
        O.unet_forward = UNET_FORWARD
    gate(got, want["A"], want["F"], "B=64 ddim tail, cfg + imputation + keyframes", track=1.5)


def test_fp16_gemm_vs_float64():
    """linear2_kernel's fp16 instantiation (cmdi_test_linear, precision 2) against a float64 product of the fp16-rounded
    operands: every result is an fp16 value, off the exact one by one fp16 rounding plus what fp32 accumulation allows."""
    lib = C.capi.load()
    p = lambda t: ctypes.c_void_p(t.data_ptr())  # noqa: E731
    for M, N, K, bn in [(300, 512, 512, -256), (1000, 256, 2048, -128), (128, 1024, 320, -256)]:
        g = torch.Generator(device="cuda").manual_seed(M + K)
        A = torch.randn(M, K, device="cuda", generator=g)
        W = torch.randn(N, K, device="cuda", generator=g) / K ** 0.5
        b = torch.randn(N, device="cuda", generator=g)
        out = torch.full((M, N), float("nan"), device="cuda")
        C.capi.check(lib.cmdi_test_linear(p(A), p(W), p(b), None, p(out), M, N, K, 0, 2, bn, None))
        torch.cuda.synchronize()
        A16, W16, b16 = A.half().double(), W.half().double(), b.half().double()
        exact = A16 @ W16.t() + b16
        ulp = exact.half().double().abs().clamp_min(2.0 ** -14) * 2.0 ** -10   # >= the fp16 spacing at the result
        acc = 2.0 ** -16 * (A16.abs() @ W16.abs().t() + b16.abs())            # fp32 accumulation of K products
        err = (out.double() - exact).abs()
        print(f"[fp16 gemm {M}x{N}x{K}] max |C - exact| / (ulp + acc) = {(err / (ulp + acc)).max():.3f}  "
              f"share off the nearest fp16 = {(out.double() != exact.half().double()).double().mean():.2e}")
        assert fp16_valued(out)
        assert bool((err <= ulp + acc).all())


def test_fp16_refused_for_the_transformer():
    with pytest.raises(RuntimeError, match="MDM_UNET"):
        C.Engine(DEV, precision=FP16, max_batch=2)


def test_bf16x3_engine_next_to_an_fp16_one_is_unchanged():
    """engine_for keys its cache on the precision: a bf16x3 engine built after an fp16 one for the same module computes
    bit for bit what a bf16x3 engine built alone computes."""
    sd = O.random_unet_state_dict(seed=5, mults=(1, 1))
    x, xo, kf, _, _, _ = xl_inputs(2, seed=3)
    t = torch.tensor([500, 500])

    def module():
        m = C.MDM_UNET(dim_mults=(1, 1), keyframe_conditioned=True)
        m.load_state_dict(sd, strict=False)
        return m.to(DEV)

    both = module()
    half = engine_forward(both, x, t, xo=xo, kf=kf)
    after = engine_forward(both, x, t, xo=xo, kf=kf, precision=C.PRECISION_BF16X3)
    alone = engine_forward(module(), x, t, xo=xo, kf=kf, precision=C.PRECISION_BF16X3)
    assert both.engine_for(DEV, max_batch=2, precision=FP16, nframes=L) is not both.engine_for(DEV, max_batch=2, nframes=L)
    assert torch.equal(after, alone)
    assert not torch.equal(half, alone)

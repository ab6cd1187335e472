"""PRECISION_BF16 (one bf16 MMA per product): the chained layer kernel and the engine against a bf16-aware fp64 model.

  F = the transformer forward in fp64 on the fp32 weights
  A = the same with BOTH operands of every matrix product (the linear layers, Q K^T, P V) rounded to bf16 and nothing else
      rounded: what one bf16 MMA per product costs when everything around the products is exact
  E = the engine at PRECISION_BF16

Contract (DESIGN.md section 3): |E - F| <= 2 |A - F| in max and in mean over a denoiser output.  |E - A| is printed: two
runs that round at the same points still part ways where an operand sits next to a bf16 rounding boundary.

The restatement below is pinned without a GPU: with no rounding it is oracle.condmdi_oracle.mdm_forward to fp32 rounding.
"""
import ctypes
import math

import pytest
import torch
import torch.nn.functional as F

import condmdi_b200 as C
from oracle import condmdi_oracle as O

DEV = "cuda:0"
BF16 = C.PRECISION_BF16
gpu = pytest.mark.gpu


def bf16r(t):
    return t.float().bfloat16().double()


def exact(t):
    return t


# ------------------------------------------------------------------------------------------------
# the model: oracle.condmdi_oracle.mdm_forward / _encoder_layer in fp64 with a rounding hook q on the products' operands
# ------------------------------------------------------------------------------------------------
def qlinear(q, x, w, b):
    return F.linear(q(x), q(w), b)


def encoder_layer(q, x, sd, pre, num_heads=4):
    S, B, d = x.shape
    dh = d // num_heads
    heads = lambda t: t.reshape(S, B, num_heads, dh).permute(1, 2, 0, 3)  # noqa: E731
    qq, k, v = (heads(t) for t in qlinear(q, x, sd[pre + "self_attn.in_proj_weight"], sd[pre + "self_attn.in_proj_bias"]).chunk(3, dim=-1))
    s = q(qq) @ q(k).transpose(-1, -2) / math.sqrt(dh)
    p = torch.exp(s - s.amax(dim=-1, keepdim=True))  # the product sees exp(s - max); the row sum divides its result
    a = (q(p) @ q(v) / p.sum(dim=-1, keepdim=True)).permute(2, 0, 1, 3).reshape(S, B, d)
    a = qlinear(q, a, sd[pre + "self_attn.out_proj.weight"], sd[pre + "self_attn.out_proj.bias"])
    x = F.layer_norm(x + a, (d,), sd[pre + "norm1.weight"], sd[pre + "norm1.bias"], 1e-5)
    h = F.gelu(qlinear(q, x, sd[pre + "linear1.weight"], sd[pre + "linear1.bias"]))
    h = qlinear(q, h, sd[pre + "linear2.weight"], sd[pre + "linear2.bias"])
    return F.layer_norm(x + h, (d,), sd[pre + "norm2.weight"], sd[pre + "norm2.bias"], 1e-5)


def mdm_model(q, sd, x, timesteps, cond_emb=None, uncond=False):
    """fp64 MDM.forward.  The timestep and text embeddings stay unrounded: the engine computes them once per weight load
    and per call at bf16x3 / fp32, not with one MMA."""
    sd = {k: v.double() for k, v in sd.items()}
    x = x.double()
    bs, njoints, nfeats, nframes = x.shape
    pe = sd["sequence_pos_encoder.pe"]
    emb = F.linear(F.silu(F.linear(pe[timesteps], sd["embed_timestep.time_embed.0.weight"], sd["embed_timestep.time_embed.0.bias"])),
                   sd["embed_timestep.time_embed.2.weight"], sd["embed_timestep.time_embed.2.bias"]).permute(1, 0, 2)
    if cond_emb is not None:
        c = torch.zeros_like(cond_emb) if uncond else cond_emb
        emb = emb + F.linear(c.double(), sd["embed_text.weight"], sd["embed_text.bias"])
    h = x.permute(3, 0, 1, 2).reshape(nframes, bs, njoints * nfeats)
    h = qlinear(q, h, sd["input_process.poseEmbedding.weight"], sd["input_process.poseEmbedding.bias"])
    xseq = torch.cat((emb, h), dim=0)
    xseq = xseq + pe[: xseq.shape[0]]
    for i in range(O.num_layers_of(sd)):
        xseq = encoder_layer(q, xseq, sd, f"seqTransEncoder.layers.{i}.")
    out = qlinear(q, xseq[1:], sd["output_process.poseFinal.weight"], sd["output_process.poseFinal.bias"])
    return out.reshape(nframes, bs, njoints, nfeats).permute(1, 2, 3, 0)


def test_model_without_rounding_is_the_oracle():
    sd = O.random_state_dict(seed=3, text=True)
    gi = O.golden_inputs()
    t = torch.tensor([999, 41])
    for kw in ({}, {"cond_emb": gi["cond"]}, {"cond_emb": gi["cond"], "uncond": True}):
        want = O.mdm_forward(sd, gi["x"], t, **kw)
        got = mdm_model(exact, sd, gi["x"], t, **kw)
        assert (got - want.double()).abs().max() < 2e-5  # fp32 rounding of an 8-layer forward, |out| ~ 1


def test_model_rounding_hook_costs_bf16_sized_error():
    sd = O.random_state_dict(seed=3, layers=2)
    gi = O.golden_inputs()
    t = torch.tensor([999, 41])
    a, f = mdm_model(bf16r, sd, gi["x"], t), mdm_model(exact, sd, gi["x"], t)
    err = (a - f).abs().max().item()
    assert 1e-4 < err < 1e-1, err  # 2^-9 per operand through two layers; fp32 rounding would be ~1e-6


# ------------------------------------------------------------------------------------------------
# one chained layer launch (cmdi_test_chain_layer) against fp64 of the same four sublayers
# ------------------------------------------------------------------------------------------------
def folded_ln_linear(q, v, w, gamma, beta, b):
    """LN(v) W^T + b as the chain computes it, rstd (v (W gamma)^T - mean c) + d: the product's operands, the ones q rounds,
    are the un-normalised v and W gamma.  With q = identity this is F.linear(F.layer_norm(v), W, b)."""
    mean = v.mean(dim=-1, keepdim=True)
    rstd = torch.rsqrt(v.var(dim=-1, unbiased=False, keepdim=True) + 1e-5)
    wf = w * gamma
    return rstd * (q(v) @ q(wf).t() - mean * wf.sum(dim=1)) + (w @ beta + b)


def chain_layer_reference(q, t):
    d = {k: v.double() for k, v in t.items()}
    ln = lambda v, g, b: F.layer_norm(v, (512,), g, b, 1e-5)  # noqa: E731
    v1 = qlinear(q, d["attn"], d["wo"], d["bo"]) + ln(d["v2_prev"], d["g2p"], d["be2p"])
    h = F.gelu(folded_ln_linear(q, v1, d["w1"], d["g1"], d["be1"], d["b1"]))
    v2 = qlinear(q, h, d["w2"], d["b2"]) + ln(v1, d["g1"], d["be1"])
    qkv = folded_ln_linear(q, v2, d["wqkv"], d["g2"], d["be2"], d["bqkv"])
    return v1, h, v2, qkv


V2_MEAN_BOUND = 3e-4  # measured 2.9e-6 (M = 2) .. 9.9e-5 on H100
CHAIN_KEYS = ["attn", "v2_prev", "g2p", "be2p", "wo", "bo", "g1", "be1", "w1", "b1", "w2", "b2", "g2", "be2", "wqkv", "bqkv"]


def chain_layer_inputs(M, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    rn = lambda *s: torch.randn(*s, device="cuda", generator=g)  # noqa: E731
    t = {"attn": rn(M, 512), "v2_prev": rn(M, 512) * 1.5 + 0.2}
    for name, (n, k) in {"wo": (512, 512), "w1": (1024, 512), "w2": (512, 1024), "wqkv": (1536, 512)}.items():
        t[name] = rn(n, k) / k ** 0.5
        t["b" + name[1:]] = rn(n) * 0.1
    for name in ("g2p", "g1", "g2"):
        t[name] = 1.0 + 0.1 * rn(512)
        t["be" + name[1:]] = 0.1 * rn(512)
    return t


@gpu
@pytest.mark.parametrize("M", [2, 197, 255, 256, 257, 394, 414, 12608, 25216])
@pytest.mark.parametrize("prec", [3, 1], ids=["bf16x3", "bf16"])
def test_chain_layer_against_fp64(M, prec):
    """Rows: a two-row launch, odd and even CTA-pair counts, a pair whose second CTA is all tail (257), 2 x 207, B = 64
    with and without CFG.  Stale lo planes hold 2^-7 (a bf16 ulp at 1, 100x the bf16x3 bound): nothing may read them before
    it is written.  A launch that cannot make its CTA pairs co-resident fails here with the library's message."""
    t = chain_layer_inputs(M, seed=M + prec)
    ins = (ctypes.c_void_p * 16)(*[t[k].data_ptr() for k in CHAIN_KEYS])
    outs = [torch.full((M, n), float("nan"), device="cuda") for n in (512, 1024, 512, 1536)]
    C.capi.check(C.capi.load().cmdi_test_chain_layer(ins, (ctypes.c_void_p * 4)(*[o.data_ptr() for o in outs]), M, prec, 2.0 ** -7, None))
    torch.cuda.synchronize()
    ref = chain_layer_reference(bf16r if prec == 1 else exact, t)
    err = {n: (o.double() - r).abs().max().item() for n, o, r in zip(("v1", "h", "v2", "qkv"), outs, ref)}
    v2_mean = (outs[2].double() - ref[2]).abs().mean().item()
    print(f"[chain layer M={M} prec={prec}] " + "  ".join(f"{k}={v:.2e}" for k, v in err.items()) + f"  mean v2={v2_mean:.2e}")
    assert all(torch.isfinite(o).all() for o in outs)
    if prec == 3:
        assert max(err.values()) < 1e-4, err  # the linear test's bound; measured 2.2e-5 .. 6.7e-5 on H100
    else:
        # v1 (hi + lo planes): fp32 accumulation only; measured 2.0e-5 .. 5.3e-5
        assert err["v1"] < 1.5e-4, err
        # v2 (hi + lo planes): where the kernel's h and the reference's round to different bf16 neighbours (|h| up to 8) one
        # product is off by 2^-8 |h w|, a few elements per row: measured max 3.4e-3 .. 5.5e-3.  That is rare, so the MEAN
        # separates it from a residual rounded to bf16 or a stale lo plane, which shift every element by ~2^-10 |LN(v1)| ~ 1e-3
        assert err["v2"] < 2e-2 and v2_mean < V2_MEAN_BOUND, (err, v2_mean)
        # h, qkv are handed back as the hi plane alone: half a bf16 ulp of |h|, |qkv| <~ 8; measured 1.0e-2 .. 1.8e-2
        assert err["h"] < 4e-2 and err["qkv"] < 4e-2, err


# ------------------------------------------------------------------------------------------------
# the engine at PRECISION_BF16
# ------------------------------------------------------------------------------------------------
def module(D=263, text=True, seed=7):
    sd = O.random_state_dict(seed=seed, feats=D, text=text)
    m = C.MDM(njoints=D, cond_mode="text" if text else "no_cond", cond_mask_prob=0.1)
    missing, unexpected = m.load_state_dict(sd, strict=False)
    assert not missing and not unexpected
    return m.to(DEV), sd


def engine_forward(m, x, t, precision=BF16, **kw):
    """one call per distinct timestep (Engine.forward takes one)"""
    eng = m.engine_for(DEV, max_batch=x.shape[0], precision=precision, nframes=x.shape[-1])
    out = torch.empty(x.shape, device=DEV)
    for tv in t.unique().tolist():
        idx = (t == tv).nonzero().reshape(-1)
        sub = {k: (v[idx].to(DEV) if torch.is_tensor(v) else v) for k, v in kw.items()}
        out[idx.to(DEV)] = eng.forward(x[idx].to(DEV), int(tv), **sub)
    return out


def model_on_gpu(q, sd, x, t, cond_emb=None, uncond=False):
    sdd = {k: v.to(DEV) for k, v in sd.items()}
    with torch.no_grad():
        return mdm_model(q, sdd, x.to(DEV), t.to(DEV), None if cond_emb is None else cond_emb.to(DEV), uncond)


def gate(got, a, f, what, c=2.0):
    """|E - F| <= c |A - F| in max and in mean; prints every ratio"""
    got, a, f = got.double().cpu(), a.double().cpu(), f.double().cpu()
    e_a, a_f, e_f = (got - a).abs(), (a - f).abs(), (got - f).abs()
    r_max, r_mean = (e_f.max() / a_f.max()).item(), (e_f.mean() / a_f.mean()).item()
    print(f"[{what}] |A-F| max={a_f.max():.3e} mean={a_f.mean():.3e}  |E-F|/|A-F| max={r_max:.3f} mean={r_mean:.3f}  "
          f"|E-A|/|A-F| max={(e_a.max() / a_f.max()).item():.3f} mean={(e_a.mean() / a_f.mean()).item():.3f}")
    assert torch.isfinite(got).all() and a_f.max() > 0
    assert r_max <= c and r_mean <= c, f"{what}: |E-F|/|A-F| max {r_max:.3f} mean {r_mean:.3f} > {c}"
    return r_max, r_mean


def inputs(B, D, L, seed):
    g = torch.Generator().manual_seed(seed)
    t = torch.tensor([0, 41, 999, 41])[torch.arange(B) % 4]
    return torch.randn(B, D, 1, L, generator=g), torch.randn(B, 512, generator=g), t, torch.full((B,), 2.5)


def forward_contract(B, D, L, what):
    m, sd = module(D)
    x, cond, t, scale = inputs(B, D, L, seed=B * 1000 + L)
    passes = {}
    for name, kw in [("text", {"cond_emb": cond}), ("uncond", {"cond_emb": cond, "uncond": True})]:
        passes[name] = got = engine_forward(m, x, t, **kw)
        gate(got, model_on_gpu(bf16r, sd, x, t, **kw), model_on_gpu(exact, sd, x, t, **kw), f"{what} B={B} {D}x{L} {name}")
    # CFG: the batch-doubled pass computes the two passes above (one shared timestep), combined in fp32
    t1 = torch.full((B,), 41)
    u, c = (engine_forward(m, x, t1, cond_emb=cond, uncond=un) for un in (True, False))
    got = engine_forward(m, x, t1, cond_emb=cond, cfg=True, text_scale=scale)
    assert torch.allclose(got, u + scale.to(DEV).view(-1, 1, 1, 1) * (c - u), rtol=0, atol=1e-5)
    return passes


@gpu
@pytest.mark.parametrize("B", [2, 64])
def test_bf16_transformer_forward_meets_the_contract(B):
    """text, unconditional and CFG passes at timesteps 0, 41, 999 on the chained path"""
    forward_contract(B, 263, 196, "chained")


@gpu
def test_bf16_unconditioned_model_meets_the_contract():
    m, sd = module(text=False)
    x, _, t, _ = inputs(2, 263, 196, seed=5)
    gate(engine_forward(m, x, t), model_on_gpu(bf16r, sd, x, t), model_on_gpu(exact, sd, x, t), "chained B=2 no_cond")


@gpu
@pytest.mark.parametrize("D,L", [(251, 120), (67, 57), (263, 1), (263, 207)])
def test_bf16_transformer_geometries(D, L):
    forward_contract(2, D, L, "chained")


@gpu
@pytest.mark.parametrize("B", [2, 64])
def test_bf16_unchained_path_meets_the_contract(monkeypatch, B):
    """CMDI_CHAIN=0: one launch per linear layer, fp32 residuals, LayerNorm kernels.  The difference between its ratios and
    the chained path's is what the plane-derived residual and the folded LayerNorm cost at bf16."""
    monkeypatch.setenv("CMDI_CHAIN", "0")
    forward_contract(B, 263, 196, "unchained")


@gpu
def test_bf16_forward_does_not_depend_on_the_calls_before_it():
    """activation planes keep nothing from an earlier pass, a guided (stashing, unchained, backward) one included"""
    m, _ = module()
    x1, cond, t, _ = inputs(2, 263, 196, seed=1)
    x2 = inputs(2, 263, 196, seed=2)[0] * 3
    t = torch.full((2,), 500)
    first = engine_forward(m, x1, t, cond_emb=cond)
    engine_forward(m, x2, t, cond_emb=cond)
    assert torch.equal(engine_forward(m, x1, t, cond_emb=cond), first)
    eng = m.engine_for(DEV, max_batch=2, precision=BF16, nframes=196)
    mask = O.get_keyframes_mask(x2, torch.tensor([196, 150]), "benchmark_sparse", 5)
    grad = eng.test_input_vjp(x2, 500, x2, mask, cond_emb=cond)
    assert torch.isfinite(grad).all()
    assert torch.equal(engine_forward(m, x1, t, cond_emb=cond), first)


@gpu
def test_bf16x3_engine_next_to_a_bf16_one_is_unchanged():
    x, cond, _, _ = inputs(2, 263, 196, seed=3)
    t = torch.full((2,), 500)
    both, _ = module()
    plain = engine_forward(both, x, t, cond_emb=cond)
    after = engine_forward(both, x, t, precision=C.PRECISION_BF16X3, cond_emb=cond)
    alone = engine_forward(module()[0], x, t, precision=C.PRECISION_BF16X3, cond_emb=cond)
    assert both.engine_for(DEV, max_batch=2, precision=BF16, nframes=196) is not both.engine_for(DEV, max_batch=2, nframes=196)
    assert torch.equal(after, alone)
    assert not torch.equal(plain, alone)

"""CPU: the per-op fp64 references of oracle/unet_ops.py, composed by name in the model's forward order (the names the
engine's UNet op lists carry), are condmdi_oracle.unet_forward -- values and input gradient -- to fp64 rounding.  So the
name -> module map the GPU op tests hold every engine op to is the model."""
import pytest
import torch

from oracle import condmdi_oracle as O
from oracle import unet_ops as U


def sd64(**kw):
    return {k: v.double() for k, v in O.random_unet_state_dict(seed=4, **kw).items()}


@pytest.mark.parametrize("mults,kf,text", [((1, 1, 1), False, False), ((1, 1), True, True), ((2, 2, 2, 2), True, True)])
def test_ops_compose_to_unet_forward(mults, kf, text):
    sd = sd64(dim=64 if len(mults) == 4 else 128, mults=mults, keyframe_conditioned=kf, text=text, feats=13)
    g = torch.Generator().manual_seed(1)
    B, D, L = 2, 13, 37
    x = torch.randn(B, D, 1, L, generator=g, dtype=torch.float64, requires_grad=True)
    xo = torch.randn(B, D, 1, L, generator=g, dtype=torch.float64) if kf else None
    mask = (torch.rand(B, D, 1, L, generator=g) < 0.3) if kf else None
    cond = torch.randn(B, 512, generator=g, dtype=torch.float64) if text else None
    t = torch.tensor([999, 37])
    seed = torch.randn(B, D, 1, L, generator=g, dtype=torch.float64)
    want = O.unet_forward(sd, x, t, cond, False, xo, mask)
    got = U.unet_forward_by_ops(sd, x, t, cond, False, xo, mask).float()
    assert got.shape == want.shape
    gw = torch.autograd.grad(want, x, seed)[0]
    gg = torch.autograd.grad(got, x, seed)[0]
    print(f"[{mults} kf={kf}] max |by ops - unet_forward| = {(got - want).abs().max():.2e}, gradient {(gg - gw).abs().max():.2e}")
    # unet_forward returns fp32 (its last op is .float()): equal up to that one rounding, and its gradient with it
    assert bool(((got - want).abs() <= 2.0 ** -24 * want.abs() + 1e-12).all())
    assert bool(((gg - gw).abs() <= 2.0 ** -22 * gw.abs() + 1e-9 * gw.abs().max()).all())


def test_forward_names_cover_every_module():
    """every convolution, linear and GroupNorm of the state dict is the module of exactly one forward op name"""
    sd = O.random_unet_state_dict(seed=0, mults=(2, 2, 2, 2), text=True)
    names = U.forward_names(sd)
    assert len(names) == len(set(names))
    modules = {k.rsplit(".", 1)[0] for k in sd if k.startswith("unet.")}
    pres = U.block_prefixes(4)
    covered = {n for n in names if n.startswith("unet.")} | {p + "time_mlp.1" for p in pres}
    assert modules == covered

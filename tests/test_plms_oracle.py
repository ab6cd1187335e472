"""CPU: the PLMS restatement in oracle/plms_oracle.py against tests/golden/plms.* (outputs of the UNMODIFIED reference's
plms_sample_loop_progressive, oracle/make_golden_plms.py), the argument errors of the PLMS entry points, and the
PLMS loops of install()."""
import numpy as np
import pytest
import torch

import condmdi_b200 as C
from oracle import condmdi_oracle as O
from oracle import plms_oracle as P
from oracle.golden_io import load_golden
from standin import StockDiffusion

B, D, L = 2, 263, 196
SHAPE = (B, D, 1, L)


@pytest.fixture(scope="module")
def gold(golden_dir):
    return load_golden(golden_dir, "plms")


@pytest.fixture(scope="module")
def gi(gold):
    gi = O.golden_inputs()
    chk = np.array([float(gi["x"].double().sum()), float(gi["tape"].double().sum()), float(gi["cond"].double().sum())])
    assert np.allclose(chk, gold["inputs.checksum"], rtol=0, atol=1e-9), "seeded inputs differ from the fixtures' inputs"
    return gi


def maxerr(a, b):
    return (torch.as_tensor(a).double() - torch.as_tensor(b).double()).abs().max().item()


@pytest.mark.parametrize("order,ks", [(2, (0, 1, 2)), (4, (3,))])
def test_plms_ddim50_loop_vs_reference_golden(gold, gi, order, ks):
    """the whole ddim50 loop: the improved Euler first step, the Adams-Bashforth ramp 2 -> 3 -> 4, the end at t = 0"""
    sd = O.random_state_dict(seed=7, text=False)
    outs = P.plms_sample_loop(sd, O.make_tables("ddim50"), SHAPE, O.Conditioning(), gi["tape"], return_all=True, order=order)
    assert len(outs) == 50
    for k in ks:
        assert maxerr(outs[k]["sample"], gold[f"o{order}.sample_k{k}"]) <= 5e-5, k
        assert len(outs[k]["old_eps"]) == min(k + 1, order - 1)
    assert maxerr(outs[-1]["sample"], gold[f"o{order}.final"]) <= 2e-4
    # the fp32 reference ends within 1e-5 of the float64 chain: PLMS does not amplify rounding the way the guided DDPM
    # tail does, so its end state is pinned at the gate directly
    assert gold[f"o{order}.ref_err_vs_f64"][0] < 1e-5


def test_plms_cfg_imputation_and_guidance_vs_reference_golden(gold, gi):
    sdt = O.random_state_dict(seed=7, text=True)
    tab = O.make_tables("ddim50")
    kw = dict(cond_emb=gi["cond"], cfg=True, text_scale=gi["text_scale"], y_mask=gi["y_mask"], imputate=True, stop_imputation_at=1,
              inpainted_motion=gi["x_obs"], inpainting_mask=gi["kf_mask"])
    got = P.plms_sample_loop(sdt, tab, SHAPE, O.Conditioning(**kw), gi["tape"], skip_timesteps=45, init_image=gi["x_obs"])
    assert maxerr(got, gold["cfg_impute.final"]) <= 1e-4
    c2 = O.Conditioning(reconstruction_guidance=True, reconstruction_weight=20.0, **kw)
    got = P.plms_sample_loop(sdt, tab, SHAPE, c2, gi["tape"], max_steps=2)
    assert maxerr(got, gold["recon.sample_k1"]) <= 1e-4


def test_plms_one_step_at_t0_vs_reference_golden(gold, gi):
    sd = O.random_state_dict(seed=7, text=False)
    outs = P.plms_sample_loop(sd, O.make_tables("ddim50"), SHAPE, O.Conditioning(), gi["tape"], skip_timesteps=49,
                              init_image=gi["x_obs"], return_all=True)
    assert len(outs) == 1
    assert torch.equal(outs[0]["sample"], outs[0]["pred_xstart"])  # at t = 0 the sample is the first evaluation's x0
    assert maxerr(outs[0]["sample"], gold["t0.sample"]) <= 5e-5


def test_plms_unet_order3_vs_reference_golden(gold, gi):
    sdu = O.random_unet_state_dict(seed=11, text=True)
    c = O.Conditioning(cond_emb=gi["cond"], cfg=True, text_scale=gi["text_scale"], obs_x0=gi["x_obs"], obs_mask=gi["kf_mask"])
    got = P.plms_sample_loop(sdu, O.make_tables("ddim50"), SHAPE, c, gi["tape"], skip_timesteps=45, init_image=gi["x_obs"],
                             order=3)
    assert maxerr(got, gold["unet.final"]) <= 5e-5


@pytest.mark.parametrize("order,exc", [(0, ValueError), (5, ValueError), (0.5, ValueError), (-1, ValueError), (1, TypeError),
                                       (2.5, NotImplementedError), (3.9, NotImplementedError)])
def test_plms_order_errors(order, exc):
    """raised at the call, before any model or device is touched"""
    d = C.create_gaussian_diffusion(timestep_respacing="ddim50")
    for fn in (d.plms_sample_loop, d.plms_sample_loop_progressive):
        with pytest.raises(exc):
            fn(None, SHAPE, model_kwargs={"y": {}}, order=order)
    with pytest.raises(exc):
        P.plms_check_order(order)


def test_plms_unsupported_arguments_raise_not_implemented():
    d = C.create_gaussian_diffusion(timestep_respacing="ddim50")
    with pytest.raises(NotImplementedError):
        d.plms_sample_loop(None, SHAPE, model_kwargs={"y": {}}, cond_fn=lambda x, t, **kw: x)
    with pytest.raises(NotImplementedError):
        d.plms_sample_loop_progressive(None, SHAPE, model_kwargs={"y": {}}, randomize_class=True)
    with pytest.raises(NotImplementedError):
        d.plms_sample_loop(None, SHAPE, model_kwargs={"y": {"gmd": True}})


class _EagerLoops(StockDiffusion):
    """A reference-like diffusion object whose own loops only record that they ran."""

    def plms_sample_loop(self, *args, **kwargs):
        return "eager plms_sample_loop"

    def plms_sample_loop_progressive(self, *args, **kwargs):
        return "eager plms_sample_loop_progressive"


@pytest.mark.parametrize("name", ["plms_sample_loop", "plms_sample_loop_progressive"])
def test_install_patches_the_plms_loops(name):
    base = C.create_gaussian_diffusion(timestep_respacing="ddim50")
    ref = C.install(_EagerLoops(base.betas, base.timestep_map))
    assert getattr(ref, name).__func__ is not getattr(_EagerLoops, name)
    # configurations the engine does not implement raise instead of running the eager loop ...
    with pytest.raises(NotImplementedError):
        getattr(ref, name)(None, SHAPE, model_kwargs={"y": {}}, cond_fn=lambda x, t, **kw: x)
    # ... and reach it only through the explicit opt-in
    ref2 = C.install(_EagerLoops(base.betas, base.timestep_map), fallback_to_reference=True)
    assert getattr(ref2, name)(None, SHAPE, model_kwargs={"y": {}}, order=2.5) == f"eager {name}"
    with pytest.raises(ValueError):  # argument errors are the reference's own: never forwarded
        getattr(ref2, name)(None, SHAPE, model_kwargs={"y": {}}, order=7)

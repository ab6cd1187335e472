"""CPU: the DDIM inversion restatement in oracle/ddim_reverse_oracle.py against tests/golden/ddim_reverse.* (outputs of the
UNMODIFIED reference's ddim_reverse_sample, oracle/make_golden_ddim_reverse.py), the argument errors of the inversion
entry points, and what install() adds."""
import numpy as np
import pytest
import torch

import condmdi_b200 as C
from oracle import condmdi_oracle as O
from oracle import ddim_reverse_oracle as R
from oracle.golden_io import load_golden
from standin import StockDiffusion

B, D, L = 2, 263, 196
SHAPE = (B, D, 1, L)


@pytest.fixture(scope="module")
def gold(golden_dir):
    return load_golden(golden_dir, "ddim_reverse")


@pytest.fixture(scope="module")
def gi(gold):
    gi = O.golden_inputs()
    chk = np.array([float(gi["x"].double().sum()), float(gi["tape"].double().sum()), float(gi["cond"].double().sum())])
    assert np.allclose(chk, gold["inputs.checksum"], rtol=0, atol=1e-9), "seeded inputs differ from the fixtures' inputs"
    return gi


def maxerr(a, b):
    return (torch.as_tensor(a).double() - torch.as_tensor(b).double()).abs().max().item()


def test_alphas_cumprod_next_table():
    tab = O.make_tables("ddim50")
    nxt = R.alphas_cumprod_next(tab)
    assert nxt[-1] == 0.0 and np.array_equal(nxt[:-1], tab.alphas_cumprod[1:])
    assert np.array_equal(C.create_gaussian_diffusion(timestep_respacing="ddim50").alphas_cumprod_next, nxt)


@pytest.mark.parametrize("name,ts", [("nocond", (0, 1, 10, 48, 49)), ("text", (0, 49)), ("cfg", (0, 10, 49))])
def test_single_steps_vs_reference_golden(gold, gi, name, ts):
    sd = O.random_state_dict(seed=7, text=name != "nocond")
    c = {"nocond": O.Conditioning(), "text": O.Conditioning(cond_emb=gi["cond"]),
         "cfg": O.Conditioning(cond_emb=gi["cond"], cfg=True, text_scale=gi["text_scale"])}[name]
    tab = O.make_tables("ddim50")
    for t in ts:
        o = R.ddim_reverse_sample(sd, tab, gi["x"], torch.tensor([t] * B), c)
        assert maxerr(o["pred_xstart"], gold[f"{name}.t{t}.pred_xstart"]) <= 5e-5, t
        assert maxerr(o["sample"], gold[f"{name}.t{t}.sample"]) <= (5e-4 if t == 0 else 5e-5), t
        # the update itself is the reference's bit for bit, given its pred_xstart
        ref_pred = torch.from_numpy(gold[f"{name}.t{t}.pred_xstart"])
        assert torch.equal(R.reverse_update(tab, gi["x"], torch.tensor([t] * B), ref_pred),
                           torch.from_numpy(gold[f"{name}.t{t}.sample"])), t


def test_whole_inversion_vs_reference_golden(gold, gi):
    sd = O.random_state_dict(seed=7, text=False)
    outs = R.ddim_reverse_sample_loop(sd, O.make_tables("ddim50"), gi["x"], O.Conditioning(), return_all=True)
    assert len(outs) == 50
    for k in (0, 1, 25):
        assert maxerr(outs[k]["sample"], gold[f"whole.k{k}.sample"]) <= 2e-4 * max(1.0, np.abs(gold[f"whole.k{k}.sample"]).max()), k
    # the end state is large (|x_T| ~ 760 for these random weights): the restatement tracks the reference to ~1e-6 of it
    end = gold["whole.k49.sample"]
    assert maxerr(outs[-1]["sample"], end) <= 1e-5 * np.abs(end).max()
    assert gold["whole.ref_err_vs_f64"][0] <= 1e-5 * np.abs(end).max()


def test_cfg_imputation_guidance_and_unet_vs_reference_golden(gold, gi):
    sdt = O.random_state_dict(seed=7, text=True)
    tab = O.make_tables("ddim50")
    kw = dict(cond_emb=gi["cond"], cfg=True, text_scale=gi["text_scale"], y_mask=gi["y_mask"], imputate=True,
              stop_imputation_at=1, inpainted_motion=gi["x_obs"], inpainting_mask=gi["kf_mask"])
    outs = R.ddim_reverse_sample_loop(sdt, tab, gi["x"], O.Conditioning(**kw), max_steps=3, return_all=True)
    for t in range(3):
        assert maxerr(outs[t]["sample"], gold[f"cfg_impute.t{t}.sample"]) <= (1e-3 if t == 0 else 2e-4), t
    M = (gi["kf_mask"] * gi["y_mask"].float()).bool()
    assert torch.equal(torch.from_numpy(gold["cfg_impute.t1.pred_xstart"])[M], gi["x_obs"][M])  # imputed at t >= 1
    c2 = O.Conditioning(reconstruction_guidance=True, reconstruction_weight=20.0, **kw)
    outs = R.ddim_reverse_sample_loop(sdt, tab, gi["x"], c2, t_start=10, max_steps=2, return_all=True)
    for j, t in enumerate((10, 11)):
        assert maxerr(outs[j]["pred_xstart"], gold[f"guided.t{t}.pred_xstart"]) <= 2e-4, t
        assert maxerr(outs[j]["sample"], gold[f"guided.t{t}.sample"]) <= 2e-4, t


def test_unet_xl_vs_reference_golden_bit_for_bit(gold, gi):
    """the restated MDM_UNET forward is the reference's bit for bit, so the inversion of it is too"""
    sdu = O.random_unet_state_dict(seed=11, text=True)
    cu = O.Conditioning(cond_emb=gi["cond"], cfg=True, text_scale=gi["text_scale"], obs_x0=gi["x_obs"], obs_mask=gi["kf_mask"])
    tab = O.make_tables("ddim50")
    o = R.ddim_reverse_sample(sdu, tab, gi["x"], torch.tensor([49, 49]), cu)
    assert np.array_equal(o["sample"].numpy(), gold["unet.t49.sample"])
    assert np.array_equal(o["pred_xstart"].numpy(), gold["unet.t49.pred_xstart"])
    got = R.ddim_reverse_sample_loop(sdu, tab, gi["x"], cu, t_start=20, max_steps=4)
    assert np.array_equal(got.numpy(), gold["unet.seg20_24.sample"])


def test_inversion_argument_errors():
    """raised at the call, before any model or device is touched"""
    d = C.create_gaussian_diffusion(timestep_respacing="ddim50")
    x = torch.zeros(SHAPE)
    with pytest.raises(AssertionError, match="Reverse ODE only for deterministic path"):
        d.ddim_reverse_sample(None, x, torch.tensor([3, 3]), model_kwargs={"y": {}}, eta=0.5)
    for fn in (d.ddim_reverse_sample_loop, d.ddim_reverse_sample_loop_progressive):
        with pytest.raises(AssertionError, match="Reverse ODE only for deterministic path"):
            fn(None, x, model_kwargs={"y": {}}, eta=0.1)
        with pytest.raises(NotImplementedError):
            fn(None, x, model_kwargs={"y": {}}, denoised_fn=lambda v: v)
    with pytest.raises(NotImplementedError, match="uniform"):
        d.ddim_reverse_sample(None, x, torch.tensor([3, 4]), model_kwargs={"y": {}})
    with pytest.raises(NotImplementedError):
        d.ddim_reverse_sample_loop(None, x, model_kwargs={"y": {"gmd": True}})
    with pytest.raises(AssertionError):
        R.ddim_reverse_sample(None, O.make_tables("ddim50"), x, torch.tensor([0, 0]), O.Conditioning(), eta=0.5)


class _EagerStep(StockDiffusion):
    """A reference-like diffusion object with its own eager ddim_reverse_sample."""

    def ddim_reverse_sample(self, *args, **kwargs):
        return "eager ddim_reverse_sample"


def test_install_adds_the_inversion_loops_and_keeps_the_reference_step():
    base = C.create_gaussian_diffusion(timestep_respacing="ddim50")
    ref = C.install(_EagerStep(base.betas, base.timestep_map))
    assert ref.ddim_reverse_sample(None, None, None) == "eager ddim_reverse_sample"
    for name in ("ddim_reverse_sample_loop", "ddim_reverse_sample_loop_progressive"):
        with pytest.raises(AssertionError, match="Reverse ODE"):
            getattr(ref, name)(None, torch.zeros(SHAPE), model_kwargs={"y": {}}, eta=1.0)
    fast = C.accelerate(_EagerStep(base.betas, base.timestep_map))
    assert isinstance(fast, C.GaussianDiffusion) and fast.ddim_reverse_sample.__func__ is C.GaussianDiffusion.ddim_reverse_sample

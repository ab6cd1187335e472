"""CPU: the keyframe classifier-free guidance restatement (oracle/keyframe_cfg_oracle.py) and the wrapper's construction.

  - the restatement equals the reference-driven fixtures tests/golden/keyframe_cfg.* (oracle/make_golden_keyframe_cfg.py);
  - at w_k = 1 it equals the CFG restatement within fp32 rounding; the no_cond model's two-pass form;
  - KeyframeClassifierFreeSampleModel refuses the transformer and a UNet without keyframe input.
"""
import os

import pytest
import torch

import condmdi_b200 as C
from oracle import condmdi_oracle as O
from oracle import keyframe_cfg_oracle as K
from oracle.golden_io import load_golden

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
D, L = 263, 196


def small_inputs(B=2, N=L, seed=0):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, D, 1, N, generator=g)
    xo = torch.randn(B, D, 1, N, generator=g)
    kf = torch.zeros(B, D, 1, N, dtype=torch.bool)
    kf[..., ::20] = True
    return x, xo, kf, torch.randn(B, 512, generator=g)


@pytest.fixture(scope="module")
def small():
    return O.random_unet_state_dict(seed=3, mults=(1, 1), text=True)


def test_unit_keyframe_scale_is_cfg_within_rounding(small):
    x, xo, kf, cond = small_inputs()
    c = O.Conditioning(cond_emb=cond, cfg=True, text_scale=torch.tensor([2.5, 1.5]), obs_x0=xo, obs_mask=kf)
    t = torch.tensor([500, 500])
    with torch.no_grad():
        cfg = O._model(small, x, t, c)
        with K.keyframe_cfg(torch.ones(2)):
            got = O._model(small, x, t, c)
    assert torch.allclose(got, cfg, rtol=0, atol=1e-5 * cfg.abs().max().item())


def test_two_pass_form_of_a_no_cond_model():
    sd = O.random_unet_state_dict(seed=4, mults=(1, 1))
    x, xo, kf, _ = small_inputs(seed=1)
    wk = torch.tensor([2.0, 0.5])
    c = O.Conditioning(obs_x0=xo, obs_mask=kf)
    t = torch.tensor([30, 30])
    with torch.no_grad():
        with K.keyframe_cfg(wk):
            got = O._model(sd, x, t, c)
        cc = O.unet_forward(sd, x, t, None, False, xo, kf)
        nn = O.unet_forward(sd, x, t, None, False, xo, torch.zeros_like(kf))
        # obs_mask = 0 is the unblended input with zero mask channels
        assert torch.equal(nn, O.unet_forward(sd, x, t, None, False, x, torch.zeros_like(kf)))
    assert torch.equal(got, nn + wk.view(-1, 1, 1, 1) * (cc - nn))


def test_restatement_equals_the_reference_fixtures():
    try:
        gold = load_golden(GOLDEN, "keyframe_cfg")
    except FileNotFoundError:
        pytest.skip("tests/golden/keyframe_cfg.* not generated")
    from oracle import make_golden_keyframe_cfg as MG
    for name, got in MG.restated_outputs(names=[k[:-len(".ref")] for k in gold if k.endswith(".ref")]).items():
        assert torch.equal(torch.from_numpy(gold[f"{name}.ref"]), got), name


def test_wrapper_refuses_other_models():
    with pytest.raises(ValueError):
        C.KeyframeClassifierFreeSampleModel(C.MDM(cond_mode="text", cond_mask_prob=0.1))
    with pytest.raises(ValueError):
        C.KeyframeClassifierFreeSampleModel(C.MDM_UNET(dim_mults=(1, 1), keyframe_conditioned=False))
    w = C.KeyframeClassifierFreeSampleModel(C.MDM_UNET(dim_mults=(1, 1), keyframe_conditioned=True, cond_mode="text"))
    for attr in ("rot2xyz", "translation", "njoints", "nfeats", "data_rep", "cond_mode", "keyframe_conditioned", "mask_value"):
        assert hasattr(w, attr), attr
    # a text model's wrapper reads y['text_scale'] as well (w_t = 1 without text guidance)
    with pytest.raises(ValueError, match="text_scale"):
        w(torch.zeros(1, D, 1, L), torch.zeros(1), {"keyframe_scale": torch.ones(1)})
    inner, is_cfg = C.resolve_model(w)
    assert inner is w.model and is_cfg
    assert C.model.is_keyframe_cfg(w) and not C.model.is_keyframe_cfg(w.model)
    assert C.model.keyframe_cfg_max_batch(64, True) == 96 and C.model.keyframe_cfg_max_batch(5, False) == 5

"""CPU: the oracle restatement against the fixtures generated from the UNMODIFIED reference
(oracle/make_golden.py).  This is what pins the oracle where /root/reference does not exist."""
import os

import numpy as np
import pytest
import torch

from oracle import condmdi_oracle as O
from oracle.golden_io import load_golden

B, D, L = 2, 263, 196


@pytest.fixture(scope="module")
def sched(golden_dir):
    return load_golden(golden_dir, "schedules")


@pytest.fixture(scope="module")
def samp(golden_dir):
    return load_golden(golden_dir, "sampler")


@pytest.mark.parametrize("name,resp", [("full", ""), ("ddim50", "ddim50"), ("ddim100", "ddim100"), ("sect", "10,15,20")])
def test_schedule_tables_bit_exact(sched, name, resp):
    t = O.make_tables(resp)
    assert np.array_equal(sched[f"{name}.timestep_map"], np.array(t.timestep_map))
    for f in ("betas", "alphas_cumprod", "alphas_cumprod_prev", "sqrt_alphas_cumprod", "sqrt_one_minus_alphas_cumprod",
              "sqrt_recip_alphas_cumprod", "sqrt_recipm1_alphas_cumprod", "posterior_variance",
              "posterior_log_variance_clipped", "posterior_mean_coef1", "posterior_mean_coef2"):
        assert np.array_equal(sched[f"{name}.{f}"], getattr(t, f)), f


@pytest.mark.parametrize("name", [None, "first-half", "last-half", "exponential", "sigmoid", "half-sigmoid"])
def test_gradient_schedule(sched, name):
    assert np.array_equal(sched[f"grad.{name}"], O.get_gradient_schedule(name, 1000))


def test_keyframe_masks_bit_exact(golden_dir):
    g = load_golden(golden_dir, "masks")
    keys = sorted(k[:-5] for k in g if k.endswith(".bits"))
    assert len(keys) == 27
    for key in keys:
        mode, T, fm = key.split(".")
        lengths = torch.tensor(g[key + ".lengths"])
        m = O.get_keyframes_mask(torch.zeros(len(lengths), D, 1, L), lengths, edit_mode=mode, trans_length=int(T), feature_mode=fm)
        assert np.array_equal(np.packbits(m.numpy().reshape(-1)), g[key + ".bits"]), key
        assert np.array_equal(m.sum(dim=(1, 2, 3)).numpy(), g[key + ".sums"])
    # the known-answer row of SURVEY.md 8(c)
    assert g["benchmark_sparse.5.pos_rot_vel.sums"].tolist() == [10520, 6312, 3156, 263]


def _inputs(samp):
    gi = O.golden_inputs()
    chk = np.array([float(gi["x"].double().sum()), float(gi["tape"].double().sum()), float(gi["cond"].double().sum())])
    assert np.allclose(chk, samp["inputs.checksum"], rtol=0, atol=1e-9), "seeded inputs differ from the ones the fixtures were made with"
    return gi


def test_forward_matches_reference(samp):
    gi = _inputs(samp)
    sd = O.random_state_dict(seed=7)
    out = O.mdm_forward(sd, gi["x"], torch.tensor(samp["fwd_nocond.t"]))
    assert torch.allclose(out, torch.tensor(samp["fwd_nocond.out"]), rtol=1e-4, atol=2e-5)


def test_text_and_cfg_forward_match_reference(samp):
    gi = _inputs(samp)
    sdt = O.random_state_dict(seed=7, text=True)
    t = torch.tensor([500, 500])
    assert torch.allclose(O.mdm_forward(sdt, gi["x"], t, gi["cond"]), torch.tensor(samp["fwd_text.out"]), rtol=1e-4, atol=2e-5)
    assert torch.allclose(O.cfg_forward(sdt, gi["x"], t, gi["cond"], gi["text_scale"]), torch.tensor(samp["fwd_cfg.out"]),
                          rtol=1e-4, atol=5e-5)


def test_ddpm_loop_matches_reference(samp):
    gi = _inputs(samp)
    sd = O.random_state_dict(seed=7)
    outs = O.sample_loop(sd, O.make_tables(""), (B, D, 1, L), O.Conditioning(), gi["tape"], "ddpm", max_steps=3, return_all=True)
    assert torch.allclose(outs[-1]["sample"], torch.tensor(samp["ddpm_uncond.sample"]), rtol=1e-4, atol=5e-5)
    assert torch.allclose(outs[-1]["pred_xstart"], torch.tensor(samp["ddpm_uncond.pred_xstart"]), rtol=1e-4, atol=5e-5)


def test_cfg_imputation_loop_matches_reference(samp):
    gi = _inputs(samp)
    sdt = O.random_state_dict(seed=7, text=True)
    c = O.Conditioning(cond_emb=gi["cond"], cfg=True, text_scale=gi["text_scale"], y_mask=gi["y_mask"], imputate=True,
                       stop_imputation_at=1, inpainted_motion=gi["x_obs"], inpainting_mask=gi["kf_mask"])
    assert np.array_equal(np.packbits(gi["kf_mask"].numpy().reshape(-1)), samp["kf_mask.bits"])
    outs = O.sample_loop(sdt, O.make_tables(""), (B, D, 1, L), c, gi["tape"], "ddpm", skip_timesteps=996,
                         init_image=gi["x_obs"], return_all=True)
    assert torch.allclose(outs[-1]["sample"], torch.tensor(samp["cfg_impute.sample"]), rtol=1e-4, atol=1e-4)
    assert torch.allclose(outs[2]["pred_xstart"], torch.tensor(samp["cfg_impute.pred_xstart_t1"]), rtol=1e-4, atol=1e-4)
    M = (gi["kf_mask"] * gi["y_mask"].float()).bool()
    assert torch.equal(outs[2]["pred_xstart"][M], gi["x_obs"][M])  # imputed entries are exactly the observations


def test_reconstruction_guidance_matches_reference(samp):
    gi = _inputs(samp)
    sdt = O.random_state_dict(seed=7, text=True)
    c = O.Conditioning(cond_emb=gi["cond"], cfg=True, text_scale=gi["text_scale"], y_mask=gi["y_mask"], imputate=True,
                       stop_imputation_at=1, inpainted_motion=gi["x_obs"], inpainting_mask=gi["kf_mask"],
                       reconstruction_guidance=True, reconstruction_weight=20.0)
    outs = O.sample_loop(sdt, O.make_tables(""), (B, D, 1, L), c, gi["tape"], "ddpm", max_steps=2, return_all=True)
    assert torch.allclose(outs[-1]["sample"], torch.tensor(samp["recon.sample"]), rtol=1e-4, atol=2e-4)
    assert torch.allclose(outs[-1]["pred_xstart"], torch.tensor(samp["recon.pred_xstart"]), rtol=1e-4, atol=2e-4)


def test_ddim50_full_loop_matches_reference(samp):
    gi = _inputs(samp)
    sd = O.random_state_dict(seed=7)
    tape50 = gi["tape"][torch.arange(51) % 8]
    out = O.sample_loop(sd, O.make_tables("ddim50"), (B, D, 1, L), O.Conditioning(), tape50, "ddim")
    assert torch.allclose(out, torch.tensor(samp["ddim50.sample"]), rtol=1e-3, atol=2e-4)


@pytest.mark.parametrize("tag,abs_3d", [("rel", False), ("abs", True)])
def test_recover_from_ric_matches_reference(golden_dir, tag, abs_3d):
    """Post-processing row (SURVEY 8f-2): the restatement of recover_from_ric / inv_transform against the
    reference's own output (sample/synthesize.py:153-157 chain)."""
    g = load_golden(golden_dir, "postprocess")
    inp = O.postprocess_inputs()
    got = O.sample_to_joints(inp["sample"], g[f"{tag}.mean"], g[f"{tag}.std"], 22, abs_3d)
    assert got.shape == (3, 22, 3, 196)
    assert torch.allclose(got, torch.from_numpy(g[f"{tag}.joints"]), rtol=1e-5, atol=2e-5)
    rag = O.recover_from_ric(inp["ragged"], 22, abs_3d)
    assert rag.shape == (2, 1, 57, 22, 3)
    assert torch.allclose(rag, torch.from_numpy(g[f"{tag}.ragged"]), rtol=1e-6, atol=1e-6)


def test_full_length_loop_fixture_last_steps(golden_dir):
    """tests/golden/long_loop.npz = the reference's own 1000-step DDPM loop (B=2).  The CPU suite replays its last
    five steps from the reference's state at t=4 (the whole chain takes minutes on a CPU; the GPU suite runs all of it)."""
    g = load_golden(golden_dir, "long_loop")
    tape = O.long_loop_tape()
    assert np.allclose([float(tape.double().sum()), float(tape[500].double().abs().sum())], g["tape_checksum"], rtol=1e-12)
    sd, tab, c = O.random_state_dict(seed=7, text=False), O.make_tables(""), O.Conditioning()
    x = torch.from_numpy(g["x_at_t4"])
    with torch.no_grad():
        for t in range(4, -1, -1):
            x = O.p_sample(sd, tab, x, torch.full((2,), t), c, tape[1 + 999 - t])["sample"]
    assert torch.allclose(x, torch.from_numpy(g["sample"]), rtol=1e-5, atol=2e-5)


def test_stock_torch_standin_equals_oracle_on_cpu():
    """tests/standin.py (stock nn.TransformerEncoder under the reference's keys; used by the GPU drop-in test where
    /root/reference is absent) computes what the oracle computes from the same state dict."""
    import sys
    sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
    from standin import ClassifierFreeSampleModel as StockCFG
    from standin import StockMDM
    torch.manual_seed(11)
    stock = StockMDM(text=True, layers=2).eval()
    gi = O.golden_inputs()
    stock.text_emb = gi["cond"]
    sd = {k: v.detach() for k, v in stock.state_dict().items()}
    assert set(sd.keys()) == set(O.random_state_dict(seed=0, text=True, layers=2).keys())
    t = torch.tensor([300, 300])
    with torch.no_grad():
        got = StockCFG(stock)(gi["x"], t, y={"text": ["a", "b"], "text_scale": gi["text_scale"]})
    want = O.cfg_forward(sd, gi["x"], t, gi["cond"], gi["text_scale"])
    assert torch.allclose(got, want, rtol=1e-4, atol=2e-5), (got - want).abs().max()


def test_oracle_long_chains_vs_reference_golden(golden_dir):
    """tests/golden/chains.npz (reference outputs): whole DDIM-100 loop and the t = 49..0 tail of CFG + imputation."""
    g = load_golden(golden_dir, "chains")
    gi = O.golden_inputs()
    tape = gi["tape"]
    sd = O.random_state_dict(seed=7, text=False)
    got = O.sample_loop(sd, O.make_tables("ddim100"), (B, D, 1, L), O.Conditioning(), tape[torch.arange(101) % 8], "ddim")
    assert torch.allclose(got, torch.from_numpy(g["ddim100.sample"]), rtol=1e-4, atol=2e-5)
    sdt = O.random_state_dict(seed=7, text=True)
    c = O.Conditioning(cond_emb=gi["cond"], cfg=True, text_scale=gi["text_scale"], y_mask=gi["y_mask"], imputate=True,
                       stop_imputation_at=1, inpainted_motion=gi["x_obs"], inpainting_mask=gi["kf_mask"])
    got = O.sample_loop(sdt, O.make_tables(""), (B, D, 1, L), c, tape[torch.arange(51) % 8], "ddpm", skip_timesteps=950,
                        init_image=gi["x_obs"])
    assert torch.allclose(got, torch.from_numpy(g["cfg_impute50.sample"]), rtol=1e-4, atol=5e-5)


def test_oracle_unet_vs_reference_golden(golden_dir):
    """tests/golden/unet.npz: the reference's MDM_UNET (dim 512 x (2,2,2,2), AdaGN, keyframe-conditioned, text)."""
    g = load_golden(golden_dir, "unet")
    gi = O.golden_inputs()
    sd = O.random_unet_state_dict(seed=11, text=True)
    assert O.is_unet(sd) and O.unet_levels_of(sd) == 4
    t = torch.from_numpy(g["fwd.t"])
    with torch.no_grad():
        got = O.unet_forward(sd, gi["x"], t, gi["cond"], False, gi["x_obs"], gi["kf_mask"])
        got_u = O.unet_forward(sd, gi["x"], t, gi["cond"], True, gi["x_obs"], gi["kf_mask"])
    assert torch.allclose(got, torch.from_numpy(g["fwd.out"]), rtol=1e-5, atol=1e-6)
    assert torch.allclose(got_u, torch.from_numpy(g["fwd_uncond.out"]), rtol=1e-5, atol=1e-6)
    c = O.Conditioning(cond_emb=gi["cond"], cfg=True, text_scale=gi["text_scale"], obs_x0=gi["x_obs"], obs_mask=gi["kf_mask"])
    tail = O.sample_loop(sd, O.make_tables(""), (B, D, 1, L), c, gi["tape"], "ddpm", skip_timesteps=996, init_image=gi["x_obs"])
    assert torch.allclose(tail, torch.from_numpy(g["tail4.sample"]), rtol=1e-5, atol=2e-6)

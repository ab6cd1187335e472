"""CPU: classifier-free guidance limited to an interval of steps (y['stop_cfg_at'] / y['start_cfg_at']).

  - the restatement (oracle/cfg_interval_oracle.py) equals the reference-driven fixtures tests/golden/cfg_interval.*
    (oracle/make_golden_cfg_interval.py): bit for bit for MDM_UNET, as the keyframe-CFG fixtures hold, and within
    2e-6 of max |x| for the transformer, whose restated forward rounds differently from the reference's (measured:
    at most 8.9e-7); and the interval changes those loops;
  - an interval covering every step is the wrapper, one covering none the inner model's conditional pass;
  - the Python refusals; run_eval_jobs merges only jobs with equal intervals and sharding copies them to every rank.
"""
import os

import pytest
import torch

import condmdi_b200 as C
from condmdi_b200.distributed import shard_model_kwargs
from condmdi_b200.eval_loop import EvalJob, _mergeable
from oracle import cfg_interval_oracle as CI
from oracle import condmdi_oracle as O
from oracle.golden_io import load_golden

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
D, L = 263, 196


def test_restatement_equals_the_reference_fixtures():
    from oracle import make_golden_cfg_interval as MG
    gold = load_golden(GOLDEN, "cfg_interval")
    names = [k[:-len(".ref")] for k in gold if k.endswith(".ref")]
    assert sorted(names) == sorted(MG.CASES)
    got = MG.restated_outputs(names)
    for name in names:
        ref = torch.from_numpy(gold[f"{name}.ref"])
        if MG.CASES[name][0] == "tf":
            err = (ref - got[name]).abs().max().item()
            assert err <= 2e-6 * ref.abs().max().item(), (name, err)
        else:
            assert torch.equal(ref, got[name]), name


def test_the_interval_changes_the_fixture_loops():
    """The same loops guided at every step differ from the fixtures far beyond the restatement's tolerance."""
    from oracle import make_golden_cfg_interval as MG
    gold = load_golden(GOLDEN, "cfg_interval")
    saved = dict(MG.CASES)
    try:
        for name in ("tf.ddim", "tf.guided.ddpm"):
            MG.CASES[name] = saved[name][:2] + ((None, None),) + saved[name][3:]
        full = MG.restated_outputs(["tf.ddim", "tf.guided.ddpm"])
    finally:
        MG.CASES.clear()
        MG.CASES.update(saved)
    for name, x in full.items():
        ref = torch.from_numpy(gold[f"{name}.ref"])
        assert (ref - x).abs().max().item() > 1e-3 * ref.abs().max().item(), name


@pytest.fixture(scope="module")
def small():
    return O.random_state_dict(seed=5, layers=2, text=True)


def test_whole_and_empty_intervals(small):
    g = torch.Generator().manual_seed(0)
    x, cond = torch.randn(2, D, 1, L, generator=g), torch.randn(2, 512, generator=g)
    tab = O.make_tables("ddim10")
    c = O.Conditioning(cond_emb=cond, cfg=True, text_scale=torch.tensor([2.5, 0.7]))
    t = torch.tensor([4, 4])
    with torch.no_grad():
        cfg = O.p_mean_variance(small, tab, x, t, c)["pred_xstart"]
        plain = O.mdm_forward(small, x, torch.tensor(tab.timestep_map)[t], cond)
        with CI.cfg_interval(tab, 0, 9):
            assert torch.equal(O.p_mean_variance(small, tab, x, t, c)["pred_xstart"], cfg)
        for stop, start in ((5, None), (None, 3), (10, 10)):
            with CI.cfg_interval(tab, stop, start):
                assert torch.equal(O.p_mean_variance(small, tab, x, t, c)["pred_xstart"], plain)
        with CI.cfg_interval(tab, 4, 4):
            assert torch.equal(O.p_mean_variance(small, tab, x, t, c)["pred_xstart"], cfg)
    assert O._model is CI._plain_model


def _y(**kw):
    y = {"text": ["a", "b"], "text_scale": torch.ones(2)}
    y.update(kw)
    return y


@pytest.mark.parametrize("y, match", [
    (_y(stop_cfg_at=2.0), "must be an int"),
    (_y(start_cfg_at=True), "must be an int"),
    (_y(stop_cfg_at=torch.tensor(2)), "must be an int"),
    (_y(stop_cfg_at=5, start_cfg_at=2), "stop_cfg_at'\\] = 5 > "),
])
def test_python_refusals(y, match):
    d = C.create_gaussian_diffusion(timestep_respacing="ddim10")
    m = C.ClassifierFreeSampleModel(C.MDM(cond_mode="text", cond_mask_prob=0.1))
    with pytest.raises(ValueError, match=match):
        d.ddim_sample_loop(m, (2, D, 1, L), model_kwargs={"y": y}, device="cpu")


@pytest.mark.parametrize("model", ["plain", "unet"])
def test_python_refuses_a_model_without_guidance(model):
    d = C.create_gaussian_diffusion(timestep_respacing="ddim10")
    m = C.MDM(cond_mode="text", cond_mask_prob=0.1) if model == "plain" else C.MDM_UNET(dim_mults=(1, 1), keyframe_conditioned=True)
    with pytest.raises(ValueError, match="ClassifierFreeSampleModel"):
        d.ddim_sample_loop(m, (2, D, 1, L), model_kwargs={"y": _y(stop_cfg_at=3)}, device="cpu")


def test_eval_jobs_merge_only_equal_intervals():
    def job(**kw):
        return EvalJob(0, 0, (2, D, 1, L), {"y": _y(**kw)})
    assert _mergeable(job(stop_cfg_at=3, start_cfg_at=7), job(stop_cfg_at=3, start_cfg_at=7))
    assert not _mergeable(job(stop_cfg_at=3, start_cfg_at=7), job(stop_cfg_at=3, start_cfg_at=8))
    assert not _mergeable(job(stop_cfg_at=3), job(start_cfg_at=3))
    assert not _mergeable(job(stop_cfg_at=3), job())


def test_sharding_copies_the_interval_to_every_rank():
    kw = {"y": _y(stop_cfg_at=3, start_cfg_at=7)}
    for lo, hi in ((0, 1), (1, 2)):
        s = shard_model_kwargs(kw, lo, hi, 2)["y"]
        assert s["stop_cfg_at"] == 3 and s["start_cfg_at"] == 7
        assert s["text"] == kw["y"]["text"][lo:hi]

"""CPU: the restatement's p_mean_variance with reconstruction guidance on the keyframe-conditioned MDM_UNET (xl), in fp32 and
under CPU fp16 autocast around the model call, against the UNMODIFIED reference's outputs (tests/golden/unet_guidance.*,
written by oracle/make_golden_unet_guidance.py, where the two agreed bit for bit).

Under autocast this pins where the forward's casts fall and which dtypes autograd's backward sees -- what
tests/test_gpu_unet_guidance.py relies on when it takes the restatement under CUDA autocast as the reference's own GPU run.
The gate is a small fraction of the autocast-vs-fp32 gap (another CPU may order a reduction differently); whether the match
is exact is printed.
"""
import pytest
import torch

from oracle import condmdi_oracle as O
from oracle.golden_io import load_golden
from oracle.make_golden_unet_guidance import cases, inputs, run_oracle


@pytest.fixture(scope="module")
def gold(golden_dir):
    return load_golden(golden_dir, "unet_guidance")


@pytest.mark.parametrize("name,cfg,t,imputate,schedule", cases(), ids=[c[0] for c in cases()])
def test_guided_p_mean_variance_matches_reference(gold, name, cfg, t, imputate, schedule):
    gi = inputs()
    sd = O.random_unet_state_dict(seed=11, text=True)
    f32 = torch.from_numpy(gold[f"fp32.{name}.pred_xstart"])
    for mode in ("fp32", "fp16"):
        pred, mean = run_oracle(sd, gi, cfg, t, imputate, schedule, mode == "fp16")
        want_p, want_m = torch.from_numpy(gold[f"{mode}.{name}.pred_xstart"]), torch.from_numpy(gold[f"{mode}.{name}.mean"])
        gap = (torch.from_numpy(gold[f"fp16.{name}.pred_xstart"]) - f32).abs().max().item()
        err = max((pred - want_p).abs().max().item(), (mean - want_m).abs().max().item())
        print(f"[{mode} {name}] exact={torch.equal(pred, want_p) and torch.equal(mean, want_m)} max|oracle - reference|={err:.3e} "
              f"max|autocast - fp32|={gap:.3e}")
        assert gap > 0
        assert err <= 0.01 * gap, (mode, name)

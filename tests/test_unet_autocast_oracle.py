"""CPU: the MDM_UNET restatement (oracle.condmdi_oracle.unet_forward) under CPU autocast against the UNMODIFIED reference's
outputs under the same autocast (tests/golden/unet_autocast.*, written by oracle/make_golden_unet_autocast.py, where the two
agreed bit for bit).

This is what lets the fp16 GPU tests use the restatement under CUDA autocast as the reference's own GPU run: a cast in a
different place would move the result by as much as autocast itself does.  The gate is therefore a small fraction of the
autocast-vs-fp32 gap (a different CPU may order a reduction differently), and the test reports whether the match is exact.
"""
import pytest
import torch

from oracle import condmdi_oracle as O
from oracle.golden_io import load_golden

DTYPES = {"bf16": torch.bfloat16, "fp16": torch.float16}


@pytest.fixture(scope="module")
def gold(golden_dir):
    return load_golden(golden_dir, "unet_autocast")


@pytest.mark.parametrize("kf", [True, False], ids=["kf", "nokf"])
def test_restatement_under_cpu_autocast_matches_reference(gold, kf):
    gi = O.golden_inputs()
    x, cond, x_obs, scale, kf_mask = (gi[k] for k in ("x", "cond", "x_obs", "text_scale", "kf_mask"))
    obs = (x_obs, kf_mask) if kf else (None, None)
    sd = O.random_unet_state_dict(seed=11, text=True, keyframe_conditioned=kf)
    tag = "kf" if kf else "nokf"
    t = torch.tensor([999, 37])
    cfg = O.Conditioning(cond_emb=cond, cfg=True, text_scale=scale, obs_x0=obs[0], obs_mask=obs[1])
    runs = {"text": lambda: O.unet_forward(sd, x, t, cond, False, *obs),
            "uncond": lambda: O.unet_forward(sd, x, t, cond, True, *obs),
            "cfg": lambda: O._model(sd, x, torch.tensor([500, 500]), cfg)}
    checked = 0
    for dname, dt in DTYPES.items():
        for what, fn in runs.items():
            key = f"{dname}.{tag}.{what}"
            if key not in gold:
                continue  # float16 CPU autocast was not available where the fixture was written
            want = torch.from_numpy(gold[key])
            with torch.no_grad():
                with torch.autocast("cpu", dtype=dt):
                    got = fn()
                f32 = fn()
            gap = (want - f32).abs().max().item()
            err = (got - want).abs().max().item()
            print(f"[{key}] exact={torch.equal(got, want)} max|oracle - reference|={err:.3e} max|autocast - fp32|={gap:.3e}")
            assert got.dtype == torch.float32 and gap > 0
            assert err <= 0.01 * gap, key
            checked += 1
    assert checked >= 3

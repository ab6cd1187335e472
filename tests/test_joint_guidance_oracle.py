"""CPU: the joint-guidance restatement (oracle/joint_guidance_oracle.py) against the oracle's recover_from_ric and finite
differences, and the host side of joint-position guidance: JointSpace, the validation that raises before any launch,
and the sharding of the new model_kwargs keys."""
import numpy as np
import pytest
import torch

import condmdi_b200 as C
from condmdi_b200.distributed import shard_model_kwargs
from oracle import condmdi_oracle as O
from oracle import joint_guidance_oracle as J
from oracle import make_golden_joint_guidance as MG
from oracle.golden_io import load_golden


@pytest.mark.parametrize("abs_3d", [True, False], ids=["abs3d", "rel"])
def test_restatement_equals_the_oracles_recover_from_ric(abs_3d, golden_dir):
    """bit for bit on the post-processing fixture's inputs and dataset statistics (the reference's own values)"""
    z = np.load(f"{golden_dir}/postprocess.npz")
    rep = "abs" if abs_3d else "rel"
    mean, std = torch.from_numpy(z[f"{rep}.mean"]).float(), torch.from_numpy(z[f"{rep}.std"]).float()
    x0 = O.postprocess_inputs()["sample"]
    data = x0[:, :, 0].transpose(1, 2) * std + mean
    assert torch.equal(J.recover_from_ric(data, abs_3d), O.recover_from_ric(data, 22, abs_3d))
    assert torch.equal(J.joint_positions(x0, mean, std, abs_3d), O.sample_to_joints(x0, mean, std, 22, abs_3d).permute(0, 3, 1, 2))


@pytest.mark.parametrize("abs_3d", [True, False], ids=["abs3d", "rel"])
def test_joint_seed_matches_finite_differences(abs_3d):
    mean, std, target, mask, g = J.inputs(2, 7, seed=3)
    x0 = torch.randn(2, 263, 1, 7, generator=g, dtype=torch.float64)
    args = (target.double(), mask, mean.double(), std.double(), abs_3d)
    grad = J.joint_seed(x0, *args)
    assert (grad[:, 67:] == 0).all()
    eps = 1e-6
    for idx in [(0, 0, 0, 2), (1, 1, 0, 0), (0, 2, 0, 5), (1, 3, 0, 4), (0, 40, 0, 1), (1, 66, 0, 6)]:
        xp, xm = x0.clone(), x0.clone()
        xp[idx] += eps
        xm[idx] -= eps
        fd = (J.joint_loss(xp, *args) - J.joint_loss(xm, *args)) / (2 * eps)
        assert abs(fd.item() - grad[idx].item()) <= 1e-5 * max(1.0, abs(fd.item())), (idx, fd.item(), grad[idx].item())


def test_joint_space():
    m = np.zeros(263)
    s = C.JointSpace(m, np.ones(263), abs_3d=False)
    assert s.mean.dtype == torch.float32 and s.std.shape == (263,) and s.abs_3d is False
    with pytest.raises(ValueError):
        C.JointSpace(np.zeros((263, 1)), np.ones((263, 1)))
    with pytest.raises(ValueError):
        C.JointSpace(m, np.ones(262))
    with pytest.raises(NotImplementedError, match="inv_proj"):
        C.JointSpace(m, np.ones(263), inv_proj=torch.eye(263))


class _Inner(torch.nn.Module):
    """just enough of a model for GaussianDiffusion._run to reach its validation: joint guidance is checked before the
    engine is created"""
    cond_mode = "no_cond"

    def __init__(self):
        super().__init__()
        self.w = torch.nn.Parameter(torch.zeros(1))

    def engine_for(self, *args, **kwargs):
        raise AssertionError("validation must raise before the engine is created")


def _y(B=2, L=196):
    return {"mask": torch.ones(B, 1, 1, L, dtype=torch.bool), "joint_guidance": True,
            "joint_target": torch.zeros(B, L, 22, 3), "joint_target_mask": torch.ones(B, L, 22, 3, dtype=torch.bool),
            "joint_guidance_weight": 1.0, "joint_gradient_schedule": None, "stop_jointguidance_at": 0,
            "diffusion_steps": 1000}


def _sample(d, y, shape=(2, 263, 1, 196)):
    C.diffusion.resolve_model = lambda m: (m, False)
    try:
        d.ddim_sample_loop(_Inner(), shape, model_kwargs={"y": y}, device="cpu")
    finally:
        C.diffusion.resolve_model = RESOLVE


RESOLVE = C.diffusion.resolve_model
SPACE = C.JointSpace(np.zeros(263), np.ones(263), abs_3d=True)


@pytest.mark.parametrize("case,exc,match", [
    ("no_space", NotImplementedError, "joint_space"),
    ("not_a_space", TypeError, "JointSpace"),
    ("D251", NotImplementedError, "263"),
    ("window", NotImplementedError, "windows"),
    ("target_shape", ValueError, "joint_target"),
    ("target_dtype", ValueError, "joint_target"),
    ("mask_dtype", ValueError, "joint_target_mask"),
    ("mask_shape", ValueError, "joint_target_mask"),
    ("weight", ValueError, "joint_guidance_weight"),
    ("stop", ValueError, "stop_jointguidance_at"),
    ("missing", ValueError, "joint_target"),
])
def test_validation_raises_before_any_launch(case, exc, match):
    d = C.create_gaussian_diffusion(timestep_respacing="ddim50")
    d.joint_space = SPACE
    y, shape = _y(), (2, 263, 1, 196)
    if case == "no_space":
        d.joint_space = None
    elif case == "not_a_space":
        d.joint_space = (np.zeros(263), np.ones(263))
    elif case == "D251":
        shape = (2, 251, 1, 196)
    elif case == "window":
        d.window = C.Window(196, 0)
    elif case == "target_shape":
        y["joint_target"] = torch.zeros(2, 196, 21, 3)
    elif case == "target_dtype":
        y["joint_target"] = torch.zeros(2, 196, 22, 3, dtype=torch.int64)
    elif case == "mask_dtype":
        y["joint_target_mask"] = torch.ones(2, 196, 22, 3)
    elif case == "mask_shape":
        y["joint_target_mask"] = torch.ones(2, 196, 22, dtype=torch.bool)
    elif case == "weight":
        y["joint_guidance_weight"] = "1"
    elif case == "stop":
        y["stop_jointguidance_at"] = 2.5
    elif case == "missing":
        del y["joint_target"]
    with pytest.raises(exc, match=match):
        _sample(d, y, shape)


def test_shard_model_kwargs_slices_the_joint_keys():
    y = _y(B=4)
    y["joint_target"] = torch.arange(4 * 196 * 66, dtype=torch.float32).reshape(4, 196, 22, 3)
    out = shard_model_kwargs({"y": y}, 1, 3, 4)["y"]
    assert torch.equal(out["joint_target"], y["joint_target"][1:3])
    assert torch.equal(out["joint_target_mask"], y["joint_target_mask"][1:3])
    assert out["joint_guidance"] is True and out["joint_guidance_weight"] == 1.0 and out["stop_jointguidance_at"] == 0


# ---------------------------------------------------------------------------------------------------------------------
# the restated guided evaluation against tests/golden/joint_guidance.* (the reference's model call, CFG wrapper and
# recover_from_ric under autograd, oracle/make_golden_joint_guidance.py)
# ---------------------------------------------------------------------------------------------------------------------
# measured when the fixtures were written: max |restatement - reference| / max |pred_xstart| <= 7.8e-6 (the
# transformer's summation order and qrot's operation order differ from the restatement's); bit for bit for MDM_UNET
# under CPU fp16 autocast, 3.5e-8 of its scale in fp32
GOLDEN_REL_TOL = 2e-5


@pytest.mark.parametrize("case", [c[0] for c in MG.CASES])
def test_restated_update_equals_the_reference_driven_fixture(case, golden_dir):
    gold = load_golden(golden_dir, "joint_guidance")
    _, which, t, abs_3d, keyframes, autocast = next(c for c in MG.CASES if c[0] == case)
    gi = O.golden_inputs()
    assert np.allclose(gold["inputs.checksum"], [float(gi["x"].double().sum()), float(MG.term(True).target.double().sum())])
    sd = O.random_state_dict(seed=7, text=True) if which == "trans" else O.random_unet_state_dict(seed=11, text=True)
    pred, mean = MG.run_oracle(sd, gi, t, MG.term(abs_3d), keyframes, which == "unet", autocast)
    for key, got in (("pred_xstart", pred), ("mean", mean)):
        want = torch.from_numpy(gold[f"{case}.{key}"])
        err = (got.double() - want.double()).abs().max().item()
        assert err <= GOLDEN_REL_TOL * want.abs().max().item(), (case, key, err)
        if which == "unet" and autocast:
            assert torch.equal(got, want), (case, key, err)

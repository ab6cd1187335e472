"""CPU: the obstacle-avoidance restatement (oracle/obstacle_oracle.py) against the fixtures driven by the reference's own
CondKeyLocationsWithSdf, the reference's collision formula, torch's subgradients at distance 0 and at distance r, the
radius-0 padding rows, finite differences, GMD's obs_list form, and the validation that raises before any launch."""
import numpy as np
import pytest
import torch

import condmdi_b200 as C
from oracle import condmdi_oracle as O
from oracle import joint_guidance_oracle as J
from oracle import make_golden_obstacle as MG
from oracle import obstacle_oracle as OB
from oracle.golden_io import load_golden


def _case(B=2, L=9, seed=3, abs_3d=True, K=3, joints=(0,), pad=0):
    mean, std, x0, obs, _ = OB.inputs(B, L, seed=seed, K=K, joints=joints, abs_3d=abs_3d, pad=pad)
    return x0.double(), mean.double(), std.double(), obs.double()


def test_loss_is_the_reference_collision_term_over_the_whole_motion():
    """GMD's loop (condition.py: dist = clamp(rad - |trajec[:, :, [0, 2]] - cent|, 0); loss += dist.sum() / L) with
    obstacles shared by the batch, the pelvis and every frame valid"""
    x0, mean, std, obs = _case(L=30)
    obs_list = [((float(o[0]), float(o[1])), float(o[2])) for o in obs[0]]
    trajec = J.joint_positions(x0, mean, std, True)[:, :, 0]
    want = 0.0
    for (cx, cz), rad in obs_list:
        dist = torch.norm(trajec[:, :, [0, 2]] - torch.tensor([cx, cz], dtype=torch.float64), dim=2)
        want = want + torch.clamp(rad - dist, min=0.0).sum() / trajec.shape[1]
    got = OB.obstacle_loss(x0, mean, std, True, OB.obstacles_from_list(obs_list, 2).double())
    assert want.item() > 0
    assert abs(got.item() - want.item()) <= 1e-12 * want.item()


@pytest.mark.parametrize("abs_3d", [True, False], ids=["abs3d", "rel"])
@pytest.mark.parametrize("joints", [(0,), (0, 10, 21)], ids=["pelvis", "three"])
def test_obstacle_seed_matches_finite_differences(abs_3d, joints):
    x0, mean, std, obs = _case(abs_3d=abs_3d, joints=joints, K=4, pad=1)
    valid = torch.ones(2, 9, dtype=torch.bool)
    valid[1, 6:] = False
    assert OB.obstacle_loss(x0, mean, std, abs_3d, obs, joints, valid) > 0
    grad = OB.obstacle_seed(x0, mean, std, abs_3d, obs, joints, valid)
    assert (grad[:, 67:] == 0).all() and grad.abs().max() > 0
    eps = 1e-6
    for b in range(2):
        for c in range(67):
            for f in (0, 3, 5, 7):
                idx = (b, c, 0, f)
                if grad[idx] == 0 and c > 3:
                    continue
                xp, xm = x0.clone(), x0.clone()
                xp[idx] += eps
                xm[idx] -= eps
                fd = (OB.obstacle_loss(xp, mean, std, abs_3d, obs, joints, valid) -
                      OB.obstacle_loss(xm, mean, std, abs_3d, obs, joints, valid)) / (2 * eps)
                assert abs(fd.item() - grad[idx].item()) <= 1e-6 * max(1.0, abs(fd.item())), (idx, fd.item(), grad[idx].item())


def _pelvis_case(dtype):
    """abs_3d with mean 0 and std 1: the pelvis XZ of frame f is x0[:, 1:3, 0, f] exactly"""
    mean, std = torch.zeros(263, dtype=dtype), torch.ones(263, dtype=dtype)
    x0 = torch.zeros(1, 263, 1, 4, dtype=dtype)
    x0[0, 1, 0] = torch.tensor([0.5, 2.0, -3.0, 8.0], dtype=dtype)
    x0[0, 2, 0] = torch.tensor([0.25, -1.0, 4.0, 8.0], dtype=dtype)
    return x0, mean, std


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
def test_subgradient_at_distance_zero_is_zero(dtype):
    x0, mean, std = _pelvis_case(dtype)
    obs = torch.tensor([[[0.5, 0.25, 1.0]]], dtype=dtype)         # centred on frame 0's pelvis, d = 0
    assert OB.obstacle_loss(x0, mean, std, True, obs).item() == 1.0 / 4
    grad = OB.obstacle_seed(x0, mean, std, True, obs)
    assert (grad == 0).all()                                       # by value: the norm's backward gives (-0, -0)


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
def test_subgradient_at_distance_r_passes_the_clamp(dtype):
    x0, mean, std = _pelvis_case(dtype)
    # frame 1's pelvis (2, -1) at distance exactly r = 1.25 from (1.25, -2): P - c = (0.75, 1.0)
    obs = torch.tensor([[[1.25, -2.0, 1.25]]], dtype=dtype)
    assert OB.obstacle_loss(x0, mean, std, True, obs).item() == 0.0
    grad = OB.obstacle_seed(x0, mean, std, True, obs)
    want = -torch.tensor([0.75, 1.0], dtype=torch.float64) / 1.25 / 4
    assert torch.allclose(grad[0, 1:3, 0, 1].double(), want, rtol=1e-6 if dtype == torch.float32 else 1e-15, atol=0)
    grad[0, 1:3, 0, 1] = 0
    assert (grad == 0).all()


@pytest.mark.parametrize("abs_3d", [True, False], ids=["abs3d", "rel"])
def test_radius_zero_rows_contribute_nothing(abs_3d):
    x0, mean, std, obs = _case(abs_3d=abs_3d, K=3)
    P = J.joint_positions(x0, mean, std, abs_3d)[:, :, 0][..., [0, 2]]
    pad = torch.zeros(2, 2, 3, dtype=torch.float64)
    pad[:, 0, :2] = P[:, 4]                                         # a padding row on the pelvis: d = 0, r = 0
    pad[:, 1, :2] = P[:, 5] + 1e-3
    padded = torch.cat((obs, pad), 1)
    assert torch.equal(OB.obstacle_loss(x0, mean, std, abs_3d, padded), OB.obstacle_loss(x0, mean, std, abs_3d, obs))
    assert torch.equal(OB.obstacle_seed(x0, mean, std, abs_3d, padded), OB.obstacle_seed(x0, mean, std, abs_3d, obs))
    assert (OB.obstacle_seed(x0, mean, std, abs_3d, pad) == 0).all()


@pytest.mark.parametrize("abs_3d", [True, False], ids=["abs3d", "rel"])
def test_small_update_lowers_the_loss(abs_3d):
    x0, mean, std, obs = _case(B=3, L=40, seed=8, abs_3d=abs_3d, K=6)
    before = OB.obstacle_loss(x0, mean, std, abs_3d, obs)
    grad = OB.obstacle_seed(x0, mean, std, abs_3d, obs)
    after = OB.obstacle_loss(x0 - 1e-3 / grad.abs().max().item() * grad, mean, std, abs_3d, obs)
    assert before > 0 and after < before, (before.item(), after.item())


def test_obs_list_is_the_shared_tensor_form():
    obs_list = [((0.5, -1.25), 0.75), ((2.0, 3.0), 0.0), ((-1.0, 0.1), 1.5)]
    want = torch.tensor([[0.5, -1.25, 0.75], [2.0, 3.0, 0.0], [-1.0, 0.1, 1.5]]).expand(3, -1, -1)
    assert torch.equal(OB.obstacles_from_list(obs_list, 3), want)
    assert torch.equal(C.diffusion._obstacles_tensor(obs_list, 3), want)
    assert torch.equal(C.diffusion._obstacles_tensor(want.double(), 3), want)
    assert C.diffusion._obstacles_tensor([], 2).shape == (2, 0, 3)
    space = C.JointSpace(np.zeros(263), np.ones(263), abs_3d=True)
    d = C.create_gaussian_diffusion(timestep_respacing="ddim50")
    args = [C.diffusion._obstacle_args(space, dict(_y(B=3), obstacles=o), 3, 263, 196, d.num_timesteps,
                                       d.sqrt_alphas_cumprod, None, "cpu") for o in (obs_list, want)]
    assert torch.equal(args[0]["obstacles"], args[1]["obstacles"])
    assert args[0]["obstacle_joints"] == 1 and args[0]["obstacle_coef"].shape == (50,)
    x0, mean, std, _ = _case(B=3)
    assert torch.equal(OB.obstacle_loss(x0, mean, std, True, OB.obstacles_from_list(obs_list, 3)),
                       OB.obstacle_loss(x0, mean, std, True, want))


def test_engine_coefficients_and_joint_mask():
    space = C.JointSpace(np.zeros(263), np.ones(263), abs_3d=False)
    d = C.create_gaussian_diffusion(timestep_respacing="ddim50")
    y = dict(_y(), obstacle_weight=3.0, obstacle_joints=[0, 7, 21], stop_obstacleguidance_at=5)
    a = C.diffusion._obstacle_args(space, y, 2, 263, 196, d.num_timesteps, d.sqrt_alphas_cumprod, None, "cpu")
    assert a["obstacle_joints"] == (1 | 1 << 7 | 1 << 21) and a["stop_obstacleguidance_at"] == 5
    assert a["joint_abs3d"] is False and a["obstacle_mask"].shape == (2, 196)
    sab = torch.from_numpy(d.sqrt_alphas_cumprod).float()
    w = torch.from_numpy(C.get_gradient_schedule(None, 1000))[torch.arange(50)].float() * 3.0
    assert np.array_equal(a["obstacle_coef"], (w * sab / 2).numpy())


class _Inner(torch.nn.Module):
    """just enough of a model for GaussianDiffusion._run to reach its validation"""
    cond_mode = "no_cond"

    def __init__(self):
        super().__init__()
        self.w = torch.nn.Parameter(torch.zeros(1))

    def engine_for(self, *args, **kwargs):
        raise AssertionError("validation must raise before the engine is created")


def _y(B=2, L=196):
    return {"mask": torch.ones(B, 1, 1, L, dtype=torch.bool), "obstacle_guidance": True, "obstacle_weight": 1.0,
            "obstacles": [((0.0, 0.0), 0.5)], "stop_obstacleguidance_at": 0, "diffusion_steps": 1000}


RESOLVE = C.diffusion.resolve_model
SPACE = C.JointSpace(np.zeros(263), np.ones(263), abs_3d=True)


@pytest.mark.parametrize("case,exc,match", [
    ("no_space", NotImplementedError, "joint_space"),
    ("not_a_space", TypeError, "JointSpace"),
    ("D251", NotImplementedError, "263"),
    ("window", NotImplementedError, "windows"),
    ("weight", ValueError, "obstacle_weight"),
    ("stop", ValueError, "stop_obstacleguidance_at"),
    ("missing", ValueError, "obstacles"),
    ("too_many", ValueError, "at most 16"),
    ("negative_r", ValueError, "negative radius"),
    ("nan", ValueError, "non-finite"),
    ("inf", ValueError, "non-finite"),
    ("shape", ValueError, r"\(2, K, 3\)"),
    ("int_tensor", ValueError, "float tensor"),
    ("bad_list", ValueError, "obs_list"),
    ("not_a_list", ValueError, "list of"),
    ("joints_empty", ValueError, "obstacle_joints"),
    ("joints_22", ValueError, "obstacle_joints"),
    ("joints_dup", ValueError, "obstacle_joints"),
    ("joints_bool", ValueError, "obstacle_joints"),
    ("mask_shape", ValueError, "mask"),
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
    elif case == "weight":
        y["obstacle_weight"] = "1"
    elif case == "stop":
        y["stop_obstacleguidance_at"] = 2.5
    elif case == "missing":
        del y["obstacles"]
    elif case == "too_many":
        y["obstacles"] = [((float(k), 0.0), 0.5) for k in range(17)]
    elif case == "negative_r":
        y["obstacles"] = torch.tensor([[[0.0, 0.0, 0.5], [1.0, 1.0, -0.1]]]).expand(2, -1, -1)
    elif case == "nan":
        y["obstacles"] = [((float("nan"), 0.0), 0.5)]
    elif case == "inf":
        y["obstacles"] = torch.tensor([[[0.0, 0.0, float("inf")]]]).expand(2, -1, -1)
    elif case == "shape":
        y["obstacles"] = torch.zeros(3, 1, 3)
    elif case == "int_tensor":
        y["obstacles"] = torch.zeros(2, 1, 3, dtype=torch.int64)
    elif case == "bad_list":
        y["obstacles"] = [(0.0, 0.0, 0.5)]
    elif case == "not_a_list":
        y["obstacles"] = "obstacles"
    elif case == "joints_empty":
        y["obstacle_joints"] = []
    elif case == "joints_22":
        y["obstacle_joints"] = [0, 22]
    elif case == "joints_dup":
        y["obstacle_joints"] = [3, 3]
    elif case == "joints_bool":
        y["obstacle_joints"] = [True]
    elif case == "mask_shape":
        y["mask"] = torch.ones(2, 1, 1, 100, dtype=torch.bool)
    C.diffusion.resolve_model = lambda m: (m, False)
    try:
        with pytest.raises(exc, match=match):
            d.ddim_sample_loop(_Inner(), shape, model_kwargs={"y": y}, device="cpu")
    finally:
        C.diffusion.resolve_model = RESOLVE


# ---------------------------------------------------------------------------------------------------------------------
# the restated guided evaluation against tests/golden/obstacle.* (the reference's model call, CFG wrapper and
# CondKeyLocationsWithSdf under autograd, oracle/make_golden_obstacle.py)
# ---------------------------------------------------------------------------------------------------------------------
# the gate of the foot-contact fixtures on the guided evaluation.  Measured when the fixtures were written: max
# |restatement - reference| / max |pred_xstart| <= 8.0e-6 (transformer, relative root), 1.7e-6 (transformer, abs_3d),
# 6.6e-8 (MDM_UNET fp32) and 0 (MDM_UNET under CPU fp16 autocast)
GOLDEN_REL_TOL = 2e-5
# dL_o/dz alone, relative to its own largest entry: measured <= 2.3e-4 (transformer, relative root: the root and
# heading are prefix sums over frames, whose summation order differs between the restatement and the reference, and
# the suffix sums of the adjoint magnify those differences), 2.5e-5 (transformer, abs_3d), 3.6e-6 (MDM_UNET fp32)
GRAD_REL_TOL = 1e-3


@pytest.mark.parametrize("case", [c[0] for c in MG.CASES])
def test_restated_update_equals_the_reference_driven_fixture(case, golden_dir):
    gold = load_golden(golden_dir, "obstacle")
    _, which, t, abs_3d, autocast = next(c for c in MG.CASES if c[0] == case)
    gi = MG.golden_inputs()
    assert np.allclose(gold["inputs.checksum"], [float(gi["x"].double().sum()), float(MG.statistics()[0].double().sum())])
    sd = O.random_state_dict(seed=7, text=True) if which == "trans" else O.random_unet_state_dict(seed=11, text=True)
    obstacles = torch.from_numpy(gold[f"{case}.obstacles"])
    assert (obstacles[..., 2] == 0).any() and (obstacles[..., 2] > 0).sum() >= 4
    pred, mean, grad = MG.run_oracle(sd, gi, t, MG.oracle_term(obstacles, abs_3d), which == "unet", autocast)
    for key, got in (("pred_xstart", pred), ("mean", mean)):
        want = torch.from_numpy(gold[f"{case}.{key}"])
        err = (got.double() - want.double()).abs().max().item()
        assert err <= GOLDEN_REL_TOL * want.abs().max().item(), (case, key, err)
    want = torch.from_numpy(gold[f"{case}.grad"])
    assert want.abs().max() > 0
    err = (grad.double() - want.double()).abs().max().item()
    assert err <= GRAD_REL_TOL * want.abs().max().item(), (case, "grad", err)

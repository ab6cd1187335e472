"""CPU: the foot-contact restatement (oracle/foot_contact_oracle.py) against the reference-driven fixtures, its limits
(no contact, no valid pair of frames, a label exactly at 0.5), finite differences, the constancy of the contact labels,
one guided update lowering the loss, and the validation that raises before any launch."""
import numpy as np
import pytest
import torch

import condmdi_b200 as C
from oracle import condmdi_oracle as O
from oracle import foot_contact_oracle as FC
from oracle import make_golden_foot_contact as MG
from oracle.golden_io import load_golden


def _case(B=2, L=9, seed=3, abs_3d=True):
    mean, std, x0, g = FC.inputs(B, L, seed=seed)
    return x0.double(), mean.double(), std.double(), abs_3d


@pytest.mark.parametrize("abs_3d", [True, False], ids=["abs3d", "rel"])
def test_contact_seed_matches_finite_differences(abs_3d):
    x0, mean, std, _ = _case(abs_3d=abs_3d)
    valid = torch.ones(2, 9, dtype=torch.bool)
    valid[1, 7:] = False
    assert FC.contact_weights(x0, mean, std, valid).sum() > 0
    grad = FC.contact_seed(x0, mean, std, abs_3d, valid)
    assert (grad[:, 67:] == 0).all()
    eps = 1e-6
    # heading, root, and the local coordinates of joints 7, 10, 8 and 11 (channels 4 + 3 (j - 1) ..)
    for idx in [(0, 0, 0, 2), (1, 1, 0, 0), (0, 2, 0, 5), (1, 3, 0, 4), (0, 22, 0, 3), (1, 31, 0, 1), (0, 25, 0, 6),
                (1, 34, 0, 7), (0, 23, 0, 8)]:
        xp, xm = x0.clone(), x0.clone()
        xp[idx] += eps
        xm[idx] -= eps
        fd = (FC.contact_loss(xp, mean, std, abs_3d, valid) - FC.contact_loss(xm, mean, std, abs_3d, valid)) / (2 * eps)
        assert abs(fd.item() - grad[idx].item()) <= 1e-5 * max(1.0, abs(fd.item())), (idx, fd.item(), grad[idx].item())


@pytest.mark.parametrize("abs_3d", [True, False], ids=["abs3d", "rel"])
def test_zero_without_contacts_or_valid_pairs(abs_3d):
    x0, mean, std, _ = _case(abs_3d=abs_3d)
    # no label above 0.5: every contact channel de-normalises to at most 0.5 (exactly 0.5 is not a contact)
    for label in (-3.0, 0.5):
        m2, x2 = mean.clone(), x0.clone()
        m2[259:263] = label
        x2[:, 259:263] = 0.0
        assert FC.contact_loss(x2, m2, std, abs_3d).item() == 0.0
        assert (FC.contact_seed(x2, m2, std, abs_3d) == 0).all()
    # no two consecutive valid frames
    alternate = (torch.arange(9) % 2 == 0).expand(2, 9)
    assert FC.contact_loss(x0, mean, std, abs_3d, alternate).item() == 0.0
    assert (FC.contact_seed(x0, mean, std, abs_3d, alternate) == 0).all()
    # one frame: no pair at all
    assert FC.contact_loss(x0[..., :1], mean, std, abs_3d).item() == 0.0


def test_contact_labels_carry_no_gradient():
    x0, mean, std, abs_3d = _case()
    z = x0.clone().requires_grad_(True)
    w = FC.contact_weights(z, mean, std, None)
    assert not w.requires_grad
    grad = FC.contact_seed(x0, mean, std, abs_3d)
    assert (grad[:, 259:263] == 0).all() and grad.abs().max() > 0
    # moving a label across 0.5 changes which displacements count, not the gradient's form: it equals autograd's with
    # the weights frozen beforehand
    with torch.enable_grad():
        z = x0.clone().requires_grad_(True)
        P = FC.J.joint_positions(z, mean, std, abs_3d)[:, :, list(FC.FOOT_JOINTS)]
        frozen = ((P[:, 1:] - P[:, :-1]).square().sum(-1) * FC.contact_weights(x0, mean, std, None)).sum()
        assert torch.equal(torch.autograd.grad(frozen, z)[0], grad)


@pytest.mark.parametrize("abs_3d", [True, False], ids=["abs3d", "rel"])
def test_small_update_lowers_the_loss(abs_3d):
    x0, mean, std, _ = _case(B=3, L=40, seed=8, abs_3d=abs_3d)
    before = FC.contact_loss(x0, mean, std, abs_3d)
    grad = FC.contact_seed(x0, mean, std, abs_3d)
    c_c = 1e-3 / grad.abs().max().item()
    after = FC.contact_loss(x0 - c_c * grad, mean, std, abs_3d)
    assert before > 0 and after < before, (before.item(), after.item())


class _Inner(torch.nn.Module):
    """just enough of a model for GaussianDiffusion._run to reach its validation"""
    cond_mode = "no_cond"

    def __init__(self):
        super().__init__()
        self.w = torch.nn.Parameter(torch.zeros(1))

    def engine_for(self, *args, **kwargs):
        raise AssertionError("validation must raise before the engine is created")


def _y(B=2, L=196):
    return {"mask": torch.ones(B, 1, 1, L, dtype=torch.bool), "foot_contact_guidance": True, "foot_contact_weight": 1.0,
            "foot_contact_gradient_schedule": None, "stop_footcontact_at": 0, "diffusion_steps": 1000}


RESOLVE = C.diffusion.resolve_model
SPACE = C.JointSpace(np.zeros(263), np.ones(263), abs_3d=True)


@pytest.mark.parametrize("case,exc,match", [
    ("no_space", NotImplementedError, "joint_space"),
    ("not_a_space", TypeError, "JointSpace"),
    ("D251", NotImplementedError, "263"),
    ("window", NotImplementedError, "windows"),
    ("weight", ValueError, "foot_contact_weight"),
    ("stop", ValueError, "stop_footcontact_at"),
    ("missing", ValueError, "foot_contact_weight"),
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
        y["foot_contact_weight"] = "1"
    elif case == "stop":
        y["stop_footcontact_at"] = 2.5
    elif case == "missing":
        del y["foot_contact_weight"]
    elif case == "mask_shape":
        y["mask"] = torch.ones(2, 1, 1, 100, dtype=torch.bool)
    C.diffusion.resolve_model = lambda m: (m, False)
    try:
        with pytest.raises(exc, match=match):
            d.ddim_sample_loop(_Inner(), shape, model_kwargs={"y": y}, device="cpu")
    finally:
        C.diffusion.resolve_model = RESOLVE


def test_random_projection_cards_are_refused():
    with pytest.raises(NotImplementedError, match="inv_proj"):
        C.JointSpace(np.zeros(263), np.ones(263), inv_proj=torch.eye(263))


# ---------------------------------------------------------------------------------------------------------------------
# the restated guided evaluation against tests/golden/foot_contact.* (the reference's model call, CFG wrapper and
# recover_from_ric under autograd, oracle/make_golden_foot_contact.py)
# ---------------------------------------------------------------------------------------------------------------------
# the gate of the joint-guidance fixtures.  Measured when the fixtures were written: max |restatement - reference| /
# max |pred_xstart| <= 1.9e-6 for the transformer (its summation order and qrot's operation order differ from the
# restatement's), 7.0e-8 for MDM_UNET in fp32 and 1.5e-6 under CPU fp16 autocast (the seed's rounding differences pass
# through the fp16 backward)
GOLDEN_REL_TOL = 2e-5


@pytest.mark.parametrize("case", [c[0] for c in MG.CASES])
def test_restated_update_equals_the_reference_driven_fixture(case, golden_dir):
    gold = load_golden(golden_dir, "foot_contact")
    _, which, t, abs_3d, keyframes, joint, autocast = next(c for c in MG.CASES if c[0] == case)
    gi = O.golden_inputs()
    assert np.allclose(gold["inputs.checksum"], [float(gi["x"].double().sum()),
                                                 float(MG.terms(True, False)[0].mean.double().sum())])
    sd = O.random_state_dict(seed=7, text=True) if which == "trans" else O.random_unet_state_dict(seed=11, text=True)
    fc, j = MG.terms(abs_3d, joint)
    pred, mean = MG.run_oracle(sd, gi, t, fc, j, keyframes, which == "unet", autocast)
    for key, got in (("pred_xstart", pred), ("mean", mean)):
        want = torch.from_numpy(gold[f"{case}.{key}"])
        err = (got.double() - want.double()).abs().max().item()
        assert err <= GOLDEN_REL_TOL * want.abs().max().item(), (case, key, err)

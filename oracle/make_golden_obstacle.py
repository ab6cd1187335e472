"""TEST INFRASTRUCTURE -- anchors the obstacle-avoidance restatement (oracle/obstacle_oracle.py) to the UNMODIFIED
reference and writes tests/golden/obstacle.*.

Run in the build container (needs the reference tree):   python -m oracle.make_golden_obstacle

The fixtures come from the reference's own guidance class, sample/gmd/condition.py's CondKeyLocationsWithSdf.__call__,
fed with its model's pred_xstart under autograd (MDM / MDM_UNET wrapped in its ClassifierFreeSampleModel).  The class's
collision term is isolated from its key-location term: the latter is an L1 loss (use_mse_loss=False) against a target
whose one masked entry is the pelvis position recover_from_ric gives on the same input, so its residual and gradient are
exactly zero (a call with obs_list=[] is asserted to return exact zeros).  motion_length_cut = L / 20 cuts nothing,
y['traj_model'] = False, inv_transform de-normalises with the statistics, and classifiler_scale = w_colli = 1, so the
class returns -dL_o/dx.  One guided evaluation (p_mean_variance's pred_xstart and mean, x0_tilde = x0_hat - c_o dL_o/dz)
per case, on golden_inputs() with full masks (the reference has none) and obstacles shared by the batch (GMD's obs_list)
placed on the pelvis paths of x0_hat, one of them a radius-0 row:
  - the transformer, CFG 2.5, t = 500, in the abs_3d and the relative representation;
  - the keyframe-conditioned MDM_UNET xl with CFG 2.5, abs_3d, t = 500, in fp32 and under CPU fp16 autocast (the model
    call inside torch.autocast("cpu", float16), the loss outside it).
It asserts that the restatement agrees and stores the REFERENCE-driven outputs and gradients with the measured gaps.
Per-sample obstacles, other joint sets and ragged masks (which the reference cannot express) are pinned against fp64
autograd of the restatement in tests/test_obstacle_oracle.py and tests/test_gpu_obstacle.py.
"""
from __future__ import annotations

import contextlib
import os
import sys
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import condmdi_oracle as O  # noqa: E402
from oracle import joint_guidance_oracle as J  # noqa: E402
from oracle import obstacle_oracle as OB  # noqa: E402
from oracle import reference_harness as RH  # noqa: E402
from oracle.golden_io import save_golden  # noqa: E402
from oracle.make_golden import GOLDEN, ref_model_with  # noqa: E402
from oracle.make_golden_unet_guidance import cpu_autocast, model_calls_under  # noqa: E402

B, D, L = 2, 263, 196
WEIGHT = 200.0
# (name, model, t, abs_3d, autocast)
CASES = [("trans.abs.t500", "trans", 500, True, False),
         ("trans.rel.t500", "trans", 500, False, False),
         ("unet.fp32.t500", "unet", 500, True, False),
         ("unet.fp16.t500", "unet", 500, True, True)]


def golden_inputs():
    """condmdi_oracle.golden_inputs with every frame valid"""
    gi = O.golden_inputs()
    gi["lengths"] = torch.tensor([L, L])
    gi["y_mask"] = torch.ones(B, 1, 1, L, dtype=torch.bool)
    return gi


def statistics():
    mean, std, _, _, _ = J.inputs(B, L, seed=9)
    return mean, std


def conditioning(gi, unet):
    obs = dict(obs_x0=gi["x_obs"], obs_mask=gi["kf_mask"]) if unet else {}
    return O.Conditioning(cond_emb=gi["cond"], cfg=True, text_scale=gi["text_scale"], y_mask=gi["y_mask"], **obs)


def obs_list_near(hat, mean, std, abs_3d):
    """GMD's obs_list: two obstacles on each sample's pelvis path of hat, and a radius-0 row"""
    near = OB.obstacles_near(hat.detach().float(), mean, std, abs_3d, 2, (0,), torch.Generator().manual_seed(21))
    rows = [((float(o[0]), float(o[1])), float(o[2])) for o in near.reshape(-1, 3)]
    return rows + [((rows[0][0][0] + 0.25, rows[0][0][1]), 0.0)]


def import_condition():
    """sample.gmd.condition with stub matplotlib modules (the class never plots; matplotlib need not be installed)"""
    RH.import_reference()
    if "matplotlib" not in sys.modules:
        mpl = types.ModuleType("matplotlib")
        plt = types.ModuleType("matplotlib.pyplot")
        patches = types.ModuleType("matplotlib.patches")
        patches.Circle = type("Circle", (), {})
        mpl.pyplot, mpl.patches = plt, patches
        sys.modules.update({"matplotlib": mpl, "matplotlib.pyplot": plt, "matplotlib.patches": patches})
    from sample.gmd import condition  # noqa: E402
    return condition


def run_reference(condition, ref_fk, model, gi, t, abs_3d, unet, autocast):
    """the reference's model call and CondKeyLocationsWithSdf under autograd; the restated update"""
    tab = O.make_tables("")
    tt = torch.tensor([t, t])
    y = {"text": ["a", "b"], "text_scale": gi["text_scale"], "mask": gi["y_mask"], "lengths": gi["lengths"],
         "traj_model": False}
    extra = {"obs_x0": gi["x_obs"], "obs_mask": gi["kf_mask"]} if unet else {}
    mean, std = statistics()
    inv = lambda x, traject_only=False, use_rand_proj=False: x * std + mean  # noqa: E731
    z = gi["x"].detach().clone().requires_grad_(True)

    def forward():
        with cpu_autocast() if autocast else contextlib.nullcontext():
            return model(z, tt, y=y, **extra).float()

    with torch.enable_grad():
        hat = forward()
        pelvis = ref_fk(inv(hat.permute(0, 2, 3, 1)), 22, abs_3d=abs_3d)[:, 0, :, 0].detach()   # (B, L, 3)
        target = torch.zeros(B, L, 22, 3)
        target_mask = torch.zeros(B, L, 22, 3, dtype=torch.bool)
        target[0, 40, 0] = pelvis[0, 40]
        target_mask[0, 40, 0, 0] = True
        obs_list = obs_list_near(hat, mean, std, abs_3d)

        def call(obs):
            cond = condition.CondKeyLocationsWithSdf(target=target, target_mask=target_mask, inv_transform=inv, abs_3d=abs_3d,
                                                     classifiler_scale=1.0, use_mse_loss=False, motion_length_cut=L / 20,
                                                     obs_list=obs, w_colli=1.0)
            return cond(z, tt, {"pred_xstart": forward()}, y=y)   # a fresh graph per call

        zero = call([])
        assert torch.equal(zero, torch.zeros_like(zero)), "the key-location term is not exactly zero"
        g_o = -call(obs_list)                                                 # dL_o/dz, classifiler_scale = w_colli = 1
    co = J._coef(None, 1000, WEIGHT, tab, tt, z.shape, z.device)
    hat = hat.detach()
    pred = hat - co * g_o
    pmean = O.extract(tab.posterior_mean_coef1, tt, z.shape) * pred + O.extract(tab.posterior_mean_coef2, tt, z.shape) * gi["x"]
    return pred, pmean, g_o, OB.obstacles_from_list(obs_list, B)


def oracle_term(obstacles, abs_3d):
    mean, std = statistics()
    return OB.ObstacleTerm(mean, std, obstacles, (0,), abs_3d, WEIGHT)


def run_oracle(sd, gi, t, ob, unet, autocast):
    """the restatement's guided evaluation (pred_xstart, mean) and its dL_o/dz"""
    c = conditioning(gi, unet)
    tt = torch.tensor([t, t])
    with model_calls_under(cpu_autocast if autocast else None):
        out = OB.p_mean_variance(sd, O.make_tables(""), gi["x"], tt, c, ob)
        with torch.enable_grad():
            z = gi["x"].detach().clone().requires_grad_(True)
            hat = O._model(sd, z, torch.tensor(O.make_tables("").timestep_map)[tt], c)
            g = torch.autograd.grad(OB.obstacle_loss(hat.float(), ob.mean, ob.std, ob.abs_3d, ob.obstacles, ob.joints,
                                                     c.y_mask), z)[0]
    return out["pred_xstart"].detach(), out["mean"].detach(), g


def golden_obstacle():
    ref = RH.import_reference()
    condition = import_condition()
    from data_loaders.humanml.scripts.motion_process import recover_from_ric as ref_fk  # noqa: E402
    gi = golden_inputs()
    sdt = O.random_state_dict(seed=7, text=True)
    mt = ref_model_with(sdt, text=True)
    mt._synthetic_text_emb = gi["cond"]
    sdu = O.random_unet_state_dict(seed=11, text=True)
    mu = RH.build_reference_unet(text=True)
    missing, unexpected = mu.load_state_dict(sdu, strict=False)
    assert not missing and not unexpected, (missing, unexpected)
    mu._synthetic_text_emb = gi["cond"]
    models = {"trans": (ref.cfg_sampler.ClassifierFreeSampleModel(mt), sdt),
              "unet": (ref.cfg_sampler.ClassifierFreeSampleModel(mu), sdu)}
    out = {"inputs.checksum": np.array([float(gi["x"].double().sum()), float(statistics()[0].double().sum())])}
    for name, which, t, abs_3d, autocast in CASES:
        model, sd = models[which]
        pred, mean, g_o, obstacles = run_reference(condition, ref_fk, model, gi, t, abs_3d, which == "unet", autocast)
        o_pred, o_mean, o_g = run_oracle(sd, gi, t, oracle_term(obstacles, abs_3d), which == "unet", autocast)
        err = max((pred - o_pred).abs().max().item(), (mean - o_mean).abs().max().item())
        g_err = (g_o - o_g).abs().max().item()
        scale, g_scale = pred.abs().max().item(), g_o.abs().max().item()
        print(f"  {name:16s} max |dL_o/dz| {g_scale:.3e}  gradient gap {g_err:.3e}  update gap {err:.3e} "
              f"(max |pred_xstart| {scale:.3e})")
        assert g_scale > 0, f"{name}: no joint enters an obstacle"
        assert g_err <= 1e-3 * g_scale, f"{name}: the restated gradient differs from the reference's by {g_err:.3e}"
        assert err <= 1e-4 * max(1.0, scale), f"{name}: the restatement differs from the reference by {err:.3e}"
        out[f"{name}.obstacles"] = obstacles.numpy()
        out[f"{name}.grad"] = g_o.numpy()
        out[f"{name}.pred_xstart"] = pred.numpy()
        out[f"{name}.mean"] = mean.numpy()
        out[f"{name}.err"] = np.array([err, g_err])
    save_golden(GOLDEN, "obstacle", **out)


def main():
    if not RH.available():
        raise SystemExit("the reference tree is required to (re)generate golden vectors")
    os.makedirs(GOLDEN, exist_ok=True)
    torch.set_num_threads(os.cpu_count() or 1)
    golden_obstacle()
    for f in sorted(os.listdir(GOLDEN)):
        if f.startswith("obstacle."):
            print(f, os.path.getsize(os.path.join(GOLDEN, f)) // 1024, "KiB")


if __name__ == "__main__":
    main()

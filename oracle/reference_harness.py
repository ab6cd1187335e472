"""TEST INFRASTRUCTURE -- imports the UNMODIFIED reference (setarehc/diffusion-motion-inbetweening) on CPU.

Only usable where /root/reference exists (the build container).  It is how the oracle restatement in
`oracle/condmdi_oracle.py` is pinned and how the fixtures under tests/golden/ are generated
(`oracle/make_golden.py`).  Nothing on the product path, the -m gpu tests, smoke() or bench.py imports it.

The reference files are not modified; the shims below are applied before import (SURVEY.md section 8c):
  * numpy aliases removed in numpy>=1.24 that the reference uses at import time
      (data_loaders/humanml/common/quaternion.py:13, data_loaders/humanml_utils.py:68-88)
  * `clip`, `smplx` stubs (model/mdm.py:6, model/smpl.py:7-8) -- neither is installed nor on this path
  * model.smpl.SMPL replaced by an empty nn.Module (MDM.__init__ builds Rotation2xyz, mdm.py:165)
  * noise tape: torch.randn / torch.randn_like read successive slices of a pre-generated tensor, because the
      loop draws from the global generator (gaussian_diffusion.py:696, :1248, :1407) and has no other hook.
"""
from __future__ import annotations

import contextlib
import os
import sys
import types

import numpy as np
import torch

REFERENCE_ROOT = os.environ.get("CONDMDI_REFERENCE_ROOT", "/root/reference")


def available() -> bool:
    return os.path.isdir(os.path.join(REFERENCE_ROOT, "diffusion"))


_imported = {}


def import_reference():
    """Returns a namespace with the reference modules of the hot path."""
    if _imported:
        return types.SimpleNamespace(**_imported)
    if not available():
        raise RuntimeError(f"reference tree not found at {REFERENCE_ROOT}")
    for alias, typ in (("float", float), ("bool", bool), ("int", int), ("object", object)):
        if not hasattr(np, alias):
            setattr(np, alias, typ)
    # stubs for packages that are not installed and not on the path being tested
    clip = types.ModuleType("clip")
    clip.load = lambda *a, **k: (torch.nn.Identity(), None)
    clip.tokenize = lambda *a, **k: torch.zeros(1, 77, dtype=torch.long)
    clip.model = types.SimpleNamespace(convert_weights=lambda m: None)
    sys.modules.setdefault("clip", clip)
    smplx = types.ModuleType("smplx")
    smplx.SMPLLayer = torch.nn.Module
    smplx_lbs = types.ModuleType("smplx.lbs")
    smplx_lbs.vertices2joints = lambda *a, **k: None
    sys.modules.setdefault("smplx", smplx)
    sys.modules.setdefault("smplx.lbs", smplx_lbs)
    if REFERENCE_ROOT not in sys.path:
        sys.path.insert(0, REFERENCE_ROOT)
    import model.smpl as ref_smpl  # noqa: E402

    class _NoSMPL(torch.nn.Module):
        def __init__(self, *a, **k):
            super().__init__()

    ref_smpl.SMPL = _NoSMPL
    import model.rotation2xyz as ref_rot  # noqa: E402

    ref_rot.SMPL = _NoSMPL
    import diffusion.gaussian_diffusion as gd  # noqa: E402
    import diffusion.respace as respace  # noqa: E402
    import model.cfg_sampler as cfg_sampler  # noqa: E402
    import model.mdm as mdm  # noqa: E402
    import utils.editing_util as editing_util  # noqa: E402

    _imported.update(gd=gd, respace=respace, mdm=mdm, cfg_sampler=cfg_sampler, editing_util=editing_util)
    return types.SimpleNamespace(**_imported)


def build_reference_model(seed: int = 0, text: bool = False, layers: int = 8, latent_dim: int = 512, ff_size: int = 1024,
                          njoints: int = 263):
    """Random-init MDM exactly as utils/model_util.py:86-119 configures it for humanml / trans_enc."""
    ref = import_reference()
    torch.manual_seed(seed)
    with contextlib.redirect_stdout(open(os.devnull, "w")):
        model = ref.mdm.MDM(modeltype="", njoints=njoints, nfeats=1, num_actions=1, translation=True, pose_rep="rot6d",
                            glob=True, glob_rot=True, latent_dim=latent_dim, ff_size=ff_size, num_layers=layers,
                            num_heads=4, dropout=0.1, activation="gelu", data_rep="hml_vec", cond_mode="no_cond",
                            cond_mask_prob=0.1, action_emb="tensor", arch="trans_enc", emb_trans_dec=False,
                            clip_version="ViT-B/32", dataset="humanml")
    if text:
        # cond_mode='text' without CLIP: a seeded embed_text layer and a synthetic, injectable encode_text
        model.cond_mode = "text"
        model.embed_text = torch.nn.Linear(512, latent_dim)
        model._synthetic_text_emb = None
        model.encode_text = lambda raw_text: model._synthetic_text_emb
    model.keyframe_conditioned = False  # SURVEY.md 8(b) note 1: read by cfg_sampler.py:20, never set by MDM
    model.eval()
    return model


def build_reference_unet(dim_mults=(2, 2, 2, 2), latent_dim: int = 512, keyframe_conditioned: bool = True, text: bool = False,
                         njoints: int = 263, dataset: str = "humanml"):
    """MDM_UNET as utils/model_util.py:30-32 builds it for configs/model.py `motion_unet_adagn_xl` (arch='unet', adagn, zero).
    njoints / dataset as utils/model_util.py:62-76 sets them (263 humanml, 251 kit, 764 amass)."""
    import_reference()
    import model.mdm_unet as ref_unet  # noqa: E402
    with contextlib.redirect_stdout(open(os.devnull, "w")):
        model = ref_unet.MDM_UNET(modeltype="", njoints=njoints, nfeats=1, num_actions=1, translation=True, pose_rep="rot6d",
                                  glob=True, glob_rot=True, latent_dim=latent_dim, dim_mults=tuple(dim_mults), data_rep="hml_vec",
                                  dataset=dataset, cond_mode="no_cond", cond_mask_prob=0.1, adagn=True, zero=True, arch="unet",
                                  keyframe_conditioned=keyframe_conditioned)
    if text:
        model.cond_mode = "text"
        model.embed_text = torch.nn.Linear(512, latent_dim)
        model._synthetic_text_emb = None
        model.encode_text = lambda raw_text: model._synthetic_text_emb
    model.eval()
    return model


def build_reference_diffusion(respacing: str = "", steps: int = 1000):
    """utils/model_util.py:122-165 with noise_schedule='cosine', sigma_small, predict_xstart."""
    ref = import_reference()
    gd, respace = ref.gd, ref.respace
    betas = gd.get_named_beta_schedule("cosine", steps, 1.0)
    use = respace.space_timesteps(steps, respacing if respacing else [steps])
    return respace.SpacedDiffusion(
        use_timesteps=use,
        conf=gd.DiffusionConfig(betas=betas, model_mean_type=gd.ModelMeanType.START_X,
                                model_var_type=gd.ModelVarType.FIXED_SMALL, loss_type=gd.LossType.MSE,
                                rescale_timesteps=False))


@contextlib.contextmanager
def noise_tape(tape: torch.Tensor):
    """Patch torch.randn / torch.randn_like so the k-th draw of the sampling loop returns tape[k]."""
    state = {"k": 0}
    real_randn, real_randn_like = torch.randn, torch.randn_like

    def take(shape):
        t = tape[state["k"]]
        assert tuple(t.shape) == tuple(shape), (t.shape, shape)
        state["k"] += 1
        return t.clone()

    def fake_randn(*shape, **kw):
        if len(shape) == 1 and isinstance(shape[0], (tuple, list, torch.Size)):
            shape = tuple(shape[0])
        return take(shape)

    def fake_randn_like(x, **kw):
        return take(x.shape)

    torch.randn, torch.randn_like = fake_randn, fake_randn_like
    try:
        yield state
    finally:
        torch.randn, torch.randn_like = real_randn, real_randn_like

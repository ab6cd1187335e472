"""condmdi_b200: H100-native sampling engine for CondMDI (setarehc/diffusion-motion-inbetweening).

The directory name follows the repository convention (`diffusion-motion-inbetweening_b200/`); it is imported
as `condmdi_b200` through the shim package next to it.
"""
from . import capi  # noqa: F401
from .diffusion import (DiffusionConfig, GaussianDiffusion, ModelMeanType, ModelVarType, SpacedDiffusion,  # noqa: F401
                        JointSpace, Window, create_gaussian_diffusion, from_reference_diffusion, get_named_beta_schedule, space_timesteps)
from .editing_util import get_gradient_schedule, get_keyframes_mask, joint_to_full_mask  # noqa: F401
from .engine import Engine  # noqa: F401
from .model import MDM, MDM_UNET, ClassifierFreeSampleModel, KeyframeClassifierFreeSampleModel, resolve_model  # noqa: F401
from .adapter import accelerate, install  # noqa: F401
from .distributed import sharded_sample  # noqa: F401
from .eval_loop import EvalJob, build_jobs, run_eval_jobs  # noqa: F401

from .capi import PRECISION_BF16, PRECISION_BF16X3, PRECISION_FP16  # noqa: F401

__version__ = "0.1.0"
from .motion_process import abs3d_to_rel, joints_to_features, recover_from_ric, rel_to_abs3d, sample_to_joints  # noqa: F401

"""Putting the engine under the reference's own objects (the drop-in boundary, SURVEY.md 8(b)).

    import condmdi_b200
    model, diffusion = create_model_and_diffusion(args, data)      # reference code, unchanged
    ...
    diffusion = condmdi_b200.accelerate(diffusion)                 # <- the one added line
    sample = diffusion.p_sample_loop(model, (B, 263, 1, 196), model_kwargs=model_kwargs, ...)

`accelerate` returns an engine-backed sampler exposing the same methods/attributes; `install` patches the
reference object in place instead (for call sites that keep their own reference to it).
"""
from __future__ import annotations

import types

from .diffusion import GaussianDiffusion, from_reference_diffusion

_LOOPS = ("p_sample_loop", "p_sample_loop_progressive", "ddim_sample_loop", "ddim_sample_loop_progressive",
          "plms_sample_loop", "plms_sample_loop_progressive")
# loops the reference lacks: DDIM inversion (it has the step, ddim_reverse_sample, which install() leaves as it is) and
# the DPM-Solver++, UniPC and SDE-DPM-Solver++ multistep samplers
_ADDED_LOOPS = ("ddim_reverse_sample_loop", "ddim_reverse_sample_loop_progressive", "dpm_solver_sample_loop",
                "dpm_solver_sample_loop_progressive", "unipc_sample_loop", "unipc_sample_loop_progressive",
                "dpm_solver_sde_sample_loop", "dpm_solver_sde_sample_loop_progressive")


def accelerate(ref_diffusion):
    """Engine-backed sampler equivalent to a reference GaussianDiffusion / SpacedDiffusion instance."""
    if isinstance(ref_diffusion, GaussianDiffusion):
        return ref_diffusion
    return from_reference_diffusion(ref_diffusion)


def install(ref_diffusion, fallback_to_reference: bool = False):
    """Replace the six sampling loops (DDPM, DDIM, PLMS and their progressive forms) of a reference diffusion object by
    the engine's, in place, and add the engine's DDIM inversion loops (ddim_reverse_sample_loop[_progressive]),
    DPM-Solver++ loops (dpm_solver_sample_loop[_progressive]), UniPC loops (unipc_sample_loop[_progressive]) and
    SDE-DPM-Solver++ loops (dpm_solver_sde_sample_loop[_progressive]).

    Configurations the engine does not implement raise NotImplementedError.  With fallback_to_reference=True those
    (and only those) are forwarded to the reference's original PyTorch loop instead -- an explicit opt-in for
    scripts that mix accelerated and non-accelerated features, never a silent CPU/eager path.
    """
    fast = from_reference_diffusion(ref_diffusion)
    ref_diffusion._condmdi_b200 = fast
    for name in _LOOPS + _ADDED_LOOPS:
        original = getattr(ref_diffusion, name, None)  # None: an object without this loop gains the engine's

        def make(name=name, original=original):
            def loop(self, *args, **kwargs):
                try:
                    # (the *_progressive loops validate their configuration when CALLED and return the step
                    # generator, so an unsupported configuration surfaces inside this try block too)
                    return getattr(fast, name)(*args, **kwargs)
                except NotImplementedError:
                    if fallback_to_reference and original is not None:
                        return original(*args, **kwargs)
                    raise
            return loop

        setattr(ref_diffusion, name, types.MethodType(make(), ref_diffusion))
    return ref_diffusion

"""TEST INFRASTRUCTURE -- shows that the MDM_UNET restatement (condmdi_oracle.unet_forward) puts autocast's casts where the
UNMODIFIED reference's MDM_UNET does, and writes tests/golden/unet_autocast.* from the reference's outputs.

Run in the build container (needs the reference tree):   python -m oracle.make_golden_unet_autocast

The GPU tests of CMDI_PRECISION_FP16 (tests/test_gpu_unet_fp16.py) take unet_forward under torch.autocast("cuda", float16)
as the stand-in for the reference's own GPU run.  That is valid when the restatement calls the same operators on the same
dtypes in the same order, so that every autocast cast falls in the same place.  Here, on the CPU, the reference and the
restatement run under CPU autocast (bfloat16, and float16 where this torch build supports it) and must agree BIT FOR BIT:
the xl geometry (configs/model.py `motion_unet_adagn_xl`) with keyframe input conditioning (text, unconditional, CFG) and
the same geometry without it.  CPU autocast's op lists are not CUDA's (GroupNorm, for one, runs in the low precision there),
so this pins where the casts fall, not what CUDA computes (DESIGN.md section 2).
"""
from __future__ import annotations

import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import condmdi_oracle as O  # noqa: E402
from oracle import reference_harness as RH  # noqa: E402
from oracle.golden_io import save_golden  # noqa: E402
from oracle.make_golden import GOLDEN  # noqa: E402

DTYPES = {"bf16": torch.bfloat16, "fp16": torch.float16}


def cpu_autocast_dtypes():
    """The low-precision dtypes CPU autocast accepts in this torch build (float16 is newer than bfloat16 there)."""
    usable = []
    for name, dt in DTYPES.items():
        try:
            with torch.autocast("cpu", dtype=dt):
                y = torch.nn.functional.linear(torch.ones(2, 4), torch.ones(3, 4))
            if y.dtype == dt:
                usable.append(name)
        except (RuntimeError, AssertionError) as ex:
            print(f"CPU autocast with {name}: not usable here ({ex})")
    return usable


def cases():
    """(name, reference model, state dict, call kwargs) of every checked evaluation."""
    gi = O.golden_inputs()
    x, cond, x_obs, scale, kf_mask = (gi[k] for k in ("x", "cond", "x_obs", "text_scale", "kf_mask"))
    t = torch.tensor([999, 37])
    out = []
    for kf in (True, False):
        sd = O.random_unet_state_dict(seed=11, text=True, keyframe_conditioned=kf)
        m = RH.build_reference_unet(text=True, keyframe_conditioned=kf)
        missing, unexpected = m.load_state_dict(sd, strict=False)
        assert not missing and not unexpected, (missing, unexpected)
        m._synthetic_text_emb = cond
        obs = {"obs_x0": x_obs, "obs_mask": kf_mask} if kf else {}
        tag = "kf" if kf else "nokf"
        out.append((f"{tag}.text", m, sd, dict(x=x, t=t, cond=cond, uncond=False, cfg=False, **obs)))
        out.append((f"{tag}.uncond", m, sd, dict(x=x, t=t, cond=cond, uncond=True, cfg=False, **obs)))
        out.append((f"{tag}.cfg", m, sd, dict(x=x, t=torch.tensor([500, 500]), cond=cond, uncond=False, cfg=True, scale=scale, **obs)))
    return out


def run_reference(ref, m, kw):
    y = {"text": ["a", "b"]}
    obs = {k: kw[k] for k in ("obs_x0", "obs_mask") if k in kw}
    if kw["cfg"]:
        return ref.cfg_sampler.ClassifierFreeSampleModel(m)(kw["x"], kw["t"], y=dict(y, text_scale=kw["scale"]), **obs)
    return m(kw["x"], kw["t"], y=dict(y, uncond=True) if kw["uncond"] else y, **obs)


def run_oracle(sd, kw):
    if kw["cfg"]:
        c = O.Conditioning(cond_emb=kw["cond"], cfg=True, text_scale=kw["scale"], obs_x0=kw.get("obs_x0"), obs_mask=kw.get("obs_mask"))
        return O._model(sd, kw["x"], kw["t"], c)
    return O.unet_forward(sd, kw["x"], kw["t"], kw["cond"], kw["uncond"], kw.get("obs_x0"), kw.get("obs_mask"))


def golden_unet_autocast():
    ref = RH.import_reference()
    out = {}
    for dname in cpu_autocast_dtypes():
        dt = DTYPES[dname]
        for name, m, sd, kw in cases():
            with torch.no_grad():
                with torch.autocast("cpu", dtype=dt):
                    r = run_reference(ref, m, kw)
                    o = run_oracle(sd, kw)
                f32 = run_oracle(sd, kw)
            assert r.dtype == torch.float32 and o.dtype == torch.float32
            gap = (r - f32).abs().max().item()
            print(f"  {dname} {name:12s} reference == restatement: {torch.equal(r, o)}   max |autocast - fp32| = {gap:.3e}")
            assert torch.equal(r, o), f"{dname} {name}: the restatement's casts differ from the reference's"
            assert gap > 0, f"{dname} {name}: autocast changed nothing"
            out[f"{dname}.{name}"] = r.numpy()
    save_golden(GOLDEN, "unet_autocast", **out)


def main():
    if not RH.available():
        raise SystemExit("the reference tree is required to (re)generate golden vectors")
    os.makedirs(GOLDEN, exist_ok=True)
    torch.set_num_threads(os.cpu_count() or 1)
    golden_unet_autocast()
    for f in sorted(os.listdir(GOLDEN)):
        if f.startswith("unet_autocast."):
            print(f, os.path.getsize(os.path.join(GOLDEN, f)) // 1024, "KiB")


if __name__ == "__main__":
    main()

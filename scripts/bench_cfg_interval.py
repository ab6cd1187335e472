"""Classifier-free guidance limited to an interval of steps on one GPU: whole ddim50 loops at B = 64 with guidance at every
step, at the 25 steps t = 12 .. 36 (about half), and at none, timed with CUDA events in one process, the arms
alternating round by round:
  - the transformer (8 layers, random weights) at bf16x3 with CFG (text scale 2.5);
  - the xl UNet (dim 512, dim_mults (2,2,2,2), keyframe input conditioning, text; random weights) at fp16 with keyframe
    CFG and text CFG (KeyframeClassifierFreeSampleModel, w_k = 1.5, w_t = 2.5).
A step outside the interval runs one pass of B rows instead of 2B (CFG) or 3B (keyframe CFG).

    python scripts/bench_cfg_interval.py [--batch 64] [--rounds 5] [--out DIR]

Prints the card, its power limit and max SM clock, and one JSON line: per arm the median loop time and steps/s.  Writes
nothing unless --out is given.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

import condmdi_b200 as C  # noqa: E402
from bench_unet_precision import card, timed  # noqa: E402
from oracle import condmdi_oracle as O  # noqa: E402

STEPS = 50
INTERVALS = {"every_step": None, "half": (12, 36), "none": (STEPS, STEPS)}


def with_interval(kw, iv):
    if iv is None:
        return kw
    return dict(kw, y=dict(kw["y"], stop_cfg_at=iv[0], start_cfg_at=iv[1]))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this benchmark measures the GPU and has no CPU fallback")
    B, D, L = args.batch, 263, 196
    g = torch.Generator().manual_seed(0)
    x_T = torch.randn(B, D, 1, L, generator=g).cuda()
    x_obs = torch.randn(B, D, 1, L, generator=g).cuda()
    kf = C.get_keyframes_mask(x_obs.cpu(), torch.full((B,), L), "benchmark_sparse", trans_length=5).cuda()
    cond = torch.randn(B, 512, generator=g).cuda()
    table = {str(i): cond[i] for i in range(B)}
    y = {"text": [str(i) for i in range(B)], "text_scale": torch.full((B,), 2.5).cuda(),
         "keyframe_scale": torch.full((B,), 1.5).cuda(), "mask": torch.ones(B, 1, 1, L, dtype=torch.bool).cuda()}

    mt = C.MDM(cond_mode="text", cond_mask_prob=0.1)
    mt.load_state_dict(O.random_state_dict(seed=0, text=True), strict=False)
    mt = mt.cuda()
    mt.encode_text = lambda texts: torch.stack([table[t] for t in texts])
    dt = C.create_gaussian_diffusion(timestep_respacing=f"ddim{STEPS}")
    mu = C.MDM_UNET(keyframe_conditioned=True, cond_mode="text", cond_mask_prob=0.1)
    mu.load_state_dict(O.random_unet_state_dict(seed=0, text=True), strict=False)
    mu = mu.cuda()
    mu.encode_text = lambda texts: torch.stack([table[t] for t in texts])
    du = C.create_gaussian_diffusion(timestep_respacing=f"ddim{STEPS}")
    du.precision = C.PRECISION_FP16
    models = {"transformer_bf16x3_cfg": (dt, C.ClassifierFreeSampleModel(mt), {"y": y}),
              "unet_xl_fp16_kf_cfg": (du, C.KeyframeClassifierFreeSampleModel(mu), {"y": y, "obs_x0": x_obs, "obs_mask": kf})}
    arms = {f"{name}.{iv_name}": (lambda d=d, w=w, kw=with_interval(kw, iv): d.ddim_sample_loop(w, (B, D, 1, L), model_kwargs=kw,
                                                                                                   noise=x_T))
            for name, (d, w, kw) in models.items() for iv_name, iv in INTERVALS.items()}
    for fn in arms.values():  # warm-up: engine creation, graph capture, module loads
        fn()
    torch.cuda.synchronize()
    times = {k: [] for k in arms}
    for _ in range(args.rounds):
        for name, fn in arms.items():
            times[name].append(timed(fn))
    res = {"card": card(), "batch": B, "schedule": f"ddim{STEPS}", "text_scale": 2.5, "keyframe_scale": 1.5,
           "intervals": {k: v for k, v in INTERVALS.items()}, "rounds": args.rounds}
    for name, tt in times.items():
        med = statistics.median(tt)
        res[name] = {"loop_ms_median": round(med, 2), "loop_ms_min": round(min(tt), 2), "loop_ms_max": round(max(tt), 2),
                     "steps_per_s": round(STEPS / (med / 1000.0), 1)}
    print(f"card: {res['card']['name']}  power limit, max SM clock: {res['card']['power_limit, max_sm_clock']}")
    print(json.dumps(res))
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_cfg_interval.json"), "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()

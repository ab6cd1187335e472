"""SDE-DPM-Solver++ order 2 against p_sample_loop at the same step count, on one GPU, in one process.

    python scripts/bench_dpm_solver_sde.py [--batch 64] [--rounds 5] [--out DIR]

Whole ddim50 loops at B = --batch of
  - the 8-layer MDM transformer (bf16x3) with CFG 2.5 and keyframe imputation, and
  - the keyframe-conditioned MDM_UNET xl at PRECISION_FP16 with CFG 2.5 and keyframe input,
for p_sample_loop and dpm_solver_sde_sample_loop(order=2), the two alternating round by round, timed with CUDA events;
medians.  Both draw their per-step noise from the engine generator.  A step of either is one denoiser pass plus one step
kernel, so the two are expected to run at the same steps/s.

Prints the card, its power limit and max SM clock, and one JSON line.  Writes nothing unless --out is given.
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
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import condmdi_b200 as C  # noqa: E402
from bench_dpm_solver import D, L, card, unet_xl  # noqa: E402
from oracle import condmdi_oracle as O  # noqa: E402

STEPS = 50


def transformer_cfg_imputation():
    m = C.MDM(cond_mode="text", cond_mask_prob=0.1)
    m.load_state_dict(O.random_state_dict(seed=0, text=True), strict=False)
    m = m.cuda()
    g = torch.Generator().manual_seed(2)
    cond = torch.randn(512, 512, generator=g).cuda()
    m.encode_text = lambda texts: cond[torch.tensor([int(t) for t in texts])]

    def kwargs(B):
        gk = torch.Generator().manual_seed(3)
        x_obs = torch.randn(B, D, 1, L, generator=gk)
        kf = C.get_keyframes_mask(x_obs, torch.full((B,), L), "benchmark_sparse", trans_length=5)
        return {"y": {"text": [str(i) for i in range(B)], "text_scale": torch.full((B,), 2.5).cuda(),
                      "mask": torch.ones(B, 1, 1, L, dtype=torch.bool).cuda(), "imputate": 1, "stop_imputation_at": 0,
                      "replacement_distribution": "conditional", "inpainted_motion": x_obs.cuda(), "inpainting_mask": kf.cuda()}}
    return C.ClassifierFreeSampleModel(m), kwargs, C.PRECISION_BF16X3


def timing(model, B, rounds):
    m, kwargs, precision = model
    d = C.create_gaussian_diffusion(timestep_respacing=f"ddim{STEPS}")
    d.precision, d.rng, d.engine_seed = precision, "engine", 1
    x_T = torch.randn(B, D, 1, L, generator=torch.Generator().manual_seed(0)).cuda()
    kw = {"model_kwargs": kwargs(B), "noise": x_T}
    shape = (B, D, 1, L)
    arms = {"p_sample_loop": lambda: d.p_sample_loop(m, shape, **kw),
            "sde_order2": lambda: d.dpm_solver_sde_sample_loop(m, shape, order=2, **kw)}
    for fn in arms.values():  # warm-up: graph capture, chained-launch tables, module loads
        fn()
    torch.cuda.synchronize()
    times = {k: [] for k in arms}
    for _ in range(rounds):
        for name, fn in arms.items():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            out = fn()
            e1.record()
            e1.synchronize()
            times[name].append(e0.elapsed_time(e1))
            assert torch.isfinite(out).all()
    res = {}
    for name, ts in times.items():
        med = statistics.median(ts)
        res[name] = {"loop_ms_median": round(med, 2), "loop_ms_min": round(min(ts), 2), "loop_ms_max": round(max(ts), 2),
                     "steps_per_s": round(STEPS / (med / 1000.0), 1)}
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this benchmark measures the GPU and has no CPU fallback")
    res = {"card": card(), "batch": args.batch, "rounds": args.rounds, "steps": STEPS}
    for name, build in (("transformer_bf16x3_cfg_imputation", transformer_cfg_imputation), ("unet_xl_fp16_cfg", unet_xl)):
        res[name] = timing(build(), args.batch, args.rounds)
    print(f"card: {res['card']['name']}  power limit, max SM clock: {res['card']['power_limit, max_sm_clock']}")
    for name in ("transformer_bf16x3_cfg_imputation", "unet_xl_fp16_cfg"):
        print(f"\n{name}: ddim{STEPS} loop at B = {args.batch}, median ms (steps/s)")
        for arm, r in res[name].items():
            print(f"  {arm:14s} {r['loop_ms_median']:9.2f} ms  ({r['steps_per_s']} steps/s)  "
                  f"min {r['loop_ms_min']:.2f}, max {r['loop_ms_max']:.2f}")
    print(json.dumps(res))
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_dpm_solver_sde.json"), "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()

"""Reconstruction guidance on MDM_UNET at fp16 ("autocast", CMDI_PRECISION_FP16) on one GPU: whole ddim50 loops of the xl
UNet (dim 512, dim_mults (2,2,2,2), keyframe input conditioning, text; random weights) at B = 64 with CFG 2.5, guided
(w = 20 on every step) against unguided, timed with CUDA events in one process, the two alternating round by round.  One
more leg times a single guided CFG evaluation of the oracle in eager PyTorch: the forward under torch.autocast("cuda",
float16) plus torch.autograd.grad, as the reference computes the guidance gradient.

    python scripts/bench_unet_guidance.py [--batch 64] [--rounds 5] [--out DIR]

Prints the card, its power limit and max SM clock, and one JSON line: per arm the median loop time and steps/s (a step is
one sampler iteration: one CFG evaluation, plus its input-VJP when guided), and the eager evaluation's median time.
Writes nothing unless --out is given.
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this benchmark measures the GPU and has no CPU fallback")
    B, D, L = args.batch, 263, 196
    sd = O.random_unet_state_dict(seed=0, text=True)
    m = C.MDM_UNET(keyframe_conditioned=True, cond_mode="text", cond_mask_prob=0.1)
    m.load_state_dict(sd, strict=False)
    m = m.cuda()
    g = torch.Generator().manual_seed(0)
    x_T = torch.randn(B, D, 1, L, generator=g).cuda()
    x_obs = torch.randn(B, D, 1, L, generator=g).cuda()
    kf = C.get_keyframes_mask(x_obs.cpu(), torch.full((B,), L), "benchmark_sparse", trans_length=5).cuda()
    cond = torch.randn(B, 512, generator=g).cuda()
    table = {str(i): cond[i] for i in range(B)}
    m.encode_text = lambda texts: torch.stack([table[t] for t in texts])
    w = C.ClassifierFreeSampleModel(m)
    y = {"text": [str(i) for i in range(B)], "text_scale": torch.full((B,), 2.5).cuda(), "mask": torch.ones(B, 1, 1, L, dtype=torch.bool).cuda()}
    yg = dict(y, reconstruction_guidance=True, reconstruction_weight=20.0, gradient_schedule=None, diffusion_steps=1000,
              stop_recguidance_at=0, inpainted_motion=x_obs, inpainting_mask=kf)
    d = C.create_gaussian_diffusion(timestep_respacing="ddim50")
    d.precision = C.PRECISION_FP16
    arms = {name: (lambda yy=yy: d.ddim_sample_loop(w, (B, D, 1, L), model_kwargs={"y": yy, "obs_x0": x_obs, "obs_mask": kf},
                                                    noise=x_T))
            for name, yy in (("fp16_unguided", y), ("fp16_guided", yg))}

    # eager PyTorch: one guided CFG evaluation, the forward under CUDA autocast and autograd.grad outside it
    sdd = {k: v.cuda() for k, v in sd.items()}
    t = torch.full((B,), 500, device="cuda")

    def eager():
        z = x_T.detach().requires_grad_(True)
        with torch.autocast("cuda", dtype=torch.float16):
            out = O.unet_forward(sdd, z, t, cond, False, x_obs, kf)
            out_u = O.unet_forward(sdd, z, t, cond, True, x_obs, kf)
            hat = out_u + 2.5 * (out - out_u)
        loss = ((x_obs - hat).square() * kf).sum()
        return torch.autograd.grad(loss, z)[0]

    for fn in list(arms.values()) + [eager] * 3:  # warm-up: graph capture, module loads, cuDNN algorithm choice
        fn()
    torch.cuda.synchronize()
    times = {k: [] for k in arms}
    eager_ms = []
    for _ in range(args.rounds):
        for name, fn in arms.items():
            times[name].append(timed(fn))
        eager_ms.append(timed(eager))
    steps = d.num_timesteps
    res = {"card": card(), "batch": B, "schedule": "ddim50", "cfg_scale": 2.5, "reconstruction_weight": 20.0, "rounds": args.rounds}
    for name, ts in times.items():
        med = statistics.median(ts)
        res[name] = {"loop_ms_median": round(med, 2), "loop_ms_min": round(min(ts), 2), "loop_ms_max": round(max(ts), 2),
                     "steps_per_s": round(steps / (med / 1000.0), 1), "ms_per_step": round(med / steps, 2)}
    res["guided_step_extra_ms"] = round(res["fp16_guided"]["ms_per_step"] - res["fp16_unguided"]["ms_per_step"], 2)
    med = statistics.median(eager_ms)
    res["eager_autocast_guided_cfg_evaluation"] = {"ms_median": round(med, 2), "ms_min": round(min(eager_ms), 2),
                                                   "per_s": round(1000.0 / med, 1)}
    print(f"card: {res['card']['name']}  power limit, max SM clock: {res['card']['power_limit, max_sm_clock']}")
    print(json.dumps(res))
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_unet_guidance.json"), "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()

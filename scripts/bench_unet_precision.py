"""MDM_UNET sampling at bf16x3 against fp16 ("autocast", CMDI_PRECISION_FP16) on one GPU: whole ddim50 loops of the xl UNet
(dim 512, dim_mults (2,2,2,2), keyframe input conditioning, text; random weights) at B = 64 with CFG 2.5, timed with CUDA
events in one process, the two precisions alternating round by round.  One more leg times a single CFG forward pass of the
oracle under torch.autocast("cuda", float16) in eager PyTorch: the reference's own GPU arithmetic.

    python scripts/bench_unet_precision.py [--batch 64] [--rounds 5] [--out DIR]

Prints the card, its power limit and max SM clock, and one JSON line: per precision the median loop time and denoising
steps/s (a step is one sampler iteration: one CFG evaluation of the denoiser, i.e. 2B sequences), and the eager
forward's median time.  Writes nothing unless --out is given.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import condmdi_b200 as C  # noqa: E402
from oracle import condmdi_oracle as O  # noqa: E402


def card() -> dict:
    info = {"name": torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30)
        info["power_limit, max_sm_clock"] = q.stdout.strip().splitlines()[0]
    except Exception as ex:  # noqa: BLE001
        info["power_limit, max_sm_clock"] = f"unavailable ({ex})"
    return info


def timed(fn) -> float:
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    out = fn()
    e1.record()
    e1.synchronize()
    assert torch.isfinite(out).all()
    return e0.elapsed_time(e1)


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
    y = {"text": [str(i) for i in range(B)], "text_scale": torch.full((B,), 2.5).cuda()}
    kw = {"model_kwargs": {"y": y, "obs_x0": x_obs, "obs_mask": kf}, "noise": x_T}
    diff = {}
    for name, prec in (("bf16x3", C.PRECISION_BF16X3), ("fp16", C.PRECISION_FP16)):
        diff[name] = C.create_gaussian_diffusion(timestep_respacing="ddim50")
        diff[name].precision = prec
    arms = {name: (lambda d=d: d.ddim_sample_loop(w, (B, D, 1, L), **kw)) for name, d in diff.items()}

    # eager PyTorch under CUDA autocast: one CFG evaluation (cond + uncond pass) of the oracle, as the reference runs it
    sdd = {k: v.cuda() for k, v in sd.items()}
    t = torch.full((B,), 500, device="cuda")

    def eager():
        with torch.no_grad(), torch.autocast("cuda", dtype=torch.float16):
            out = O.unet_forward(sdd, x_T, t, cond, False, x_obs, kf)
            out_u = O.unet_forward(sdd, x_T, t, cond, True, x_obs, kf)
            return out_u + 2.5 * (out - out_u)

    for fn in list(arms.values()) + [eager] * 3:  # warm-up: graph capture, module loads, cuDNN algorithm choice
        fn()
    torch.cuda.synchronize()
    times = {k: [] for k in arms}
    eager_ms = []
    for _ in range(args.rounds):
        for name, fn in arms.items():
            times[name].append(timed(fn))
        eager_ms.append(timed(eager))
    steps = diff["fp16"].num_timesteps
    res = {"card": card(), "batch": B, "schedule": "ddim50", "cfg_scale": 2.5, "rounds": args.rounds}
    for name, ts in times.items():
        med = statistics.median(ts)
        res[name] = {"loop_ms_median": round(med, 2), "loop_ms_min": round(min(ts), 2), "loop_ms_max": round(max(ts), 2),
                     "steps_per_s": round(steps / (med / 1000.0), 1)}
    res["fp16_over_bf16x3"] = round(res["fp16"]["steps_per_s"] / res["bf16x3"]["steps_per_s"], 3)
    med = statistics.median(eager_ms)
    res["eager_autocast_cfg_forward"] = {"ms_median": round(med, 2), "ms_min": round(min(eager_ms), 2),
                                         "steps_per_s": round(1000.0 / med, 1)}
    print(f"card: {res['card']['name']}  power limit, max SM clock: {res['card']['power_limit, max_sm_clock']}")
    print(json.dumps(res))
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_unet_precision.json"), "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()

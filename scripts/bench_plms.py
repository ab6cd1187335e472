"""PLMS against DDIM on one GPU: whole ddim50 loops at B = 64 of the 8-layer MDM transformer (random weights, no
conditioning), timed with CUDA events in one process, the samplers alternating round by round.

    python scripts/bench_plms.py [--batch 64] [--rounds 5] [--out DIR]

Prints the card, its power limit and one JSON line: per sampler, the median loop time and denoising steps/s (a step is
one sampler iteration; the PLMS loop evaluates the denoiser once more, in its first step).  Writes nothing unless --out
is given.
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this benchmark measures the GPU and has no CPU fallback")
    B, D, L = args.batch, 263, 196
    m = C.MDM()
    m.load_state_dict(O.random_state_dict(seed=0), strict=False)
    m = m.cuda()
    d = C.create_gaussian_diffusion(timestep_respacing="ddim50")
    x_T = torch.randn(B, D, 1, L, generator=torch.Generator().manual_seed(0)).cuda()
    kw = {"model_kwargs": {"y": {}}, "noise": x_T}
    arms = {
        "ddim": lambda: d.ddim_sample_loop(m, (B, D, 1, L), **kw),
        "plms_order2": lambda: d.plms_sample_loop(m, (B, D, 1, L), order=2, **kw),
        "plms_order4": lambda: d.plms_sample_loop(m, (B, D, 1, L), order=4, **kw),
    }
    for fn in arms.values():  # warm-up: graph capture, chained-launch tables, module loads
        fn()
    torch.cuda.synchronize()
    times = {k: [] for k in arms}
    for _ in range(args.rounds):
        for name, fn in arms.items():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            out = fn()
            e1.record()
            e1.synchronize()
            times[name].append(e0.elapsed_time(e1))
            assert torch.isfinite(out).all()
    steps = d.num_timesteps
    res = {"card": card(), "batch": B, "schedule": "ddim50", "rounds": args.rounds}
    for name, ts in times.items():
        med = statistics.median(ts)
        res[name] = {"loop_ms_median": round(med, 2), "loop_ms_min": round(min(ts), 2), "loop_ms_max": round(max(ts), 2),
                     "steps_per_s": round(steps / (med / 1000.0), 1)}
    print(f"card: {res['card']['name']}  power limit, max SM clock: {res['card']['power_limit, max_sm_clock']}")
    print(json.dumps(res))
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_plms.json"), "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()

"""UniPC against DDIM and DPM-Solver++ on one GPU, in one process.

    python scripts/bench_unipc.py [--batch 64] [--rounds 5] [--err-batch 8] [--out DIR]

1. Loop time: whole ddim50 loops of DDIM, DPM-Solver++ orders 2 / 3 and UniPC orders 2 / 3 (bh2, with the corrector) at
   B = --batch, for the 8-layer MDM transformer (bf16x3, no conditioning) and the keyframe-conditioned MDM_UNET xl at fp16
   with CFG 2.5, timed with CUDA events, the samplers alternating round by round; medians.
2. Discretisation error: the end state of every arm, UniP (no corrector) and UniPC bh1 included, at 10, 20, 50 and 100
   steps against a 1000-step order-1 solution from the same x_T (B = --err-batch), max and mean of the absolute
   difference.  The grids are the section respacings "10" / "20" / "50" / "100", which keep t = 999 like the 1000 steps,
   so every run starts from the same x_T at the same noise level.  The weights are random: this measures how accurately
   the ODE is discretised, not sample quality.

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

import condmdi_b200 as C  # noqa: E402,F401
from bench_dpm_solver import D, L, card, transformer, unet_xl  # noqa: E402

TIMED = ("ddim", "dpm_order2", "dpm_order3", "unipc_order2", "unipc_order3")
ERROR_ARMS = ("ddim", "dpm_order2", "dpm_order3", "unip_order2", "unip_order3", "unipc_order1", "unipc_order2",
              "unipc_order3", "unipc_bh1_order2", "unipc_bh1_order3")


def loops(d, m, shape, kw):
    return {
        "ddim": lambda: d.ddim_sample_loop(m, shape, **kw),
        "dpm_order2": lambda: d.dpm_solver_sample_loop(m, shape, order=2, **kw),
        "dpm_order3": lambda: d.dpm_solver_sample_loop(m, shape, order=3, **kw),
        "unip_order2": lambda: d.unipc_sample_loop(m, shape, order=2, corrector=False, **kw),
        "unip_order3": lambda: d.unipc_sample_loop(m, shape, order=3, corrector=False, **kw),
        "unipc_order1": lambda: d.unipc_sample_loop(m, shape, order=1, **kw),
        "unipc_order2": lambda: d.unipc_sample_loop(m, shape, order=2, **kw),
        "unipc_order3": lambda: d.unipc_sample_loop(m, shape, order=3, **kw),
        "unipc_bh1_order2": lambda: d.unipc_sample_loop(m, shape, order=2, variant="bh1", **kw),
        "unipc_bh1_order3": lambda: d.unipc_sample_loop(m, shape, order=3, variant="bh1", **kw),
    }


def timing(model, B, rounds):
    m, kwargs, precision = model
    d = C.create_gaussian_diffusion(timestep_respacing="ddim50")
    d.precision, d.rng = precision, "engine"
    x_T = torch.randn(B, D, 1, L, generator=torch.Generator().manual_seed(0)).cuda()
    arms = {k: v for k, v in loops(d, m, (B, D, 1, L), {"model_kwargs": kwargs(B), "noise": x_T}).items() if k in TIMED}
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
                     "steps_per_s": round(50 / (med / 1000.0), 1)}
    return res


def errors(model, B):
    m, kwargs, precision = model
    x_T = torch.randn(B, D, 1, L, generator=torch.Generator().manual_seed(4)).cuda()
    kw = {"model_kwargs": kwargs(B), "noise": x_T}

    def diffusion(respacing):
        d = C.create_gaussian_diffusion(timestep_respacing=respacing)
        d.precision, d.rng = precision, "engine"
        return d

    ref = diffusion("").dpm_solver_sample_loop(m, (B, D, 1, L), order=1, **kw).double()
    res = {}
    for n in (10, 20, 50, 100):
        d = diffusion(str(n))
        assert d.timestep_map[-1] == 999 and d.num_timesteps == n
        for name, fn in loops(d, m, (B, D, 1, L), kw).items():
            e = (fn().double() - ref).abs()
            res[f"{name}@{n}"] = {"max": float(f"{e.max().item():.4g}"), "mean": float(f"{e.mean().item():.4g}")}
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--err-batch", type=int, default=8)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this benchmark measures the GPU and has no CPU fallback")
    res = {"card": card(), "batch": args.batch, "rounds": args.rounds, "err_batch": args.err_batch}
    for name, build in (("transformer_bf16x3", transformer), ("unet_xl_fp16_cfg", unet_xl)):
        model = build()
        res[name] = {"time_ddim50": timing(model, args.batch, args.rounds), "end_error_vs_1000_order1": errors(model, args.err_batch)}
    print(f"card: {res['card']['name']}  power limit, max SM clock: {res['card']['power_limit, max_sm_clock']}")
    for name in ("transformer_bf16x3", "unet_xl_fp16_cfg"):
        print(f"\n{name}: ddim50 loop at B = {args.batch}, median ms (steps/s)")
        for arm, r in res[name]["time_ddim50"].items():
            print(f"  {arm:16s} {r['loop_ms_median']:9.2f} ms  ({r['steps_per_s']} steps/s)")
        print(f"{name}: end state vs 1000-step order 1, B = {args.err_batch}: max / mean |x - x_1000|")
        for arm in ERROR_ARMS:
            row = "  ".join(f"{n:3d}: {res[name]['end_error_vs_1000_order1'][f'{arm}@{n}']['max']:.3e} / "
                            f"{res[name]['end_error_vs_1000_order1'][f'{arm}@{n}']['mean']:.3e}" for n in (10, 20, 50, 100))
            print(f"  {arm:16s} {row}")
    print(json.dumps(res))
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_unipc.json"), "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()

"""RePaint resampling against p_sample_loop on the same schedule, on one GPU, in one process.

    python scripts/bench_repaint.py [--batch 64] [--rounds 3] [--jump-length 10] [--jump-n-sample 10] [--out DIR]

At B = --batch:
  - the 8-layer MDM transformer (bf16x3) with CFG 2.5, keyframe imputation and reconstruction guidance w = 20 (BASELINE
    config 4), on the last 30 steps of the 1000-step schedule (as bench.py times that config);
  - the keyframe-conditioned MDM_UNET xl at PRECISION_FP16 with CFG 2.5 and keyframe input, whole ddim50 loops;
for p_sample_loop and repaint_sample_loop, the two alternating round by round, timed with CUDA events; medians.  Both
draw their noise from the engine generator.  Reported: p_sample_loop steps/s, and for RePaint denoiser passes/s (denoise
ops) and walk ops/s (denoise + undo ops).  A denoise op costs a p_sample_loop step, so passes/s should match steps/s.
Then one UNet walk runs under torch.profiler: an undo op is a repaint_step_kernel launch that directly follows another
(a denoise op's follows the denoiser's last kernel), and their median device time is the undo op's time per launch.

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
from oracle import repaint_oracle as R  # noqa: E402


def transformer_cfg_imputation_guidance():
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
                      "mask": torch.ones(B, 1, 1, L, dtype=torch.bool).cuda(), "imputate": 1, "stop_imputation_at": 1,
                      "replacement_distribution": "conditional", "inpainted_motion": x_obs.cuda(), "inpainting_mask": kf.cuda(),
                      "reconstruction_guidance": True, "reconstruction_weight": 20.0, "gradient_schedule": None,
                      "diffusion_steps": 1000, "stop_recguidance_at": 0}}
    return C.ClassifierFreeSampleModel(m), kwargs, C.PRECISION_BF16X3


def setup(model, respacing, skip, B):
    m, kwargs, precision = model
    d = C.create_gaussian_diffusion(timestep_respacing=respacing)
    d.precision, d.rng, d.engine_seed = precision, "engine", 1
    x_T = torch.randn(B, D, 1, L, generator=torch.Generator().manual_seed(0)).cuda()
    return d, m, {"model_kwargs": kwargs(B), "noise": x_T, "skip_timesteps": skip}


def timing(model, respacing, skip, B, rounds, j, r):
    d, m, kw = setup(model, respacing, skip, B)
    shape = (B, D, 1, L)
    steps = d.num_timesteps - skip
    n_den, n_undo = R.op_counts(steps - 1, j, r)
    arms = {"p_sample_loop": lambda: d.p_sample_loop(m, shape, **kw),
            "repaint": lambda: d.repaint_sample_loop(m, shape, jump_length=j, jump_n_sample=r, **kw)}
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
    res = {"steps": steps, "jump_length": j, "jump_n_sample": r, "denoise_ops": n_den, "undo_ops": n_undo}
    for name, ts in times.items():
        med = statistics.median(ts)
        row = {"loop_ms_median": round(med, 2), "loop_ms_min": round(min(ts), 2), "loop_ms_max": round(max(ts), 2)}
        if name == "p_sample_loop":
            row["steps_per_s"] = round(steps / (med / 1000.0), 2)
        else:
            row["passes_per_s"] = round(n_den / (med / 1000.0), 2)
            row["walk_ops_per_s"] = round((n_den + n_undo) / (med / 1000.0), 2)
        res[name] = row
    return res


def undo_kernel_time(model, B, j, r):
    """median / min / max device time of the undo launches of one ddim50 walk, from a torch.profiler trace"""
    from torch.profiler import ProfilerActivity, profile

    d, m, kw = setup(model, "ddim50", 0, B)
    d.repaint_sample_loop(m, (B, D, 1, L), jump_length=j, jump_n_sample=r, **kw)  # warm-up
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        d.repaint_sample_loop(m, (B, D, 1, L), jump_length=j, jump_n_sample=r, **kw)
        torch.cuda.synchronize()
    kernels = sorted((e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA
                      and "memcpy" not in e.name.lower() and "memset" not in e.name.lower()),
                     key=lambda e: e.time_range.start)
    undo = [b.time_range.elapsed_us() for a, b in zip(kernels, kernels[1:])
            if "repaint_step_kernel" in a.name and "repaint_step_kernel" in b.name]
    n_den, n_undo = R.op_counts(49, j, r)
    assert len(undo) == n_undo, (len(undo), n_undo)
    return {"launches": len(undo), "us_median": round(statistics.median(undo), 2), "us_min": round(min(undo), 2),
            "us_max": round(max(undo), 2)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--jump-length", type=int, default=10)
    ap.add_argument("--jump-n-sample", type=int, default=10)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this benchmark measures the GPU and has no CPU fallback")
    j, r, B = args.jump_length, args.jump_n_sample, args.batch
    res = {"card": card(), "batch": B, "rounds": args.rounds}
    res["transformer_bf16x3_cfg_imputation_guidance"] = timing(transformer_cfg_imputation_guidance(), "", 970, B,
                                                               args.rounds, j, r)
    unet = unet_xl()
    res["unet_xl_fp16_cfg"] = timing(unet, "ddim50", 0, B, args.rounds, j, r)
    try:  # a separate, traced run: it does not touch the timings above
        res["undo_op_unet_xl_ddim50"] = undo_kernel_time(unet, B, j, r)
    except Exception as ex:  # noqa: BLE001  (reported, not hidden: the JSON line carries the error)
        res["undo_op_unet_xl_ddim50"] = {"error": repr(ex)}
    print(f"card: {res['card']['name']}  power limit, max SM clock: {res['card']['power_limit, max_sm_clock']}")
    for name in ("transformer_bf16x3_cfg_imputation_guidance", "unet_xl_fp16_cfg"):
        x = res[name]
        print(f"\n{name}: {x['steps']} steps at B = {B}; RePaint j {j}, r {r}: {x['denoise_ops']} denoise + "
              f"{x['undo_ops']} undo ops")
        p, w = x["p_sample_loop"], x["repaint"]
        print(f"  p_sample_loop {p['loop_ms_median']:10.2f} ms  {p['steps_per_s']} steps/s")
        print(f"  repaint       {w['loop_ms_median']:10.2f} ms  {w['passes_per_s']} passes/s, {w['walk_ops_per_s']} walk ops/s")
    u = res["undo_op_unet_xl_ddim50"]
    if "error" in u:
        print(f"\nundo op: not measured ({u['error']})")
    else:
        print(f"\nundo op: {u['launches']} launches, median {u['us_median']} us (min {u['us_min']}, max {u['us_max']})")
    print(json.dumps(res))
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_repaint.json"), "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()

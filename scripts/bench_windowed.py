"""Overlapping windows against plain sequences of the same row count, on one GPU, in one process.

    python scripts/bench_windowed.py [--batch 16] [--frames 600] [--window 196] [--overlap 48] [--rounds 3] [--out DIR]

Windowed: B = --batch motions of --frames frames in windows of --window frames overlapping by at least --overlap (the
defaults give K = 4 windows, 64 window rows).  Plain: B * K sequences of --window frames, the same denoiser work.  For
  - the 8-layer MDM transformer (bf16x3) with text and CFG 2.5,
  - the keyframe-conditioned MDM_UNET xl at PRECISION_FP16 with CFG 2.5 and keyframe input,
whole ddim50 loops, the two arms alternating round by round, timed with CUDA events; medians, as steps/s.  Both draw
their noise from the engine generator.  Then one loop of each arm runs under torch.profiler, and the median device
time of its step kernel (diffusion_step_kernel: the blended instance on windows, the plain one otherwise) is reported
per launch.

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
from bench_dpm_solver import D, card  # noqa: E402
from oracle import condmdi_oracle as O  # noqa: E402


def models():
    """(name, CFG-wrapped model, kwargs(B, N), precision): prompts are str(i), embeddings from a fixed table"""
    g = torch.Generator().manual_seed(2)
    cond = torch.randn(512, 512, generator=g).cuda()
    enc = lambda texts: cond[torch.tensor([int(t) for t in texts])]  # noqa: E731
    tr = C.MDM(cond_mode="text", cond_mask_prob=0.1)
    tr.load_state_dict(O.random_state_dict(seed=0, text=True), strict=False)
    tr = tr.cuda()
    tr.encode_text = enc
    un = C.MDM_UNET(keyframe_conditioned=True, cond_mode="text", cond_mask_prob=0.1)
    un.load_state_dict(O.random_unet_state_dict(seed=1, text=True), strict=False)
    un = un.cuda()
    un.encode_text = enc

    def text_kw(B, N):
        return {"y": {"text": [str(i) for i in range(B)], "text_scale": torch.full((B,), 2.5).cuda()}}

    def unet_kw(B, N):
        gk = torch.Generator().manual_seed(3)
        x_obs = torch.randn(B, D, 1, N, generator=gk)
        kf = C.get_keyframes_mask(x_obs, torch.full((B,), N), "benchmark_sparse", trans_length=5)
        return dict(text_kw(B, N), obs_x0=x_obs.cuda(), obs_mask=kf.cuda())
    return [("transformer_bf16x3_cfg", C.ClassifierFreeSampleModel(tr), text_kw, C.PRECISION_BF16X3),
            ("unet_xl_fp16_cfg", C.ClassifierFreeSampleModel(un), unet_kw, C.PRECISION_FP16)]


def arms(model, kwargs, precision, B, N, window):
    K = len(window.placement(N))
    out = {}
    for name, w, shape in (("windowed", window, (B, D, 1, N)), ("plain", None, (B * K, D, 1, window.frames))):
        d = C.create_gaussian_diffusion(timestep_respacing="ddim50")
        d.precision, d.rng, d.engine_seed, d.window = precision, "engine", 1, w
        kw = kwargs(shape[0], shape[-1])
        out[name] = (lambda d=d, shape=shape, kw=kw: d.ddim_sample_loop(model, shape, model_kwargs=kw))
    return out, K


def step_kernel_us(fn):
    from torch.profiler import ProfilerActivity, profile

    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    us = [e.time_range.elapsed_us() for e in prof.events()
          if e.device_type == torch.autograd.DeviceType.CUDA and "diffusion_step_kernel" in e.name]
    return {"launches": len(us), "us_median": round(statistics.median(us), 2), "us_min": round(min(us), 2),
            "us_max": round(max(us), 2)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--frames", type=int, default=600)
    ap.add_argument("--window", type=int, default=196)
    ap.add_argument("--overlap", type=int, default=48)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this benchmark measures the GPU and has no CPU fallback")
    B, N, window = args.batch, args.frames, C.Window(args.window, args.overlap)
    res = {"card": card(), "batch": B, "frames": N, "window": args.window, "overlap": args.overlap, "rounds": args.rounds,
           "placement": window.placement(N)}
    names = []
    for name, model, kwargs, precision in models():
        names.append(name)
        fns, K = arms(model, kwargs, precision, B, N, window)
        for fn in fns.values():  # warm-up: graph capture, chained-launch tables, module loads
            fn()
        torch.cuda.synchronize()
        times = {k: [] for k in fns}
        for _ in range(args.rounds):
            for arm, fn in fns.items():
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                out = fn()
                e1.record()
                e1.synchronize()
                times[arm].append(e0.elapsed_time(e1))
                assert torch.isfinite(out).all()
        row = {"window_rows": B * K}
        for arm, ts in times.items():
            med = statistics.median(ts)
            row[arm] = {"loop_ms_median": round(med, 2), "loop_ms_min": round(min(ts), 2), "loop_ms_max": round(max(ts), 2),
                        "steps_per_s": round(50 / (med / 1000.0), 2)}
        for arm, fn in fns.items():  # separate traced runs: they do not touch the timings above
            try:
                row[arm]["step_kernel"] = step_kernel_us(fn)
            except Exception as ex:  # noqa: BLE001  (reported, not hidden: the JSON line carries the error)
                row[arm]["step_kernel"] = {"error": repr(ex)}
        res[name] = row
    print(f"card: {res['card']['name']}  power limit, max SM clock: {res['card']['power_limit, max_sm_clock']}")
    print(f"{B} motions x {N} frames, windows of {args.window} overlapping >= {args.overlap}: {res['placement']}")
    for name in names:
        x = res[name]
        print(f"\n{name}: {x['window_rows']} window rows against {x['window_rows']} plain sequences, ddim50")
        for arm in ("windowed", "plain"):
            r, k = x[arm], x[arm]["step_kernel"]
            ks = f"{k['us_median']} us/launch over {k['launches']}" if "us_median" in k else f"not measured ({k['error']})"
            print(f"  {arm:8s} {r['loop_ms_median']:10.2f} ms  {r['steps_per_s']} steps/s  step kernel {ks}")
    print(json.dumps(res))
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_windowed.json"), "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()

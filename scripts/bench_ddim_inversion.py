"""Whole ddim50 DDIM inversions (ddim_reverse_sample_loop) at B = 64 on one GPU, against the loop a user runs today: the
reference's reverse step, eagerly, on the same GPU (the restatement's denoiser and update in torch; fp32, or CUDA fp16
autocast for the fp16 UNet).  A DDIM sampling loop of the same length on the engine is timed too, for comparison.

    python scripts/bench_ddim_inversion.py [--batch 64] [--rounds 3] [--out DIR]

Workloads: the 8-layer MDM transformer (no conditioning), and the keyframe-conditioned MDM_UNET xl with CFG 2.5 at bf16x3
and at fp16 (random weights).  Arms alternate round by round; CUDA events; medians.  Prints the card, its power limit and
one JSON line; writes nothing unless --out is given.
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
from oracle import ddim_reverse_oracle as R  # noqa: E402

D, L = 263, 196


def card() -> dict:
    info = {"name": torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30)
        info["power_limit, max_sm_clock"] = q.stdout.strip().splitlines()[0]
    except Exception as ex:  # noqa: BLE001
        info["power_limit, max_sm_clock"] = f"unavailable ({ex})"
    return info


def eager_inversion(sdd, tab, x, c, autocast):
    """for t in range(T): x = ddim_reverse_sample(x, t): the restated step, every tensor on the GPU"""
    dev = x.device
    nxt = R.alphas_cumprod_next(tab)
    tmap = torch.tensor(tab.timestep_map, device=dev)
    with torch.no_grad():
        for t in range(tab.num_timesteps):
            tt = torch.full((x.shape[0],), t, device=dev, dtype=torch.long)
            ctx = torch.autocast("cuda", dtype=torch.float16) if autocast else torch.autocast("cuda", enabled=False)
            with ctx:
                x0 = O._model(sdd, x, tmap[tt], c).float()
            r1 = torch.tensor(tab.sqrt_recip_alphas_cumprod[t], device=dev).float()
            r2 = torch.tensor(tab.sqrt_recipm1_alphas_cumprod[t], device=dev).float()
            an = torch.tensor(nxt[t], device=dev).float()
            eps = (r1 * x - x0) / r2
            x = x0 * torch.sqrt(an) + torch.sqrt(1 - an) * eps
    return x


def workloads(B):
    g = torch.Generator().manual_seed(0)
    x0 = torch.randn(B, D, 1, L, generator=g).cuda()
    out = {}
    sd = O.random_state_dict(seed=0)
    m = C.MDM()
    m.load_state_dict(sd, strict=False)
    out["transformer"] = dict(model=m.cuda(), sd=sd, kw={"y": {}}, c=O.Conditioning(), precision=C.PRECISION_BF16X3, fp16=False)
    sdu = O.random_unet_state_dict(seed=11, text=True)
    xo = torch.randn(B, D, 1, L, generator=g)
    lengths = torch.randint(40, L + 1, (B,), generator=g)
    kf = C.get_keyframes_mask(xo, lengths, "benchmark_sparse", trans_length=5)
    cond = torch.randn(B, 512, generator=g)
    scale = torch.full((B,), 2.5)
    for name, prec in (("unet_xl_cfg_kf_bf16x3", C.PRECISION_BF16X3), ("unet_xl_cfg_kf_fp16", C.PRECISION_FP16)):
        mu = C.MDM_UNET(keyframe_conditioned=True, cond_mode="text", cond_mask_prob=0.1)
        mu.load_state_dict(sdu, strict=False)
        mu = mu.cuda()
        table = {str(i): cond[i].cuda() for i in range(B)}
        mu.encode_text = lambda texts, table=table: torch.stack([table[s] for s in texts])
        kw = {"y": {"text": [str(i) for i in range(B)], "text_scale": scale.cuda()}, "obs_x0": xo.cuda(), "obs_mask": kf.cuda()}
        c = O.Conditioning(cond_emb=cond.cuda(), cfg=True, text_scale=scale.cuda(), obs_x0=xo.cuda(), obs_mask=kf.cuda())
        out[name] = dict(model=C.ClassifierFreeSampleModel(mu), sd=sdu, kw=kw, c=c, precision=prec, fp16=prec == C.PRECISION_FP16)
    return x0, out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this benchmark measures the GPU and has no CPU fallback")
    B = args.batch
    x0, wl = workloads(B)
    tab = O.make_tables("ddim50")
    res = {"card": card(), "batch": B, "schedule": "ddim50", "rounds": args.rounds}
    for name, w in wl.items():
        d = C.create_gaussian_diffusion(timestep_respacing="ddim50")
        d.precision = w["precision"]
        sdd = {k: v.cuda() for k, v in w["sd"].items()}
        arms = {
            "engine_inversion": lambda: d.ddim_reverse_sample_loop(w["model"], x0, model_kwargs=w["kw"]),
            "eager_inversion": lambda: eager_inversion(sdd, tab, x0, w["c"], w["fp16"]),
            "engine_ddim_sampling": lambda: d.ddim_sample_loop(w["model"], (B, D, 1, L), noise=x0, model_kwargs=w["kw"]),
        }
        outs = {k: fn() for k, fn in arms.items()}  # warm-up: graph capture, module loads, cuDNN algorithm choice
        torch.cuda.synchronize()
        diff = (outs["engine_inversion"] - outs["eager_inversion"]).abs()
        times = {k: [] for k in arms}
        for _ in range(args.rounds):
            for arm, fn in arms.items():
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                out = fn()
                e1.record()
                e1.synchronize()
                times[arm].append(e0.elapsed_time(e1))
                assert torch.isfinite(out).all()
        r = {"max|engine - eager| at x_T": float(diff.max()), "max|x_T|": float(outs["eager_inversion"].abs().max())}
        for arm, ts in times.items():
            med = statistics.median(ts)
            r[arm] = {"loop_ms_median": round(med, 2), "loop_ms_min": round(min(ts), 2), "loop_ms_max": round(max(ts), 2),
                      "steps_per_s": round(d.num_timesteps / (med / 1000.0), 1)}
        r["speedup_vs_eager"] = round(r["eager_inversion"]["loop_ms_median"] / r["engine_inversion"]["loop_ms_median"], 2)
        res[name] = r
        print(name, json.dumps(r), flush=True)
        del sdd
        torch.cuda.empty_cache()
    print(f"card: {res['card']['name']}  power limit, max SM clock: {res['card']['power_limit, max_sm_clock']}")
    print(json.dumps(res))
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_ddim_inversion.json"), "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()

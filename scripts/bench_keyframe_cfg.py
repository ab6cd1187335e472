"""Keyframe classifier-free guidance on one GPU: whole ddim50 loops of the xl UNet (dim 512, dim_mults (2,2,2,2), keyframe
input conditioning, text; random weights) at B = 64, CFG (text scale 2.5) against keyframe + text CFG
(KeyframeClassifierFreeSampleModel, w_k = 1.5), at fp16 and at bf16x3, timed with CUDA events in one process, the arms
alternating round by round.  One more leg times a single eager evaluation of the three-pass restatement under
torch.autocast("cuda", float16).

    python scripts/bench_keyframe_cfg.py [--batch 64] [--rounds 5] [--out DIR]

Prints the card, its power limit and max SM clock, and one JSON line: per arm the median loop time and steps/s, the
keyframe-CFG / CFG time ratio per precision, and the eager evaluation's median time.  Writes nothing unless --out is given.
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
from oracle import keyframe_cfg_oracle as K  # noqa: E402


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
    y = {"text": [str(i) for i in range(B)], "text_scale": torch.full((B,), 2.5).cuda(), "keyframe_scale": torch.full((B,), 1.5).cuda(),
         "mask": torch.ones(B, 1, 1, L, dtype=torch.bool).cuda()}
    kw = {"y": y, "obs_x0": x_obs, "obs_mask": kf}
    models = {"cfg": C.ClassifierFreeSampleModel(m), "kf_cfg": C.KeyframeClassifierFreeSampleModel(m)}
    diffs = {}
    for prec_name, prec in (("fp16", C.PRECISION_FP16), ("bf16x3", C.PRECISION_BF16X3)):
        d = C.create_gaussian_diffusion(timestep_respacing="ddim50")
        d.precision = prec
        d.max_batch = (3 * B + 1) // 2  # one engine per precision serves both arms
        diffs[prec_name] = d
    arms = {f"{p}_{w}": (lambda d=d, mw=mw: d.ddim_sample_loop(mw, (B, D, 1, L), model_kwargs=kw, noise=x_T))
            for p, d in diffs.items() for w, mw in models.items()}

    sdd = {k: v.cuda() for k, v in sd.items()}
    t = torch.full((B,), 500, device="cuda")
    c = O.Conditioning(cond_emb=cond, cfg=True, obs_x0=x_obs, obs_mask=kf)
    ts, wk = y["text_scale"], y["keyframe_scale"]

    def eager():
        with torch.no_grad(), torch.autocast("cuda", dtype=torch.float16):
            passes = K.passes(sdd, x_T, t, c)
        return K.combine(*passes, ts, wk)

    for fn in list(arms.values()) + [eager] * 3:  # warm-up: graph capture, module loads, cuDNN algorithm choice
        fn()
    torch.cuda.synchronize()
    times = {k: [] for k in arms}
    eager_ms = []
    for _ in range(args.rounds):
        for name, fn in arms.items():
            times[name].append(timed(fn))
        eager_ms.append(timed(eager))
    steps = 50
    res = {"card": card(), "batch": B, "schedule": "ddim50", "text_scale": 2.5, "keyframe_scale": 1.5, "rounds": args.rounds}
    for name, tt in times.items():
        med = statistics.median(tt)
        res[name] = {"loop_ms_median": round(med, 2), "loop_ms_min": round(min(tt), 2), "loop_ms_max": round(max(tt), 2),
                     "steps_per_s": round(steps / (med / 1000.0), 1), "ms_per_step": round(med / steps, 2)}
    for p in diffs:
        res[f"{p}_kf_cfg_over_cfg"] = round(res[f"{p}_kf_cfg"]["loop_ms_median"] / res[f"{p}_cfg"]["loop_ms_median"], 3)
    med = statistics.median(eager_ms)
    res["eager_autocast_three_pass_evaluation"] = {"ms_median": round(med, 2), "ms_min": round(min(eager_ms), 2)}
    print(f"card: {res['card']['name']}  power limit, max SM clock: {res['card']['power_limit, max_sm_clock']}")
    print(json.dumps(res))
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_keyframe_cfg.json"), "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()

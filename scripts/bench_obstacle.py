"""Obstacle-avoidance guidance on one GPU: whole ddim50 loops at B = 64 with CFG 2.5 of the transformer (bf16x3) and of
the xl MDM_UNET (fp16, keyframe input conditioning), each guided on every step by reconstruction + joint guidance
(w = 20 and 0.1, pelvis XZ on every frame and every joint on 4 keyframes, abs_3d) and by reconstruction + obstacle
guidance (w = 20 and 20, the pelvis, K = 1, 8 and 16 cylinders per sample); the arms alternate round by round in one
process and are timed with CUDA events.  One more leg times the seed kernel's obstacle instance alone
(cmdi_obstacle_seed on B x 196 frame-major rows of 264 columns, K = 16, every joint in S) next to the joint instance:
the kernels' device times from torch.profiler.  Random weights.

    python scripts/bench_obstacle.py [--batch 64] [--rounds 5] [--out DIR]

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
from oracle import joint_guidance_oracle as J  # noqa: E402
from oracle import obstacle_oracle as OB  # noqa: E402

KS = (1, 8, 16)


def arms_of(name, m, precision, B, D, L, g, unet):
    x_T = torch.randn(B, D, 1, L, generator=g).cuda()
    x_obs = torch.randn(B, D, 1, L, generator=g).cuda()
    kf = C.get_keyframes_mask(x_obs.cpu(), torch.full((B,), L), "benchmark_sparse", trans_length=5).cuda()
    cond = torch.randn(B, 512, generator=g).cuda()
    table = {str(i): cond[i] for i in range(B)}
    m.encode_text = lambda texts: torch.stack([table[t] for t in texts])
    w = C.ClassifierFreeSampleModel(m)
    mean, std, jt, jm, _ = J.inputs(B, L, seed=1)
    y = {"text": [str(i) for i in range(B)], "text_scale": torch.full((B,), 2.5).cuda(),
         "mask": torch.ones(B, 1, 1, L, dtype=torch.bool).cuda(), "diffusion_steps": 1000}
    recon = dict(reconstruction_guidance=True, reconstruction_weight=20.0, gradient_schedule=None, stop_recguidance_at=0,
                 inpainted_motion=x_obs, inpainting_mask=kf)
    joint = dict(joint_guidance=True, joint_target=jt.cuda(), joint_target_mask=jm.cuda(), joint_guidance_weight=0.1,
                 joint_gradient_schedule=None, stop_jointguidance_at=0)

    def obstacles(K):
        o = torch.rand(B, K, 3, generator=g)
        o[..., :2] = o[..., :2] * 2 - 1
        o[..., 2] = 0.2 + 0.8 * o[..., 2]
        return dict(obstacle_guidance=True, obstacles=o.cuda(), obstacle_weight=20.0, obstacle_gradient_schedule=None,
                    stop_obstacleguidance_at=0)

    d = C.create_gaussian_diffusion(timestep_respacing="ddim50")
    d.precision = precision
    d.joint_space = C.JointSpace(mean, std, abs_3d=True)
    extra = {"obs_x0": x_obs, "obs_mask": kf} if unet else {}
    arms = [("recon_joint", dict(recon, **joint))] + [(f"recon_obstacle_k{K}", dict(recon, **obstacles(K))) for K in KS]
    return {f"{name}_{arm}": (lambda yy=dict(y, **kw): d.ddim_sample_loop(w, (B, D, 1, L), model_kwargs={"y": yy, **extra},
                                                                          noise=x_T))
            for arm, kw in arms}, d.num_timesteps


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
    mt = C.MDM(cond_mode="text", cond_mask_prob=0.1)
    mt.load_state_dict(O.random_state_dict(seed=0, text=True), strict=False)
    mu = C.MDM_UNET(keyframe_conditioned=True, cond_mode="text", cond_mask_prob=0.1)
    mu.load_state_dict(O.random_unet_state_dict(seed=0, text=True), strict=False)
    arms, steps = arms_of("transformer_bf16x3", mt.cuda(), C.PRECISION_BF16X3, B, D, L, g, False)
    arms.update(arms_of("unet_xl_fp16", mu.cuda(), C.PRECISION_FP16, B, D, L, g, True)[0])
    for fn in arms.values():  # warm-up: graph capture, module loads
        fn()
    torch.cuda.synchronize()
    times = {k: [] for k in arms}
    for _ in range(args.rounds):
        for name, fn in arms.items():
            times[name].append(timed(fn))
    res = {"card": card(), "batch": B, "schedule": "ddim50", "cfg_scale": 2.5, "rounds": args.rounds}
    for name in arms:
        med = statistics.median(times[name])
        res[name] = {"loop_ms_median": round(med, 2), "steps_per_s": round(steps / (med / 1000.0), 1),
                     "ms_per_step": round(med / steps, 3),
                     "spread_ms": [round(min(times[name]), 2), round(max(times[name]), 2)]}
    # the seed kernel's joint and obstacle instances alone in the engine's layout (frame-major rows of D_pad = 264)
    mean, std, x0, obs, _ = OB.inputs(B, L, seed=2, K=16, joints=tuple(range(22)))
    _, _, jt, jm, _ = J.inputs(B, L, seed=2)
    rows = torch.zeros(B, L, 264)
    rows[:, :, :263] = x0[:, :, 0].transpose(1, 2)
    rows, jt, jm, mean, std = rows.cuda(), jt.cuda().contiguous(), jm.cuda().to(torch.uint8).contiguous(), mean.cuda(), std.cuda()
    obs = obs.cuda().contiguous()
    grad = torch.empty_like(rows)
    lib, stream = C.capi.load(), torch.cuda.current_stream().cuda_stream

    def seeds(obstacle):
        for _ in range(200):
            if obstacle:
                C.capi.check(lib.cmdi_obstacle_seed(rows.data_ptr(), B, D, L, 264, None, jt.data_ptr(), jm.data_ptr(),
                                                    mean.data_ptr(), std.data_ptr(), 1, 0.5, 0, 0.0, obs.data_ptr(), 16,
                                                    (1 << 22) - 1, 0.5, grad.data_ptr(), stream))
            else:
                C.capi.check(lib.cmdi_joint_guidance_seed(rows.data_ptr(), B, D, L, 264, jt.data_ptr(), jm.data_ptr(),
                                                          mean.data_ptr(), std.data_ptr(), 1, grad.data_ptr(), stream))

    seeds(False)
    seeds(True)
    torch.cuda.synchronize()
    for obstacle, key, kernel in ((False, "joint_seed_kernel_us", "joint_seed_kernel"),
                                  (True, "obstacle_seed_kernel_us_k16_all_joints", "obstacle_seed_kernel")):
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            seeds(obstacle)
            torch.cuda.synchronize()
        dev_us = [e.device_time for e in prof.events() if kernel in e.name]
        res[key] = round(statistics.median(dev_us), 1) if dev_us else None
    print(f"card: {res['card']['name']}  power limit, max SM clock: {res['card']['power_limit, max_sm_clock']}")
    print(json.dumps(res))
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_obstacle.json"), "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()

"""Representation conversions on the GPU against the CPU restatement on the host, at B = 64 x 196 frames.

    python scripts/bench_motion_features.py [--batch 64] [--frames 196] [--repeats 50] [--out DIR]

GPU: `abs3d_to_rel`, `rel_to_abs3d` (with and without the inverse random projection) and `joints_to_features`, each
one launch, timed with CUDA events over `repeats` back-to-back calls after a warm-up (median of 5 rounds).
Host: oracle/motion_features_oracle.py, called once per sequence as the reference's conversions loop over the batch
(dataset.py:1205, :1264).  This is the restatement, not the reference (which this benchmark does not need or read); it
uses the same numpy / torch / scipy operations per sequence.

Prints the card, its power limit, the host core count and one JSON line.  Writes nothing unless --out is given.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import condmdi_b200 as C  # noqa: E402
from oracle import motion_features_oracle as MF  # noqa: E402


def card() -> dict:
    info = {"name": torch.cuda.get_device_name(0), "host_cores": os.cpu_count(), "torch_threads": torch.get_num_threads()}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30)
        info["power_limit, max_sm_clock"] = q.stdout.strip().splitlines()[0]
    except Exception as ex:  # noqa: BLE001
        info["power_limit, max_sm_clock"] = f"unavailable ({ex})"
    return info


def inputs(B: int, L: int, seed: int = 0):
    """Seeded, motion-like inputs: a synthetic walk (joints), its normalised features, a random projection."""
    g = np.random.default_rng(seed)
    t = np.arange(L, dtype=np.float64)[:, None] / 20.0
    offs = MF.T2M_RAW_OFFSETS.astype(np.float64) * 0.25
    joints = np.zeros((B, L, 22, 3))
    for chain in MF.T2M_KINEMATIC_CHAIN:
        for j0, j1 in zip(chain[:-1], chain[1:]):
            joints[:, :, j1] = joints[:, :, j0] + offs[j1]
    joints[..., 1] += 0.9
    joints[..., 2] += 1.2 * t                                   # walk along +z
    joints += g.normal(0, 0.02, joints.shape)
    joints = joints.astype(np.float32)
    mean = np.zeros(263)
    std = np.ones(263)
    f = MF.extract_features(joints)
    rel = torch.cat((f, f[:, -1:]), 1).permute(0, 2, 1)[:, :, None, :].contiguous().float()
    P = g.normal(0, 1, (263, 263)) / np.sqrt(263)
    return joints, rel, mean, std, np.linalg.inv(P).astype(np.float32)


def gpu_ms(fn, repeats: int) -> float:
    fn()
    torch.cuda.synchronize()
    times = []
    for _ in range(5):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(repeats):
            fn()
        b.record()
        torch.cuda.synchronize()
        times.append(a.elapsed_time(b) / repeats)
    return statistics.median(times)


def host_ms(fn, B: int) -> float:
    t0 = time.perf_counter()
    for b in range(B):
        fn(b)
    return (time.perf_counter() - t0) * 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--frames", type=int, default=196)
    ap.add_argument("--repeats", type=int, default=50)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this benchmark measures the GPU and has no CPU fallback")
    B, L = args.batch, args.frames
    joints, rel, mean, std, inv_proj = inputs(B, L)
    dev = torch.device("cuda:0")
    rel_d, joints_d = rel.to(dev), torch.from_numpy(joints).to(dev)
    gpu = {
        "rel_to_abs3d": gpu_ms(lambda: C.rel_to_abs3d(rel_d, mean, std, mean, std), args.repeats),
        "rel_to_abs3d_proj": gpu_ms(lambda: C.rel_to_abs3d(rel_d, mean, std, mean, std, inv_proj=inv_proj), args.repeats),
        "abs3d_to_rel": gpu_ms(lambda: C.abs3d_to_rel(rel_d, mean, std, mean, std), args.repeats),
        "abs3d_to_rel_proj": gpu_ms(lambda: C.abs3d_to_rel(rel_d, mean, std, mean, std, inv_proj=inv_proj), args.repeats),
        "joints_to_features": gpu_ms(lambda: C.joints_to_features(joints_d), args.repeats),
    }
    host = {
        "rel_to_abs3d": host_ms(lambda b: MF.rel_to_abs3d(rel[b:b + 1], mean, std, mean, std), B),
        "abs3d_to_rel_proj": host_ms(lambda b: MF.abs3d_to_rel(rel[b:b + 1], mean, std, mean, std, inv_proj), B),
        "joints_to_features": host_ms(lambda b: MF.extract_features(joints[b]), B),
    }
    res = {"batch": B, "frames": L, "card": card(), "gpu_ms_per_batch": {k: round(v, 4) for k, v in gpu.items()},
           "host_restatement_ms_per_batch": {k: round(v, 1) for k, v in host.items()},
           "host_restatement_ms_per_motion": {k: round(v / B, 2) for k, v in host.items()}}
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_motion_features.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()

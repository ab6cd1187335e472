"""A/B of two builds of libcondmdi_b200.so on the flagship workload, on one GPU.

    python scripts/ab_bench.py A.so B.so [--rounds 5] [--steps 200] [--warmup 10] [--full] [--out DIR]

Each round runs `bench.py --skip-configs` once per build (A, then B) in a subprocess of its own, the library chosen with
CONDMDI_B200_LIB; the builds alternate round by round so that drift of the card's clocks hits both alike.  Per round it
prints steps/s, the clocks bench.py sampled and the per-kernel ms per step of its profiled pass.  Then:
  - outputs: the first round at bf16x3 and one extra run at bf16 dump the samples of the last timed step (same seeds);
    the two builds' sample.npy files are compared byte for byte;
  - one profile pass per build with CMDI_CHAIN_DBG=1, which prints the chained kernel's cycles per tile (warp 0:
    epi0_acc_wait = mainloop, epi0_slices = epilogue, epi0_publish = publish wait);
  - with --full, the whole bench.py (configs[2..4] and the eager PyTorch baseline) and scripts/bench_unet_precision.py
    once per build.
Prints the card's name, power limit and max SM clock first.  Writes nothing in the tree: dumps go to a temporary
directory, and a JSON summary to --out only if it is given.  Every subprocess is waited for (or killed on timeout).
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TIMEOUT_S = 1800

DBG_SNIPPET = r"""
import sys, torch
sys.path.insert(0, sys.argv[1])
import bench, condmdi_b200 as C
torch.manual_seed(0)
m = C.MDM(njoints=bench.D, nfeats=1, latent_dim=bench.D_MODEL, ff_size=bench.FF, num_layers=bench.LAYERS,
          num_heads=bench.HEADS, cond_mode="no_cond").cuda()
eng = m.engine_for(torch.device("cuda", 0), max_batch=bench.B, precision=C.capi.PRECISION_BF16X3)
eng.profile_pass(bench.B)
print("--- warm pass ---", file=sys.stderr, flush=True)
eng.profile_pass(bench.B)
"""


def card() -> str:
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=60)
        return q.stdout.strip().splitlines()[0]
    except Exception as ex:  # noqa: BLE001
        return f"unavailable ({ex})"


def run(cmd, lib, extra_env=None):
    env = dict(os.environ, CONDMDI_B200_LIB=os.path.abspath(lib), **(extra_env or {}))
    r = subprocess.run(cmd, cwd=ROOT, env=env, capture_output=True, text=True, timeout=TIMEOUT_S)
    if r.returncode != 0:
        raise SystemExit(f"{' '.join(cmd)} with {lib} failed ({r.returncode}):\n{r.stderr[-4000:]}")
    return r


def bench(lib, args, precision="bf16x3", dump=None, full=False):
    cmd = [sys.executable, "bench.py", "--gpus", "1", "--steps", str(args.steps), "--warmup", str(args.warmup),
           "--precision", precision]
    if not full:
        cmd.append("--skip-configs")
    if dump:
        cmd += ["--dump-outputs", dump]
    return json.loads(run(cmd, lib).stdout.strip().splitlines()[-1])


def same_bytes(a, b):
    with open(a, "rb") as fa, open(b, "rb") as fb:
        same = fa.read() == fb.read()
    if same:
        return {"identical": True}
    import numpy as np

    x, y = np.load(a), np.load(b)
    return {"identical": False, "max_abs_diff": float(np.abs(x.astype(np.float64) - y).max())}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("lib_a")
    ap.add_argument("lib_b")
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--full", action="store_true", help="also the whole bench.py and bench_unet_precision.py once per build")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    arms = {"A": args.lib_a, "B": args.lib_b}
    for lib in arms.values():
        if not os.path.exists(lib):
            raise SystemExit(f"{lib}: no such library")
    res = {"card (name, power limit, max SM clock)": card(), "libs": arms, "rounds": []}
    print("card (name, power limit, max SM clock):", res["card (name, power limit, max SM clock)"], flush=True)
    with tempfile.TemporaryDirectory(prefix="ab_bench_") as tmp:
        compare(arms, args, res, tmp)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "ab_bench.json"), "w") as f:
            json.dump(res, f, indent=1)


def compare(arms, args, res, tmp):
    values = {k: [] for k in arms}
    for r in range(args.rounds):
        for arm, lib in arms.items():
            dump = os.path.join(tmp, arm, "bf16x3") if r == 0 else None
            line = bench(lib, args, dump=dump)
            row = {"round": r, "arm": arm, "value": round(line["value"], 2), "clocks": line["clocks"],
                   "per_kernel_ms_per_step": line["roofline"]["per_kernel_ms_per_step"]}
            values[arm].append(line["value"])
            res["rounds"].append(row)
            print(json.dumps(row), flush=True)
    summary = {arm: {"median": round(statistics.median(v), 2), "min": round(min(v), 2), "max": round(max(v), 2)} for arm, v in values.items()}
    summary["B_median_over_A"] = round(statistics.median(values["B"]) / statistics.median(values["A"]), 4)
    summary["every_B_round_beats_every_A_round"] = min(values["B"]) > max(values["A"])
    res["summary"] = summary
    print("summary:", json.dumps(summary), flush=True)

    outputs = {}
    for arm, lib in arms.items():
        line = bench(lib, args, precision="bf16", dump=os.path.join(tmp, arm, "bf16"))
        outputs.setdefault("bf16_steps_per_s", {})[arm] = round(line["value"], 2)
    for prec in ("bf16x3", "bf16"):
        outputs[prec] = same_bytes(*(os.path.join(tmp, arm, prec, "sample.npy") for arm in arms))
    res["outputs"] = outputs
    print("outputs (sample.npy, A vs B):", json.dumps(outputs), flush=True)

    res["chain_dbg"] = {}
    for arm, lib in arms.items():
        r_ = run([sys.executable, "-c", DBG_SNIPPET, ROOT], lib, {"CMDI_CHAIN_DBG": "1"})
        warm = r_.stderr.split("--- warm pass ---")[-1]
        lines = [ln for ln in warm.splitlines() if ln.startswith("chain dbg")]
        res["chain_dbg"][arm] = lines
        print(f"chain dbg {arm}:", *lines, sep="\n  ", flush=True)

    if args.full:
        res["full"] = {}
        for arm, lib in arms.items():
            line = bench(lib, args, full=True)
            res["full"][arm] = {"value": round(line["value"], 2), "configs": line["configs"], "library_baseline": line["library_baseline"]}
            print(f"full bench {arm}:", json.dumps(res["full"][arm]), flush=True)
        for arm, lib in arms.items():
            out = run([sys.executable, os.path.join("scripts", "bench_unet_precision.py")], lib).stdout.strip().splitlines()
            res["full"][arm]["bench_unet_precision"] = json.loads(out[-1])
            print(f"bench_unet_precision {arm}:", out[-1], flush=True)


if __name__ == "__main__":
    main()

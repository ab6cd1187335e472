"""A/B of two builds of libcondmdi_b200.so on the flagship workload, on one GPU.

    python scripts/ab_bench.py A.so B.so [--rounds 5] [--steps 200] [--warmup 10] [--full] [--out DIR]

Each round runs `bench.py --skip-configs` once per build (A, then B) in a subprocess of its own, the library chosen with
CONDMDI_B200_LIB; the builds alternate round by round so that drift of the card's clocks hits both alike.  Per round it
prints steps/s, the clocks bench.py sampled and the per-kernel ms per step of its profiled pass.  Then:
  - outputs: the first round at bf16x3 and one extra run at bf16 dump the samples of the last timed step (same seeds);
    the two builds' sample.npy files are compared byte for byte;
  - one profile pass per build with CMDI_CHAIN_DBG=1, which prints the chained kernel's cycles per tile (warp 0:
    epi0_acc_wait = mainloop, epi0_slices = epilogue, epi0_publish = publish wait);
  - the samplers bench.py does not drive (its workload is DDPM): SAMPLER_SNIPPET runs short loops of DDIM eta = 1 with
    CFG + imputation, PLMS order 4 down to t = 0, DPM-Solver++ order 3 (fused, and the generator, which resumes the
    history), DDIM inversion and a reconstruction-guided loop under each build, same seeds; every tensor is compared
    byte for byte and every launch count exactly;
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


SAMPLER_SNIPPET = r"""
import sys, numpy as np, torch
sys.path.insert(0, sys.argv[1])
import condmdi_b200 as C
from oracle import condmdi_oracle as O
dev = torch.device("cuda", 0)
gi = O.golden_inputs()
B, D, L = gi["x"].shape[0], gi["x"].shape[1], gi["x"].shape[3]
shape = (B, D, 1, L)
m = C.MDM(cond_mode="text", cond_mask_prob=0.1)
m.load_state_dict(O.random_state_dict(seed=7, text=True), strict=False)
m = m.to(dev)
m.encode_text = lambda texts: gi["cond"].to(dev)
w = C.ClassifierFreeSampleModel(m)
eng = m.engine_for(dev, max_batch=B)
x_obs, x_T = gi["x_obs"].to(dev), gi["x"].to(dev)
y = {"text": ["a", "b"], "text_scale": gi["text_scale"].to(dev), "mask": gi["y_mask"].to(dev), "lengths": gi["lengths"],
     "imputate": 1, "stop_imputation_at": 1, "replacement_distribution": "conditional", "inpainted_motion": x_obs,
     "inpainting_mask": gi["kf_mask"].to(dev)}
y_guided = dict(y, reconstruction_guidance=True, reconstruction_weight=20.0, gradient_schedule=None, diffusion_steps=1000,
                stop_recguidance_at=2)
d = C.create_gaussian_diffusion(timestep_respacing="ddim50")
d.rng, d.engine_seed = "engine", 5
out, counts = {}, {}

def record(name, fn):
    n0 = eng.launch_count
    res = fn()
    torch.cuda.synchronize()
    counts[name] = eng.launch_count - n0
    steps = res if isinstance(res, list) else [{"sample": res}]
    for i, st in enumerate(steps):
        for k, v in st.items():
            for j, t in enumerate(v if isinstance(v, (list, tuple)) else [v]):
                out[f"{name}.{i}.{k}.{j}"] = t.cpu().numpy()

kw = dict(model_kwargs={"y": y}, init_image=x_obs)
record("ddim_eta1", lambda: d.ddim_sample_loop(w, shape, eta=1.0, skip_timesteps=44, **kw))
record("ddim_eta1_gen", lambda: list(d.ddim_sample_loop_progressive(w, shape, eta=1.0, skip_timesteps=46, **kw)))
record("plms4", lambda: d.plms_sample_loop(w, shape, noise=x_T, order=4, skip_timesteps=43, **kw))
record("plms4_gen", lambda: list(d.plms_sample_loop_progressive(w, shape, noise=x_T, order=4, skip_timesteps=45, **kw)))
record("plms_first_at_zero", lambda: d.plms_sample_loop(w, shape, noise=x_T, order=4, skip_timesteps=49, **kw))
record("dpm3", lambda: d.dpm_solver_sample_loop(w, shape, noise=x_T, order=3, skip_timesteps=44, **kw))
record("dpm3_gen", lambda: list(d.dpm_solver_sample_loop_progressive(w, shape, noise=x_T, order=3, skip_timesteps=45, **kw)))
record("inversion", lambda: d.ddim_reverse_sample_loop(w, x_obs, model_kwargs={"y": y}))
record("inversion_gen", lambda: list(d.ddim_reverse_sample_loop_progressive(w, x_obs, model_kwargs={"y": y}))[-3:])
kw["model_kwargs"] = {"y": y_guided}
record("guided_ddim", lambda: d.ddim_sample_loop(w, shape, noise=x_T, skip_timesteps=45, **kw))
record("guided_plms", lambda: d.plms_sample_loop(w, shape, noise=x_T, order=3, skip_timesteps=45, **kw))
record("guided_dpm_gen", lambda: list(d.dpm_solver_sample_loop_progressive(w, shape, noise=x_T, order=2, skip_timesteps=45, **kw)))
np.savez(sys.argv[2], **out)
print("launch counts:", counts)
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

    res["samplers"] = samplers(arms, tmp)
    print("samplers (A vs B):", json.dumps(res["samplers"]), flush=True)

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


def samplers(arms, tmp):
    import numpy as np

    counts, dumps = {}, {}
    for arm, lib in arms.items():
        path = os.path.join(tmp, arm, "samplers.npz")
        r_ = run([sys.executable, "-c", SAMPLER_SNIPPET, ROOT, path], lib)
        counts[arm] = r_.stdout.strip().splitlines()[-1]
        dumps[arm] = np.load(path)
    a, b = dumps["A"], dumps["B"]
    differ = sorted(set(a.files) ^ set(b.files)) + [k for k in a.files if k in b.files and a[k].tobytes() != b[k].tobytes()]
    return {"tensors": len(a.files), "tensors_that_differ": differ, "launch_counts_equal": counts["A"] == counts["B"],
            "launch_counts": counts}


if __name__ == "__main__":
    main()

"""TEST INFRASTRUCTURE -- pins the oracle against the UNMODIFIED reference at the model geometries the reference builds
besides HumanML3D's 263 features x 196 frames, and writes tests/golden/geometries.* from the reference's outputs.

Run where the reference tree is available:   python -m oracle.make_golden_geometries

utils/model_util.py:62-76 sets njoints = 263 (humanml), 67 (humanml, drop_redundant), 251 (kit) or 764 (amass), and
sample/gmd/generate.py:110-112 asks for min(196, motion_length * fps) frames.  The cases below cover those widths with
frame counts that are not multiples of 4, 8 or 16, the transformer's longest sequence (207 frames) and the UNet's
unpadded one (224 frames):

    mdm.251x120     MDM trans_enc (8 layers, ff 1024), KIT width, text + classifier-free guidance
    mdm.67x57       MDM trans_enc, drop_redundant width, 57 frames
    mdm.764x207     MDM trans_enc, AMASS width, the longest sequence the engine accepts
    unet.263x120    MDM_UNET (AdaGN) dim_mults (1, 1), keyframe input conditioning
    unet.764x120    MDM_UNET xl, dataset 'amass', keyframe input conditioning (5 * 1528 input taps)
    unet.263x224    MDM_UNET xl, keyframe input conditioning, 224 frames: no padding

Per case: one evaluation at per-sample timesteps [999, 37] (and the CFG-wrapped one where the model has text) and the
last four steps (t = 3 .. 0) of p_sample_loop from a noise tape, with keyframe imputation over ragged lengths (and, for
the UNets, the keyframes as top-level obs_x0 / obs_mask).  The observation masks are seeded random booleans, whole frames
and single features (O.get_keyframes_mask knows only the 263-feature layout).  Weights come from the oracle's seeded
state dicts; only the reference's outputs are stored.
"""
from __future__ import annotations

import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import condmdi_oracle as O  # noqa: E402
from oracle import reference_harness as RH  # noqa: E402
from oracle.golden_io import save_golden  # noqa: E402

GOLDEN = os.path.join(ROOT, "tests", "golden")
B = 2
T_FWD = (999, 37)
SKIP = 996  # p_sample_loop tail: t = 3, 2, 1, 0

# name -> geometry.  kind "mdm": 8-layer trans_enc; kind "unet": AdaGN MDM_UNET
CASES = {
    "mdm.251x120": dict(kind="mdm", D=251, L=120, text=True),
    "mdm.67x57": dict(kind="mdm", D=67, L=57, text=False),
    "mdm.764x207": dict(kind="mdm", D=764, L=207, text=False),
    "unet.263x120": dict(kind="unet", D=263, L=120, mults=(1, 1), dataset="humanml"),
    "unet.764x120": dict(kind="unet", D=764, L=120, mults=(2, 2, 2, 2), dataset="amass"),
    "unet.263x224": dict(kind="unet", D=263, L=224, mults=(2, 2, 2, 2), dataset="humanml"),
}

# the tolerances tests/test_oracle_golden.py holds the oracle to (rtol, atol)
TOL = {"mdm.fwd": (1e-4, 2e-5), "mdm.cfg": (1e-4, 5e-5), "mdm.tail": (1e-4, 5e-5),
       "unet.fwd": (1e-5, 1e-6), "unet.tail": (1e-5, 2e-6)}


def random_obs_mask(g: torch.Generator, batch: int, D: int, L: int, p: float = 0.1) -> torch.Tensor:
    """Seeded observation mask (batch, D, 1, L), about 2p observed: whole frames, and single features anywhere."""
    frames = torch.rand(batch, 1, 1, L, generator=g) < p
    feats = torch.rand(batch, D, 1, L, generator=g) < p
    return frames | feats


def case_inputs(name: str, batch: int = B) -> dict:
    """Seeded inputs of one case (the GPU tests draw theirs from here too)."""
    c = CASES[name]
    D, L = c["D"], c["L"]
    g = torch.Generator().manual_seed(4242 + D * 1000 + L)
    x = torch.randn(batch, D, 1, L, generator=g)
    x_obs = torch.randn(batch, D, 1, L, generator=g)
    tape = torch.randn(1 + 1000 - SKIP, batch, D, 1, L, generator=g)
    cond = torch.randn(batch, 512, generator=g)
    mask = random_obs_mask(g, batch, D, L)
    lengths = torch.tensor([L] + [max(1, (3 * L) // 4 - 7 * i) for i in range(batch - 1)])
    y_mask = (torch.arange(L)[None, :] < lengths[:, None]).view(batch, 1, 1, L)
    scale = torch.tensor([2.5, 0.7] * batch)[:batch]
    return dict(x=x, x_obs=x_obs, tape=tape, cond=cond, mask=mask, lengths=lengths, y_mask=y_mask, text_scale=scale,
                t=torch.tensor(T_FWD * batch)[:batch])


def case_state_dict(name: str) -> dict:
    c = CASES[name]
    if c["kind"] == "mdm":
        return O.random_state_dict(seed=7, feats=c["D"], text=c["text"])
    return O.random_unet_state_dict(seed=11, mults=c["mults"], feats=c["D"], keyframe_conditioned=True)


def case_conditioning(name: str, gi: dict) -> O.Conditioning:
    """What the tail's model_kwargs amount to: imputation of the observed entries inside each length (+ CFG 2.5 / 0.7 for
    the text model, + keyframe input conditioning for the UNets)."""
    c = CASES[name]
    kw = dict(y_mask=gi["y_mask"], imputate=True, stop_imputation_at=1, inpainted_motion=gi["x_obs"], inpainting_mask=gi["mask"])
    if c["kind"] == "unet":
        kw.update(obs_x0=gi["x_obs"], obs_mask=gi["mask"])
    elif c["text"]:
        kw.update(cond_emb=gi["cond"], cfg=True, text_scale=gi["text_scale"])
    return O.Conditioning(**kw)


def oracle_outputs(name: str) -> dict:
    """The oracle's values of every stored array of one case."""
    c, gi, sd = CASES[name], case_inputs(name), case_state_dict(name)
    out = {}
    with torch.no_grad():
        if c["kind"] == "mdm":
            cond = gi["cond"] if c["text"] else None
            out["fwd"] = O.mdm_forward(sd, gi["x"], gi["t"], cond)
            if c["text"]:
                out["fwd_cfg"] = O.cfg_forward(sd, gi["x"], gi["t"], gi["cond"], gi["text_scale"])
        else:
            out["fwd"] = O.unet_forward(sd, gi["x"], gi["t"], None, False, gi["x_obs"], gi["mask"])
    cc = case_conditioning(name, gi)
    out["tail"] = O.sample_loop(sd, O.make_tables(""), tuple(gi["x"].shape), cc, gi["tape"], "ddpm", skip_timesteps=SKIP,
                                init_image=gi["x_obs"])
    return out


def tolerance(name: str, key: str):
    kind = CASES[name]["kind"]
    return TOL[f"{kind}.cfg" if key == "fwd_cfg" else f"{kind}.{key}"]


def reference_outputs(name: str) -> dict:
    ref = RH.import_reference()
    c, gi, sd = CASES[name], case_inputs(name), case_state_dict(name)
    if c["kind"] == "mdm":
        m = RH.build_reference_model(seed=0, text=c["text"], njoints=c["D"])
    else:
        m = RH.build_reference_unet(dim_mults=c["mults"], keyframe_conditioned=True, njoints=c["D"], dataset=c["dataset"])
    missing, unexpected = m.load_state_dict(sd, strict=False)
    assert not missing and not unexpected, (missing, unexpected)
    text = c.get("text", False)
    if text:
        m._synthetic_text_emb = gi["cond"]
    model = ref.cfg_sampler.ClassifierFreeSampleModel(m) if text else m
    obs = {"obs_x0": gi["x_obs"], "obs_mask": gi["mask"]} if c["kind"] == "unet" else {}
    y = {"text": ["a", "b"]} if text else {}
    out = {}
    with torch.no_grad():
        out["fwd"] = m(gi["x"], gi["t"], y=dict(y), **obs)
        if text:
            out["fwd_cfg"] = model(gi["x"], gi["t"], y=dict(y, text_scale=gi["text_scale"]))
    ykw = dict(y, mask=gi["y_mask"], lengths=gi["lengths"], imputate=1, stop_imputation_at=1,
               replacement_distribution="conditional", inpainted_motion=gi["x_obs"], inpainting_mask=gi["mask"])
    if text:
        ykw["text_scale"] = gi["text_scale"]
    diff = RH.build_reference_diffusion("")
    with RH.noise_tape(gi["tape"]):
        out["tail"] = diff.p_sample_loop(model, tuple(gi["x"].shape), model_kwargs=dict(y=ykw, **obs), device="cpu",
                                         clip_denoised=False, skip_timesteps=SKIP, init_image=gi["x_obs"])
    return out


def golden_geometries():
    arrays = {}
    for name in CASES:
        print(name)
        r, o = reference_outputs(name), oracle_outputs(name)
        assert set(r) == set(o)
        for key in r:
            rtol, atol = tolerance(name, key)
            err = (r[key].double() - o[key].double()).abs()
            print(f"  {key:8s} max|ref - oracle| = {err.max():.3e}  mean = {err.mean():.3e}  (held to rtol {rtol:g} / atol {atol:g})")
            assert torch.allclose(o[key], r[key], rtol=rtol, atol=atol), (name, key)
            # one array per sample: a whole 764 x 207 batch would not fit in one fixture file of under 1 MB
            for i, row in enumerate(r[key].numpy()):
                arrays[f"{name}.{key}.{i}"] = row
    save_golden(GOLDEN, "geometries", **arrays)


def fixture(gold: dict, key: str) -> np.ndarray:
    """The batch `key` (e.g. "mdm.764x207.fwd") of the loaded geometries fixture, reassembled from its per-sample arrays."""
    return np.stack([gold[f"{key}.{i}"] for i in range(B)])


def main():
    if not RH.available():
        raise SystemExit("the reference tree is required to (re)generate golden vectors")
    os.makedirs(GOLDEN, exist_ok=True)
    torch.set_num_threads(os.cpu_count() or 1)
    golden_geometries()
    for f in sorted(os.listdir(GOLDEN)):
        if f.startswith("geometries."):
            print(f, os.path.getsize(os.path.join(GOLDEN, f)) // 1024, "KiB")


if __name__ == "__main__":
    main()

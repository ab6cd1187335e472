"""Generate tests/golden/motion_features.* from the UNMODIFIED reference's representation conversions.

Runs, through `reference_harness` (which puts the reference on the path and shims removed numpy aliases):
  * extract_features (data_loaders/humanml/scripts/motion_process.py:50-187) with the 22-joint skeleton arguments
    HumanML3D.__init__ builds (dataset.py:1182-1183);
  * abs3d_to_rel / rel_to_abs3d (dataset.py:1327-1401), whose `dataset` is a namespace carrying what the two functions
    read: Text2MotionDatasetV2.inv_transform with and without use_rand_proj (:378-382, :536-539) and
    HumanML3D.motion_to_rel_data / motion_to_abs_data (:1198-1288, recover_root_rot_pos :402-441), called unbound;
  * rot2xyz stubbed to the identity it is for pose_rep='xyz' (model/rotation2xyz.py).
`spacy` (imported by dataset.py for its text pipeline, not used by these functions) is stubbed.

Inputs are the reference's bundled data: dataset/000021.npy (real joints), t2m_mean / t2m_std (float64, standing in
for the relative statistics), HumanML3D_abs/Mean_abs_3d / Std_abs_3d (float32) and rand_proj / inv_rand_proj.
The script asserts that oracle/motion_features_oracle.py reproduces every output bit for bit.

    python oracle/make_golden_features.py
"""
from __future__ import annotations

import os
import sys
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import motion_features_oracle as MF  # noqa: E402
from oracle import reference_harness as RH  # noqa: E402
from oracle.golden_io import save_golden  # noqa: E402

CONV_CASES = [(196, 2), (57, 2), (2, 2)]   # (frames, batch)


def load_reference():
    RH.import_reference()
    sys.modules.setdefault("spacy", types.ModuleType("spacy"))
    import data_loaders.humanml.data.dataset as ds  # noqa: E402
    import data_loaders.humanml.scripts.motion_process as mp  # noqa: E402
    from data_loaders.humanml.utils.paramUtil import t2m_kinematic_chain, t2m_raw_offsets  # noqa: E402
    return ds, mp, t2m_raw_offsets, t2m_kinematic_chain


def reference_dataset(ds, offsets, chain, mean, std, mean_rel, std_rel, mean_abs, std_abs, inv_proj):
    """The attributes abs3d_to_rel / rel_to_abs3d read from `dataset`, bound to the reference's own methods."""
    t2m = types.SimpleNamespace(mean=mean, std=std, std_scale_shift=(1.0, 0.0), traject_only=False, drop_redundant=False,
                                use_rand_proj=inv_proj is not None, inv_proj_matrix=inv_proj)
    t2m.get_std_mean = lambda traject_only=None, drop_redundant=None: ds.Text2MotionDatasetV2.get_std_mean(t2m, traject_only,
                                                                                                           drop_redundant)
    t2m.inv_random_projection = lambda data, mode="np": ds.Text2MotionDatasetV2.inv_random_projection(t2m, data, mode)
    t2m.inv_transform = lambda data, traject_only=None: ds.Text2MotionDatasetV2.inv_transform(t2m, data, traject_only)
    d = types.SimpleNamespace(t2m_dataset=t2m, n_raw_offsets=torch.from_numpy(offsets), kinematic_chain=chain,
                              mean_rel=mean_rel, std_rel=std_rel, mean_abs=mean_abs, std_abs=std_abs)
    d.motion_to_rel_data = lambda motion, model: ds.HumanML3D.motion_to_rel_data(d, motion, model)
    d.motion_to_abs_data = lambda motion, model: ds.HumanML3D.motion_to_abs_data(d, motion, model)
    return d


def gap(a, b) -> float:
    return float((torch.as_tensor(a).double() - torch.as_tensor(b).double()).abs().max())


def main():
    ds, mp, offsets, chain = load_reference()
    ref = RH.REFERENCE_ROOT
    motion = np.load(os.path.join(ref, "dataset", "000021.npy"))
    mean_rel = np.load(os.path.join(ref, "dataset", "t2m_mean.npy"))
    std_rel = np.load(os.path.join(ref, "dataset", "t2m_std.npy"))
    mean_abs = np.load(os.path.join(ref, "dataset", "HumanML3D_abs", "Mean_abs_3d.npy"))
    std_abs = np.load(os.path.join(ref, "dataset", "HumanML3D_abs", "Std_abs_3d.npy"))
    proj = np.load(os.path.join(ref, "dataset", "rand_proj.npy"))
    inv_proj = np.load(os.path.join(ref, "dataset", "inv_rand_proj.npy"))
    model = types.SimpleNamespace(rot2xyz=lambda x, **kw: x)   # pose_rep='xyz': rot2xyz returns x
    out = dict(mean_rel=mean_rel, std_rel=std_rel, mean_abs=mean_abs, std_abs=std_abs, inv_proj=inv_proj)

    # ---- extract_features ----------------------------------------------------------------------------------------
    joints = MF.fixture_joints(motion)
    for name, j in joints.items():
        want = mp.extract_features(j.copy(), 0.002, torch.from_numpy(offsets), chain, [2, 1, 17, 16], [8, 11], [7, 10])
        got = MF.extract_features(j)
        assert torch.equal(got.double(), torch.from_numpy(want)), (name, gap(got, want))
        out[f"feat.{name}.joints"] = j
        out[f"feat.{name}.features"] = want.astype(np.float32)   # float32 values (contacts 0/1)
        print(f"extract_features[{name}] L={len(j)}: oracle == reference; contacts on: {int(want[:, -4:].sum())}")

    # ---- the two conversions ---------------------------------------------------------------------------------------
    base = MF.ping_pong(joints["real"], 196)
    rng = np.random.default_rng(57)
    for L, B in CONV_CASES:
        # relative samples: the real motion (shifted in time per sequence) through extract_features, normalised
        seqs = np.stack([np.roll(base, 23 * b, axis=0)[:L] if L > 2 else base[40 * b:40 * b + 2] for b in range(B)])
        feats = MF.extract_features(seqs)
        feats = torch.cat((feats, feats[:, -1:]), 1).double()
        rel = ((feats - torch.from_numpy(mean_rel)) / torch.from_numpy(std_rel)).permute(0, 2, 1)[:, :, None, :].float()
        rel = rel + torch.from_numpy(rng.normal(0, 0.02, rel.shape).astype(np.float32))
        # projected inputs are made contiguous, as a sampler output is: np.matmul's summation order depends on the layout
        for use_proj in (False, True):
            tag = f"conv{L}{'.proj' if use_proj else ''}"
            P = inv_proj if use_proj else None
            # rel -> abs (de-normalised with the relative statistics, normalised with the absolute ones)
            x_rel = rel if not use_proj else torch.from_numpy(np.matmul(rel.permute(0, 2, 3, 1).numpy(), proj)).permute(0, 3, 1, 2).contiguous()
            d = reference_dataset(ds, offsets, chain, mean_rel, std_rel, mean_rel, std_rel, mean_abs, std_abs, P)
            want_abs = ds.rel_to_abs3d(x_rel.clone(), d, model)
            got_abs = MF.rel_to_abs3d(x_rel, mean_rel, std_rel, mean_abs, std_abs, P)
            assert torch.equal(got_abs, want_abs), (tag, "rel_to_abs3d", gap(got_abs, want_abs))
            # abs -> rel: the absolute batch just computed, perturbed (and projected), back to the relative statistics
            a = want_abs.float() + torch.from_numpy(rng.normal(0, 0.02, want_abs.shape).astype(np.float32))
            x_abs = a if not use_proj else torch.from_numpy(np.matmul(a.permute(0, 2, 3, 1).numpy(), proj)).permute(0, 3, 1, 2).contiguous()
            d = reference_dataset(ds, offsets, chain, mean_abs, std_abs, mean_rel, std_rel, mean_abs, std_abs, P)
            want_rel = ds.abs3d_to_rel(x_abs.clone(), d, model)
            got_rel = MF.abs3d_to_rel(x_abs, mean_abs, std_abs, mean_rel, std_rel, P)
            assert torch.equal(got_rel, want_rel), (tag, "abs3d_to_rel", gap(got_rel, want_rel))
            # sample_to_motion's positions (inv_transform + recover_from_ric(abs_3d=True)) for sample_to_joints(inv_proj=)
            pos = ds.recover_from_ric(d.t2m_dataset.inv_transform(x_abs.clone().permute(0, 2, 3, 1)).float(), 22, abs_3d=True)
            pos = pos.view(-1, *pos.shape[2:]).permute(0, 2, 3, 1)
            assert torch.equal(MF.sample_to_joints(x_abs, mean_abs, std_abs, True, P), pos), tag
            out.update({f"{tag}.rel_in": x_rel.numpy(), f"{tag}.abs_out": want_abs.float().numpy(),
                        f"{tag}.abs_in": x_abs.numpy(), f"{tag}.rel_out": want_rel.float().numpy(),
                        f"{tag}.joints_abs": pos.float().numpy()})
            print(f"{tag}: rel_to_abs3d {tuple(want_abs.shape)} {want_abs.dtype}, abs3d_to_rel {tuple(want_rel.shape)} "
                  f"{want_rel.dtype}: oracle == reference")
    print("every oracle output is bit-identical to the reference's")
    save_golden(os.path.join(ROOT, "tests", "golden"), "motion_features", **out)


if __name__ == "__main__":
    main()

"""CPU: the representation-conversion restatement (oracle/motion_features_oracle.py) against the reference's outputs in
tests/golden/motion_features.* (made by oracle/make_golden_features.py from the unmodified reference functions)."""
import numpy as np
import pytest
import torch

from oracle import motion_features_oracle as MF
from oracle.golden_io import load_golden

FEAT_CASES = ["real", "pert1", "pert2", "still", "two"]
CONV_TAGS = ["conv196", "conv196.proj", "conv57", "conv57.proj", "conv2", "conv2.proj"]


@pytest.fixture(scope="module")
def g(golden_dir):
    return load_golden(golden_dir, "motion_features")


@pytest.mark.parametrize("name", FEAT_CASES)
def test_extract_features_restatement_matches_reference(g, name):
    got = MF.extract_features(g[f"feat.{name}.joints"])
    assert torch.equal(got, torch.from_numpy(g[f"feat.{name}.features"]))


def test_still_stretch_sets_contacts(g):
    f = g["feat.still.features"]
    assert (f[41:89, -4:] == 1).all()     # frames 40..89 are one pose: every foot is in contact


@pytest.mark.parametrize("tag", CONV_TAGS)
def test_conversion_restatement_matches_reference(g, tag):
    P = g["inv_proj"] if tag.endswith(".proj") else None
    got_abs = MF.rel_to_abs3d(torch.from_numpy(g[f"{tag}.rel_in"]), g["mean_rel"], g["std_rel"], g["mean_abs"], g["std_abs"], P)
    assert torch.equal(got_abs.float(), torch.from_numpy(g[f"{tag}.abs_out"]))
    x_abs = torch.from_numpy(g[f"{tag}.abs_in"])
    got_rel = MF.abs3d_to_rel(x_abs, g["mean_abs"], g["std_abs"], g["mean_rel"], g["std_rel"], P)
    assert torch.equal(got_rel.float(), torch.from_numpy(g[f"{tag}.rel_out"]))
    got_pos = MF.sample_to_joints(x_abs, g["mean_abs"], g["std_abs"], True, P)
    assert torch.equal(got_pos, torch.from_numpy(g[f"{tag}.joints_abs"]))


def test_fixture_files_stay_small(golden_dir):
    import glob
    import os
    files = glob.glob(os.path.join(golden_dir, "motion_features.*"))
    assert files and all(os.path.getsize(f) < 1_000_000 for f in files)
    assert np.load(files[0]).files

"""GPU: extract_features and the absolute <-> relative conversions (csrc/motion_features.cu) against the reference's
outputs (tests/golden/motion_features.*) and against the CPU restatement (oracle/motion_features_oracle.py) at B = 64."""
import numpy as np
import pytest
import torch

import condmdi_b200 as C
from oracle import condmdi_oracle as O
from oracle import motion_features_oracle as MF
from oracle.golden_io import load_golden

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
GATE = dict(rtol=1e-3, atol=1e-4)          # normalised features: the project's gate
FEAT = dict(rtol=1e-4, atol=1e-5)          # de-normalised joints_to_features
GROUPS = {"root": slice(0, 4), "ric": slice(4, 67), "rot": slice(67, 193), "vel": slice(193, 259), "contacts": slice(259, 263)}
FEAT_CASES = ["real", "pert1", "pert2", "still", "two"]
CONV_TAGS = ["conv196", "conv196.proj", "conv57", "conv57.proj", "conv2", "conv2.proj"]


@pytest.fixture(scope="module")
def g(golden_dir):
    return load_golden(golden_dir, "motion_features")


def report(what, got, want, channel_dim):
    """Print max / mean |error| per channel group."""
    d = (torch.as_tensor(got).double().cpu() - torch.as_tensor(want).double()).abs()
    parts = []
    for name, sl in GROUPS.items():
        e = d.narrow(channel_dim, sl.start, sl.stop - sl.start)
        parts.append(f"{name} {e.max().item():.1e}/{e.mean().item():.1e}")
    print(f"{what}: max/mean |err| " + ", ".join(parts))


def near_threshold(joints: np.ndarray, thre: float = MF.FEET_THRE) -> np.ndarray:
    """(B, L, 22, 3) -> (B, L-1, 4) bool: the squared foot displacement lies within 1e-6 relative of the threshold."""
    fid = list(MF.FID_L) + list(MF.FID_R)
    d = joints[:, 1:, fid] - joints[:, :-1, fid]
    s = d[..., 0] ** 2 + d[..., 1] ** 2 + d[..., 2] ** 2
    return np.abs(s.astype(np.float64) - thre) <= 1e-6 * thre


def check_contacts(what, got, want, near):
    """Contacts (..., rows, 4) bit-equal except where the reference's displacement sits on the threshold."""
    got, want = np.asarray(got), np.asarray(want)
    diff = got != want
    n_near = int(near.sum())
    print(f"{what}: {n_near} contact element(s) within 1e-6 relative of the threshold, {int(diff.sum())} differ")
    assert not (diff & ~near).any()
    assert n_near <= max(4, near.size // 1000)


def close(got, want, rtol, atol, mask=None):
    got = torch.as_tensor(got).double().cpu()
    want = torch.as_tensor(want).double()
    ok = (got - want).abs() <= atol + rtol * want.abs()
    if mask is not None:
        ok |= mask
    return bool(ok.all())


def joints_of(sample: torch.Tensor, mean, std, abs_3d: bool, P) -> np.ndarray:
    """The positions extract_features sees inside a conversion (CPU restatement): (B, L, 22, 3)."""
    return O.recover_from_ric(MF.inv_transform(sample, mean, std, P), 22, abs_3d)[:, 0].numpy()


def conditioning_mask(got, want, std, what):
    """Gate misses the B = 64 comparison accepts, and bounds: the root velocities (channels 0..2) have dataset std
    5e-4..7e-4, so one float32 ulp of an input position moves them by ~3.5e-4 normalised, more than the gate's atol.
    (On the L = 224 projected batch, perturbing the inputs by 1.2e-7 relative makes 15091 elements of the CPU
    restatement's own output leave the gate.)  A miss must be in those channels, within 4e-6 once de-normalised, and
    rare."""
    got = torch.as_tensor(got).double().cpu()
    want = torch.as_tensor(want).double()
    miss = (got - want).abs() > GATE["atol"] + GATE["rtol"] * want.abs()
    n = int(miss.sum())
    s = torch.as_tensor(np.asarray(std, dtype=np.float64)).view(1, -1, 1, 1)
    denorm = ((got - want).abs() * s)[miss]
    print(f"{what}: {n} gate miss(es) in root-velocity channels, de-normalised max "
          f"{denorm.max().item() if n else 0.0:.1e}")
    assert not miss[:, 3:].any()
    assert n <= miss[:, :3].numel() // 1000
    assert n == 0 or denorm.max().item() <= 4e-6
    return miss


def contact_mask(near: np.ndarray, L: int) -> torch.Tensor:
    """(B, L-1, 4) near-threshold flags -> a (B, 263, 1, L) mask over the converted layout (last row duplicated)."""
    m = torch.zeros(near.shape[0], 263, 1, L, dtype=torch.bool)
    n = torch.from_numpy(near).permute(0, 2, 1)
    m[:, 259:, 0, :L - 1] = n
    m[:, 259:, 0, L - 1] = n[:, :, -1]
    return m


# ---- extract_features ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", FEAT_CASES)
def test_joints_to_features_vs_reference(g, name):
    j = g[f"feat.{name}.joints"]
    want = g[f"feat.{name}.features"]
    got = C.joints_to_features(torch.from_numpy(j).to(DEV))
    assert got.is_cuda and got.shape == want.shape
    report(f"joints_to_features[{name}]", got, want, -1)
    got = got.cpu()
    assert close(got[:, :259], want[:, :259], **FEAT)
    check_contacts(f"joints_to_features[{name}]", got[:, 259:].numpy(), want[:, 259:], near_threshold(j[None])[0])
    if name == "still":
        assert (got[41:89, 259:] == 1).all()


# ---- the conversions against the reference's outputs ------------------------------------------------------------------
@pytest.mark.parametrize("tag", CONV_TAGS)
def test_rel_to_abs3d_vs_reference(g, tag):
    P = g["inv_proj"] if tag.endswith(".proj") else None
    x = torch.from_numpy(g[f"{tag}.rel_in"])
    want = g[f"{tag}.abs_out"]
    got = C.rel_to_abs3d(x.to(DEV), g["mean_rel"], g["std_rel"], g["mean_abs"], g["std_abs"], inv_proj=P)
    assert got.is_cuda and got.shape == want.shape
    report(f"rel_to_abs3d[{tag}]", got, want, 1)
    near = near_threshold(joints_of(x, g["mean_rel"], g["std_rel"], False, P))
    check_contacts(f"rel_to_abs3d[{tag}]", got.cpu()[:, 259:, 0, :-1].permute(0, 2, 1).numpy(),
                   torch.from_numpy(want)[:, 259:, 0, :-1].permute(0, 2, 1).numpy(), near)
    assert close(got, want, **GATE, mask=contact_mask(near, x.shape[-1]))


@pytest.mark.parametrize("tag", CONV_TAGS)
def test_abs3d_to_rel_vs_reference(g, tag):
    P = g["inv_proj"] if tag.endswith(".proj") else None
    x = torch.from_numpy(g[f"{tag}.abs_in"])
    want = g[f"{tag}.rel_out"]
    got = C.abs3d_to_rel(x.to(DEV), g["mean_abs"], g["std_abs"], g["mean_rel"], g["std_rel"], inv_proj=P)
    assert got.is_cuda and got.shape == want.shape
    report(f"abs3d_to_rel[{tag}]", got, want, 1)
    near = near_threshold(joints_of(x, g["mean_abs"], g["std_abs"], True, P))
    check_contacts(f"abs3d_to_rel[{tag}]", got.cpu()[:, 259:, 0, :-1].permute(0, 2, 1).numpy(),
                   torch.from_numpy(want)[:, 259:, 0, :-1].permute(0, 2, 1).numpy(), near)
    assert close(got, want, **GATE, mask=contact_mask(near, x.shape[-1]))
    # the duplicated last row (dataset.py:1214)
    assert torch.equal(got[..., -1], got[..., -2])


@pytest.mark.parametrize("tag", ["conv196.proj", "conv57.proj"])
def test_sample_to_joints_with_inv_proj_vs_reference(g, tag):
    x = torch.from_numpy(g[f"{tag}.abs_in"]).to(DEV)
    got = C.sample_to_joints(x, g["mean_abs"], g["std_abs"], 22, True, inv_proj=g["inv_proj"])
    want = g[f"{tag}.joints_abs"]
    assert got.shape == want.shape
    assert close(got, want, rtol=1e-4, atol=1e-4), (got.cpu() - torch.from_numpy(want)).abs().max()


# ---- B = 64 against the CPU restatement ---------------------------------------------------------------------------------
def batch64(g, L: int, seed: int):
    """64 relative-representation motions: the bundled motion, time-shifted and perturbed, normalised."""
    rng = np.random.default_rng(seed)
    base = MF.ping_pong(g["feat.real.joints"], 360)
    seqs = np.stack([base[(5 * b) % 130:(5 * b) % 130 + L] for b in range(64)]).astype(np.float32)
    seqs += rng.normal(0, 0.01, seqs.shape).astype(np.float32)
    f = MF.extract_features(seqs)
    f = torch.cat((f, f[:, -1:]), 1).double()
    rel = ((f - torch.from_numpy(g["mean_rel"])) / torch.from_numpy(g["std_rel"])).permute(0, 2, 1)[:, :, None, :].float()
    return rel + torch.from_numpy(rng.normal(0, 0.02, rel.shape).astype(np.float32))


def project(x: torch.Tensor, P) -> torch.Tensor:
    if P is None:
        return x
    return torch.from_numpy(np.matmul(x.permute(0, 2, 3, 1).numpy(), np.linalg.inv(P.astype(np.float64)).astype(np.float32))
                            ).permute(0, 3, 1, 2).contiguous()


@pytest.mark.parametrize("L", [196, 224])
@pytest.mark.parametrize("proj", [False, True])
def test_conversions_b64_vs_oracle(g, L, proj):
    P = g["inv_proj"] if proj else None
    rel = project(batch64(g, L, seed=L + proj), P)
    want_abs = MF.rel_to_abs3d(rel, g["mean_rel"], g["std_rel"], g["mean_abs"], g["std_abs"], P)
    got_abs = C.rel_to_abs3d(rel.to(DEV), g["mean_rel"], g["std_rel"], g["mean_abs"], g["std_abs"], inv_proj=P)
    report(f"rel_to_abs3d B=64 L={L} proj={proj}", got_abs, want_abs, 1)
    near = near_threshold(joints_of(rel, g["mean_rel"], g["std_rel"], False, P))
    check_contacts(f"rel_to_abs3d B=64 L={L}", got_abs.cpu()[:, 259:, 0, :-1].permute(0, 2, 1).numpy(),
                   want_abs.float()[:, 259:, 0, :-1].permute(0, 2, 1).numpy(), near)
    miss = conditioning_mask(got_abs, want_abs, g["std_abs"], f"rel_to_abs3d B=64 L={L} proj={proj}")
    assert close(got_abs, want_abs, **GATE, mask=contact_mask(near, L) | miss)

    ab = project(want_abs.float(), P)
    want_rel = MF.abs3d_to_rel(ab, g["mean_abs"], g["std_abs"], g["mean_rel"], g["std_rel"], P)
    got_rel = C.abs3d_to_rel(ab.to(DEV), g["mean_abs"], g["std_abs"], g["mean_rel"], g["std_rel"], inv_proj=P)
    report(f"abs3d_to_rel B=64 L={L} proj={proj}", got_rel, want_rel, 1)
    near = near_threshold(joints_of(ab, g["mean_abs"], g["std_abs"], True, P))
    check_contacts(f"abs3d_to_rel B=64 L={L}", got_rel.cpu()[:, 259:, 0, :-1].permute(0, 2, 1).numpy(),
                   want_rel.float()[:, 259:, 0, :-1].permute(0, 2, 1).numpy(), near)
    miss = conditioning_mask(got_rel, want_rel, g["std_rel"], f"abs3d_to_rel B=64 L={L} proj={proj}")
    assert close(got_rel, want_rel, **GATE, mask=contact_mask(near, L) | miss)


@pytest.mark.parametrize("L", [2, 57, 196, 224])
def test_joints_to_features_b64_vs_oracle(g, L):
    base = MF.ping_pong(g["feat.pert1.joints"], 420)
    j = np.stack([base[3 * b:3 * b + L] for b in range(64)]).astype(np.float32)
    want = MF.extract_features(j)
    got = C.joints_to_features(torch.from_numpy(j).to(DEV))
    report(f"joints_to_features B=64 L={L}", got, want, -1)
    got = got.cpu()
    assert close(got[..., :259], want[..., :259], **FEAT)
    check_contacts(f"joints_to_features B=64 L={L}", got[..., 259:].numpy(), want[..., 259:].numpy(), near_threshold(j))


# ---- determinism, limits, and the unchanged sample_to_joints ----------------------------------------------------------
def test_two_calls_are_bit_identical(g):
    P = g["inv_proj"]
    x = torch.from_numpy(g["conv196.proj.abs_in"]).to(DEV)
    a = C.abs3d_to_rel(x, g["mean_abs"], g["std_abs"], g["mean_rel"], g["std_rel"], inv_proj=P)
    b = C.abs3d_to_rel(x, g["mean_abs"], g["std_abs"], g["mean_rel"], g["std_rel"], inv_proj=P)
    assert torch.equal(a, b)
    y = torch.from_numpy(g["conv196.rel_in"]).to(DEV)
    a = C.rel_to_abs3d(y, g["mean_rel"], g["std_rel"], g["mean_abs"], g["std_abs"])
    b = C.rel_to_abs3d(y, g["mean_rel"], g["std_rel"], g["mean_abs"], g["std_abs"])
    assert torch.equal(a, b)
    j = torch.from_numpy(g["feat.real.joints"]).to(DEV)
    assert torch.equal(C.joints_to_features(j), C.joints_to_features(j))


def test_limits_and_cpu_tensors_raise(g):
    stats = (g["mean_abs"], g["std_abs"], g["mean_rel"], g["std_rel"])
    with pytest.raises(RuntimeError, match="CUDA"):
        C.abs3d_to_rel(torch.zeros(1, 263, 1, 196), *stats)
    with pytest.raises(RuntimeError, match="CUDA"):
        C.joints_to_features(torch.zeros(1, 196, 22, 3))
    for L in (1, 225):
        with pytest.raises(RuntimeError, match=r"2 <= nframes <= 224"):
            C.abs3d_to_rel(torch.zeros(1, 263, 1, L, device=DEV), *stats)
        with pytest.raises(RuntimeError, match=r"2 <= nframes <= 224"):
            C.rel_to_abs3d(torch.zeros(1, 263, 1, L, device=DEV), *stats)
        with pytest.raises(RuntimeError, match=r"2 <= nframes <= 224"):
            C.joints_to_features(torch.zeros(1, L, 22, 3, device=DEV))
    with pytest.raises(RuntimeError, match="joints_num must be 22"):
        C.joints_to_features(torch.zeros(1, 10, 21, 3, device=DEV))


def test_sample_to_joints_without_inv_proj_is_unchanged():
    gen = torch.Generator().manual_seed(9)
    sample = torch.randn(8, 263, 1, 196, generator=gen).to(DEV)
    mean, std = torch.randn(263, generator=gen) * 0.3, torch.rand(263, generator=gen) * 0.2 + 0.01
    for abs_3d in (False, True):
        got = C.sample_to_joints(sample, mean, std, 22, abs_3d)
        # the path it always took: x * std + mean fused into cmdi_recover_from_ric (separately rounded, as below)
        x = sample.permute(0, 2, 3, 1) * std.to(DEV) + mean.to(DEV)
        want = C.recover_from_ric(x, 22, abs_3d)
        assert torch.equal(got, want.reshape(-1, 196, 22, 3).permute(0, 2, 3, 1))

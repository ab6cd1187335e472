"""CPU: the overlapping-window restatement (oracle/windowed_oracle.py) and the package's Window option: placement,
tent weights, one window == the plain restatement bit for bit, shared frames agreeing bit for bit, and the argument
errors."""
import pytest
import torch

import condmdi_b200 as C
from oracle import condmdi_oracle as O
from oracle import windowed_oracle as W


@pytest.mark.parametrize("n,F,O_", [(600, 196, 48), (196, 196, 0), (197, 196, 98), (400, 196, 0), (1000, 207, 103),
                                    (250, 120, 60), (33, 8, 4), (7, 8, 2), (9, 1, 0), (300, 224, 112)])
def test_placement_covers_every_frame_with_overlaps_of_at_least_O(n, F, O_):
    f0 = W.placement(n, F, O_)
    assert f0 == C.Window(F, O_).placement(n)
    if n <= F:
        assert f0 == [0]
        return
    step = F - O_
    assert len(f0) == 1 + -(-(n - F) // step)
    assert f0[0] == 0 and f0[-1] == n - F
    assert all(b > a for a, b in zip(f0, f0[1:]))
    assert all(a + F - b >= O_ for a, b in zip(f0, f0[1:]))  # adjacent windows share at least O frames
    covered = torch.zeros(n, dtype=torch.int64)
    for f in f0:
        covered[f:f + F] += 1
    assert bool((covered >= 1).all())


def test_issue_geometry_and_three_way_cover():
    assert W.placement(600, 196, 48) == [0, 148, 296, 404]  # K = 4: the bench's 16 x 600 frames -> 64 window rows
    f0 = W.placement(250, 120, 60)  # the end-aligned window overlaps two others
    assert f0 == [0, 60, 120, 130]
    cover = [sum(f <= g < f + 120 for f in f0) for g in range(250)]
    assert max(cover) == 3


def test_weights_are_exact_integers_in_fp32():
    for F in (1, 2, 8, 196, 207, 224):
        w = W.weights([0, 5], F)
        assert w.dtype == torch.float32
        assert torch.equal(w, w.round()) and torch.equal(w.double(), w.double().round())
        assert w[0, 0] == 1 and w[0, F - 1] == 1 and w.max() == (F + 1) // 2
        # sums of up to 3 weights stay exact (integers below 2^24)
        assert float(w.sum(0).max()) == float(w.double().sum(0).max())


def test_blend_keeps_singly_covered_frames_and_agrees_on_shared_ones():
    g = torch.Generator().manual_seed(5)
    f0, F, n = [0, 6, 12, 14], 10, 24
    x0 = torch.randn(2 * len(f0), 3, 1, F, generator=g)
    out = W.blend(x0, f0, n)
    xw, ow = x0.view(2, 4, 3, 1, F), out.view(2, 4, 3, 1, F)
    for gf in range(n):
        cover = [k for k in range(4) if f0[k] <= gf < f0[k] + F]
        vals = [ow[:, k, ..., gf - f0[k]] for k in cover]
        if len(cover) == 1:
            assert torch.equal(vals[0], xw[:, cover[0], ..., gf - f0[cover[0]]])
        for v in vals[1:]:
            assert torch.equal(v, vals[0])
    # frame 15 is covered by windows 1, 2, 3 at local frames 9, 3, 1: weights 1, 4, 2
    want = (1 * xw[:, 1, ..., 9] + 4 * xw[:, 2, ..., 3]) + 2 * xw[:, 3, ..., 1]
    assert torch.equal(ow[:, 1, ..., 9], want / 7)


def _tiny():
    sd = O.random_state_dict(seed=3, layers=2, d=64, ff=128, feats=8, text=True)
    return sd


def test_one_window_is_the_plain_restatement_bit_for_bit():
    sd = _tiny()
    g = torch.Generator().manual_seed(9)
    B, D, L = 2, 8, 24
    tab = O.make_tables("ddim5")
    tape = torch.randn(6, B, D, 1, L, generator=g)
    c = O.Conditioning(cond_emb=torch.randn(B, 512, generator=g), cfg=True, text_scale=torch.tensor([2.5, 0.5]))
    for sampler in ("ddpm", "ddim"):
        plain = O.sample_loop(sd, tab, (B, D, 1, L), c, tape, sampler=sampler)
        win = W.sample_loop(sd, tab, (B, D, 1, L), c, tape, W.placement(L, 30, 10), 24, sampler=sampler)
        assert torch.equal(plain, win)


def test_windowed_restatement_agrees_on_shared_frames():
    sd = _tiny()
    g = torch.Generator().manual_seed(10)
    B, D, N, F = 2, 8, 40, 16
    f0 = W.placement(N, F, 6)
    K = len(f0)
    assert f0 == [0, 10, 20, 24]
    tab = O.make_tables("ddim5")
    tape = torch.randn(6, B, D, 1, N, generator=g)
    x_obs = torch.randn(B, D, 1, N, generator=g)
    kf = torch.rand(B, D, 1, N, generator=g) < 0.3
    c = O.Conditioning(cond_emb=torch.randn(B, 512, generator=g), cfg=True, text_scale=torch.tensor([2.5, 0.5]), imputate=True,
                       inpainted_motion=x_obs, inpainting_mask=kf)
    xw = W.sample_loop(sd, tab, (B, D, 1, N), c, tape, f0, F, sampler="ddpm", windows=True).view(B, K, D, 1, F)
    for gf in range(N):
        cover = [k for k in range(K) if f0[k] <= gf < f0[k] + F]
        for k in cover[1:]:
            assert torch.equal(xw[:, k, ..., gf - f0[k]], xw[:, cover[0], ..., gf - f0[cover[0]]])
    out = W.gather(xw.reshape(B * K, D, 1, F), f0, N)
    assert out.shape == (B, D, 1, N)
    assert torch.equal(W.crop(out, f0, F), xw.reshape(B * K, D, 1, F))


@pytest.mark.parametrize("args,match", [((0, 0), "frames must be >= 1"), ((10, 6), r"overlap must be in \[0, frames // 2 = 5\]"),
                                        ((10, -1), "overlap must be in"), ((10.0, 2), "frames must be an int"),
                                        ((10, True), "overlap must be an int"), (("196", 0), "frames must be an int")])
def test_window_argument_errors(args, match):
    with pytest.raises(ValueError, match=match):
        C.Window(*args)


def test_window_defaults_and_overlap_limit():
    w = C.Window(frames=196)
    assert w.overlap == 0
    assert C.Window(196, 98).placement(600) == [0, 98, 196, 294, 392, 404]
    d = C.create_gaussian_diffusion(timestep_respacing="ddim20")
    assert d.window is None


def test_out_of_scope_entry_points_refuse_windows():
    d = C.create_gaussian_diffusion(timestep_respacing="ddim20")
    d.window = C.Window(196, 48)
    with pytest.raises(NotImplementedError, match="overlapping windows"):
        C.sharded_sample(d, None, (2, 263, 1, 600))
    with pytest.raises(NotImplementedError, match="overlapping windows"):
        C.run_eval_jobs(d, None, [])


@pytest.fixture(scope="module")
def gold(golden_dir):
    from oracle.golden_io import load_golden
    return load_golden(golden_dir, "windowed")


@pytest.mark.parametrize("name", sorted(W.FIXTURES))
def test_restatement_equals_the_reference_driven_fixtures(name, gold):
    """tests/golden/windowed.*: the unmodified reference's p_sample / ddim_sample on the window rows, blended by a shim
    around its p_mean_variance (oracle/make_golden_windowed.py)"""
    x_obs, _, cond_w, _, tape = W.fixture_inputs(name)
    want = [float(x_obs.double().sum()), float(tape.double().sum()), float(cond_w.double().sum())]
    assert gold[f"{name}.checksum"].tolist() == want  # the fixture was made from these inputs
    unet = W.FIXTURES[name][-1]
    sd = O.random_unet_state_dict(seed=11, text=True) if unet else O.random_state_dict(seed=7, text=True)
    got = W.fixture_restatement(name, sd)
    err = (got.double() - torch.as_tensor(gold[f"{name}.ref"]).double()).abs().max().item()
    print(f"[{name}] max|restatement - reference| = {err:.3e}")
    assert err <= 2e-5


def test_fixtures_cover_the_issue_geometries():
    geo = {name: W.placement(*W.FIXTURES[name][:3]) for name in W.FIXTURES}
    assert len(geo["text_k2"]) == 2
    f0, F = geo["guided_k3"], W.FIXTURES["guided_k3"][1]
    assert len(f0) == 3 and f0[-1] == W.FIXTURES["guided_k3"][0] - F
    assert max(sum(f <= g < f + F for f in f0) for g in range(W.FIXTURES["guided_k3"][0])) == 3


def test_blend_reaches_every_sampler_restatement():
    from oracle import dpm_solver_oracle, dpm_solver_sde_oracle, plms_oracle, unipc_oracle
    mods = (O, plms_oracle, dpm_solver_oracle, unipc_oracle, dpm_solver_sde_oracle)
    plain = [m.p_mean_variance for m in mods]
    with W.blended([0, 4], 12):
        assert all(m.p_mean_variance is O.p_mean_variance for m in mods) and O.p_mean_variance is not plain[0]
    assert [m.p_mean_variance for m in mods] == plain


def test_per_window_prompts_with_one_window():
    from condmdi_b200.diffusion import _window_prompts
    assert _window_prompts([["a"], ["b"]], 2, 1) == ["a", "b"]
    assert _window_prompts(["a", "b"], 2, 1) == ["a", "b"]
    assert _window_prompts([["a", "b"], ["c", "d"]], 2, 2) == ["a", "b", "c", "d"]
    assert _window_prompts(["a", "b"], 2, 3) == ["a", "a", "a", "b", "b", "b"]
    with pytest.raises(ValueError, match="one entry per sample"):
        _window_prompts(["a"], 2, 1)

"""CPU: the RePaint restatement in oracle/repaint_oracle.py.

- The walk builder: op counts, +-1 moves, the end at -1, jump points under skip_timesteps, jump_n_sample = 1 as the plain
  descent, and the package's own walk (which its generators use to split and count draws) equal to it.
- jump_n_sample = 1 equals the restated p_sample_loop bit for bit; the undo op equals its formula.
- The restatement against tests/golden/repaint.* -- the UNMODIFIED reference's p_sample driven along the walk
  (oracle/make_golden_repaint.py).
- The exact law of the samples on correlated Gaussian data with imputation and the exact denoiser, against a Monte Carlo
  run of the restatement, and its distance to the true conditional law as jump_n_sample grows.
- The argument errors of the public loops, and install().
"""
import numpy as np
import pytest
import torch

import condmdi_b200 as C
from condmdi_b200 import diffusion as CD
from oracle import condmdi_oracle as O
from oracle import repaint_oracle as R
from oracle.golden_io import load_golden
from standin import StockDiffusion

B, D, L = 2, 263, 196
SHAPE = (B, D, 1, L)
# measured when the fixtures were written (oracle/make_golden_repaint.py prints the per-case gaps)
ANCHOR_TOL = 2e-5


@pytest.fixture(scope="module")
def gold(golden_dir):
    return load_golden(golden_dir, "repaint")


@pytest.fixture(scope="module")
def gi(gold):
    gi = O.golden_inputs()
    chk = np.array([float(gi["x"].double().sum()), float(gi["tape"].double().sum()), float(gi["cond"].double().sum())])
    assert np.allclose(chk, gold["inputs.checksum"], rtol=0, atol=1e-9), "seeded inputs differ from the fixtures' inputs"
    return gi


def cycled(gi, n):
    return gi["tape"][torch.arange(n + 1) % 8]


def maxerr(a, b):
    return (torch.as_tensor(a).double() - torch.as_tensor(b).double()).abs().max().item()


# ------------------------------------------------------------------------------------------------
# the walk
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("t0, j, r", [(49, 5, 3), (49, 10, 10), (9, 4, 3), (5, 3, 2), (4, 2, 2), (9, 10, 5), (9, 9, 2),
                                      (0, 1, 4), (1, 1, 3), (999, 10, 10), (37, 7, 1), (20, 1, 1)])
def test_walk_counts_moves_and_end(t0, j, r):
    walk = R.build_walk(t0, j, r)
    n_denoise, n_undo = R.op_counts(t0, j, r)
    K = t0 // j if j <= t0 else 0
    assert n_denoise == t0 + 1 + (r - 1) * j * K and n_undo == (r - 1) * j * K
    assert sum(k == R.DENOISE for k, _ in walk) == n_denoise and sum(k == R.UNDO for k, _ in walk) == n_undo
    pos = t0
    for kind, p in walk:
        if kind == R.DENOISE:
            assert p == pos  # denoise at the current position, which moves down by one
            pos -= 1
        else:
            assert p == pos + 1 and 1 <= p <= t0  # undo into the position above; never out of -1
            pos += 1
    assert pos == -1 and walk[-1] == (R.DENOISE, 0)
    # every step is denoised r times inside a jumped stretch, once outside
    jumped = {u for t in range(0, t0 + 1) if t % j == 0 and t + j <= t0 for u in range(t + 1, t + j + 1)}
    for p in range(t0 + 1):
        assert sum(1 for k, q in walk if k == R.DENOISE and q == p) == (r if p in jumped else 1), p
    # the package's walk (diffusion._repaint_walk, the engine's schedule) is the same
    assert CD._repaint_walk(t0, j, r) == [(p, k == R.UNDO) for k, p in walk]


def test_jump_points_respect_skip_timesteps():
    """a walk started at t0 = T - 1 - skip only jumps from t with t + j <= t0: never above its start"""
    for skip in (0, 3, 40, 45):
        t0 = 49 - skip
        walk = R.build_walk(t0, 5, 3)
        assert max(p for _, p in walk) == t0
        starts = sorted({p - 1 for i, (k, p) in enumerate(walk) if k == R.UNDO and (i == 0 or walk[i - 1][0] == R.DENOISE)})
        assert starts == [t for t in range(0, t0 + 1, 5) if t + 5 <= t0]


@pytest.mark.parametrize("t0, j", [(49, 5), (9, 4), (0, 3), (12, 1)])
def test_one_sample_is_the_plain_descent(t0, j):
    assert R.build_walk(t0, j, 1) == [(R.DENOISE, p) for p in range(t0, -1, -1)]


def test_walk_example():
    assert R.build_walk(5, 3, 2) == [(R.DENOISE, 5), (R.DENOISE, 4), (R.DENOISE, 3), (R.DENOISE, 2), (R.DENOISE, 1),
                                     (R.UNDO, 1), (R.UNDO, 2), (R.UNDO, 3), (R.DENOISE, 3), (R.DENOISE, 2),
                                     (R.DENOISE, 1), (R.DENOISE, 0)]


# ------------------------------------------------------------------------------------------------
# the loop
# ------------------------------------------------------------------------------------------------
def test_one_sample_equals_p_sample_loop_bit_for_bit(gi):
    sd = O.random_state_dict(seed=7, text=False, layers=2)
    tab = O.make_tables("ddim50")
    tape = cycled(gi, 6)
    for skip in (44, 46):
        want = O.sample_loop(sd, tab, SHAPE, O.Conditioning(), tape, "ddpm", skip_timesteps=skip, init_image=gi["x_obs"])
        got = R.repaint_sample_loop(sd, tab, SHAPE, O.Conditioning(), tape, 3, 1, skip_timesteps=skip, init_image=gi["x_obs"])
        assert torch.equal(got, want)


def test_undo_matches_its_formula():
    for resp in ("ddim50", "ddim20", ""):
        tab = O.make_tables(resp)
        a, b = R.undo_coefficients(tab)
        assert a.dtype == torch.float32 and b.dtype == torch.float32
        assert torch.equal(a, torch.tensor([np.float32(np.sqrt(1.0 - x)) for x in tab.betas]))
        assert torch.equal(b, torch.tensor([np.float32(np.sqrt(x)) for x in tab.betas]))
        # one forward step of the spaced chain: a^2 + b^2 = 1 to fp32 rounding
        assert (a.double() ** 2 + b.double() ** 2 - 1).abs().max() < 1e-6
    g = torch.Generator().manual_seed(3)
    x, z = torch.randn(2, 1000, generator=g)
    a_p, b_p = torch.tensor(0.75, dtype=torch.float32), torch.tensor(0.6614378, dtype=torch.float32)
    got = R.undo(x, a_p, b_p, z)
    want = torch.from_numpy(np.float32(np.float32(0.75) * x.numpy()) + np.float32(np.float32(0.6614378) * z.numpy()))
    assert torch.equal(got, want)


def test_walk_records_each_denoise_op(gi):
    sd = O.random_state_dict(seed=7, text=False, layers=2)
    tab = O.make_tables("ddim50")
    walk = R.build_walk(4, 2, 2)
    tape = cycled(gi, len(walk))
    outs = R.repaint_sample_loop(sd, tab, SHAPE, O.Conditioning(), tape, 2, 2, skip_timesteps=45, return_all=True)
    assert [o["t"] for o in outs] == [p for k, p in walk if k == R.DENOISE]
    assert torch.equal(outs[-1]["sample"], outs[-1]["pred_xstart"])  # step 0 returns x0


@pytest.mark.parametrize("name", ["no_cond", "cfg_impute", "guided", "unet"])
def test_restatement_vs_reference_golden(gold, gi, name):
    skip, j, r = (int(v) for v in gold[f"{name}.config"])
    kw = dict(cond_emb=gi["cond"], cfg=True, text_scale=gi["text_scale"], y_mask=gi["y_mask"], imputate=True,
              stop_imputation_at=1, inpainted_motion=gi["x_obs"], inpainting_mask=gi["kf_mask"])
    if name == "no_cond":
        sd, c = O.random_state_dict(seed=7, text=False), O.Conditioning()
    elif name == "cfg_impute":
        sd, c = O.random_state_dict(seed=7, text=True), O.Conditioning(**kw)
    elif name == "guided":
        sd = O.random_state_dict(seed=7, text=True)
        c = O.Conditioning(reconstruction_guidance=True, reconstruction_weight=20.0, stop_recguidance_at=2, **kw)
    else:
        sd = O.random_unet_state_dict(seed=11, text=True)
        c = O.Conditioning(cond_emb=gi["cond"], cfg=True, text_scale=gi["text_scale"], obs_x0=gi["x_obs"],
                           obs_mask=gi["kf_mask"])
    n_ops = len(R.build_walk(49 - skip, j, r))
    got = R.repaint_sample_loop(sd, O.make_tables("ddim50"), SHAPE, c, cycled(gi, n_ops), j, r, skip_timesteps=skip,
                                init_image=gi["x_obs"] if skip else None)
    err = maxerr(got, gold[f"{name}.ref"])
    print(f"[{name}] skip {skip}, j {j}, r {r}: |restatement - reference p_sample walk| = {err:.3e}")
    assert err <= ANCHOR_TOL


# ------------------------------------------------------------------------------------------------
# the exact law on correlated Gaussian data
# ------------------------------------------------------------------------------------------------
N_DIM = 4
_idx = np.arange(N_DIM)
COV = 0.25 * 0.9 ** np.abs(_idx[:, None] - _idx[None, :]) + 0.01 * np.eye(N_DIM)  # strongly correlated neighbours
MU = np.array([0.5, -0.3, 0.2, 0.4])
MASK = np.array([True, False, False, True])  # coordinates 0 and 3 observed and imputed, 1 and 2 generated
X_OBS = np.array([1.2, 0.0, 0.0, -0.6])


def _distances(tab, j, r):
    m, S = R.gaussian_law(tab, MU, COV, MASK, X_OBS, j, r)
    U = ~MASK
    cm, cS = R.conditional_law(MU, COV, MASK, X_OBS)
    return R.gaussian_kl(m[U], S[np.ix_(U, U)], cm, cS), np.abs(m[U] - cm).max(), np.abs(S[np.ix_(U, U)] - cS).max()


def test_exact_law_agrees_with_monte_carlo_of_the_restatement():
    """the walk's loop (run_walk, undo) on 400k samples with the exact imputed denoiser in p_sample's arithmetic, against
    the propagated mean and covariance; observed coordinates end exactly at x_obs"""
    tab = O.make_tables("ddim50")
    j, r, n = 5, 5, 400_000
    g = torch.Generator().manual_seed(17)
    a, b = R.undo_coefficients(tab)

    def denoise(x, p, z):
        A, c = R.exact_denoiser(tab, p, MU, COV, MASK, X_OBS)
        x0 = x @ torch.from_numpy(A).T + torch.from_numpy(c)
        t = torch.tensor([p])
        mean = O.extract(tab.posterior_mean_coef1, t, (1, 1)).double() * x0 + \
            O.extract(tab.posterior_mean_coef2, t, (1, 1)).double() * x
        sd = torch.exp(0.5 * O.extract(tab.posterior_log_variance_clipped, t, (1, 1)).double())
        return {"sample": mean + float(p != 0) * sd * z, "pred_xstart": x0}

    walk = R.build_walk(49, j, r)
    x = torch.randn(n, N_DIM, generator=g, dtype=torch.float64)
    x = R.run_walk(walk, x, lambda d: torch.randn(n, N_DIM, generator=g, dtype=torch.float64),
                   a.double(), b.double(), denoise)
    m, S = R.gaussian_law(tab, MU, COV, MASK, X_OBS, j, r)
    xs = x.numpy()
    print(f"\nMC mean {xs.mean(0)}\nexact   {m}")
    assert np.array_equal(xs[:, MASK], np.broadcast_to(X_OBS[MASK], (n, 2)))
    assert np.abs(xs.mean(0) - m).max() < 3e-3  # standard error ~ 0.5 / sqrt(4e5) = 8e-4
    assert np.abs(np.cov(xs.T) - S).max() < 3e-3


def test_resampling_brings_the_generated_coordinates_to_the_conditional_law():
    """KL(law of the generated coordinates || true conditional) as jump_n_sample grows: imputation alone (r = 1) is far
    from the conditional; resampling shrinks the distance on both grids, with diminishing returns on ddim50."""
    print("\ngrid      j   r   KL          max|mean err|  max|cov err|")
    got = {}
    for resp, j in (("ddim50", 5), ("", 10)):
        tab = O.make_tables(resp)
        for r in (1, 2, 5, 10):
            got[resp, r] = _distances(tab, j, r)
            print(f"{resp or 'T=1000':8s} {j:3d} {r:3d}   {got[resp, r][0]:.4e}  {got[resp, r][1]:.4e}    {got[resp, r][2]:.4e}")
    pinned = {("ddim50", 1): 4.7928e-01, ("ddim50", 2): 1.6299e-01, ("ddim50", 5): 7.8911e-02, ("ddim50", 10): 7.4061e-02,
              ("", 1): 4.5808e-01, ("", 2): 1.1982e-01, ("", 5): 1.6505e-02, ("", 10): 4.4986e-03}
    for k, kl in pinned.items():
        assert got[k][0] == pytest.approx(kl, rel=1e-3), k
    for resp in ("ddim50", ""):
        kls = [got[resp, r][0] for r in (1, 2, 5, 10)]
        assert all(x > y for x, y in zip(kls, kls[1:])), resp  # every r shrinks it further
    assert got["", 10][0] < got["", 1][0] / 100


# ------------------------------------------------------------------------------------------------
# the public loops' argument checks
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("bad", [0, -1, 1.0, 2.5, True, "2", None])
def test_argument_errors(bad):
    """raised at the call, before any model or device is touched"""
    d = C.create_gaussian_diffusion(timestep_respacing="ddim50")
    for fn in (d.repaint_sample_loop, d.repaint_sample_loop_progressive):
        for kw in ({"jump_length": bad}, {"jump_n_sample": bad}):
            with pytest.raises(ValueError):
                fn(None, SHAPE, model_kwargs={"y": {}}, **kw)
    with pytest.raises(ValueError):
        R.check_args(bad, 1)
    with pytest.raises(ValueError):
        R.check_args(1, bad)


def test_unsupported_arguments():
    d = C.create_gaussian_diffusion(timestep_respacing="ddim50")
    for fn in (d.repaint_sample_loop, d.repaint_sample_loop_progressive):
        with pytest.raises(NotImplementedError):
            fn(None, SHAPE, model_kwargs={"y": {}}, cond_fn=lambda x, t, **kw: x)
        with pytest.raises(NotImplementedError):
            fn(None, SHAPE, model_kwargs={"y": {}}, denoised_fn=lambda x: x)
        with pytest.raises(NotImplementedError):
            fn(None, SHAPE, model_kwargs={"y": {}}, const_noise=True)
        for kw in ({"eta": 0.0}, {"dump_steps": [1]}):
            with pytest.raises(TypeError):
                fn(None, SHAPE, model_kwargs={"y": {}}, **kw)


@pytest.mark.parametrize("name", ["repaint_sample_loop", "repaint_sample_loop_progressive"])
def test_install_adds_the_repaint_loops(name):
    base = C.create_gaussian_diffusion(timestep_respacing="ddim50")
    stock = StockDiffusion(base.betas, base.timestep_map)
    assert not hasattr(stock, name)
    ref = C.install(stock)
    with pytest.raises(ValueError):
        getattr(ref, name)(None, SHAPE, model_kwargs={"y": {}}, jump_length=0)
    with pytest.raises(NotImplementedError):  # nothing to fall back to: the reference has no such loop
        ref2 = C.install(StockDiffusion(base.betas, base.timestep_map), fallback_to_reference=True)
        getattr(ref2, name)(None, SHAPE, model_kwargs={"y": {}}, cond_fn=lambda x, t, **kw: x)
    assert hasattr(C.accelerate(StockDiffusion(base.betas, base.timestep_map)), name)

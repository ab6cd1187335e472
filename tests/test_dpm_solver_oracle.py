"""CPU: the DPM-Solver++ restatement in oracle/dpm_solver_oracle.py.

- Order 1 against tests/golden/dpm_solver.* -- the UNMODIFIED reference's ddim_sample_loop at eta = 0
  (oracle/make_golden_dpm_solver.py) -- and orders 2 / 3 against the values stored there.
- The folded coefficient table against the unfolded formulas, the effective-order rule and the final step.
- Convergence of the ODE discretisation on a small transformer.
- The argument errors of the public loops, and install().
"""
import numpy as np
import pytest
import torch

import condmdi_b200 as C
from oracle import condmdi_oracle as O
from oracle import dpm_solver_oracle as S
from oracle.golden_io import load_golden
from standin import StockDiffusion

B, D, L = 2, 263, 196
SHAPE = (B, D, 1, L)
# The folded fp32 update rounds differently from the reference's eps form: measured 5.5e-6 (no_cond, whole loop),
# 2.4e-5 (CFG + imputation), 5.6e-5 (guidance w = 20, the largest x0), 3.8e-5 (UNet xl) -- within the parity gate's
# atol of 1e-4.
ANCHOR_TOL = 1e-4
# the stored order-2 / order-3 values come from this same restatement: only thread-count dependent summation order differs
REGRESSION_TOL = 1e-5


@pytest.fixture(scope="module")
def gold(golden_dir):
    return load_golden(golden_dir, "dpm_solver")


@pytest.fixture(scope="module")
def gi(gold):
    gi = O.golden_inputs()
    chk = np.array([float(gi["x"].double().sum()), float(gi["tape"].double().sum()), float(gi["cond"].double().sum())])
    assert np.allclose(chk, gold["inputs.checksum"], rtol=0, atol=1e-9), "seeded inputs differ from the fixtures' inputs"
    return gi


def maxerr(a, b):
    return (torch.as_tensor(a).double() - torch.as_tensor(b).double()).abs().max().item()


def case_args(name, gi):
    """(state dict, conditioning, skip_timesteps, init_image) of each fixture configuration"""
    kw = dict(cond_emb=gi["cond"], cfg=True, text_scale=gi["text_scale"], y_mask=gi["y_mask"], imputate=True,
              stop_imputation_at=1, inpainted_motion=gi["x_obs"], inpainting_mask=gi["kf_mask"])
    if name == "no_cond":
        return O.random_state_dict(seed=7, text=False), O.Conditioning(), 0, None
    if name == "cfg_impute":
        return O.random_state_dict(seed=7, text=True), O.Conditioning(**kw), 45, gi["x_obs"]
    if name == "guided":
        c = O.Conditioning(reconstruction_guidance=True, reconstruction_weight=20.0, stop_recguidance_at=2, **kw)
        return O.random_state_dict(seed=7, text=True), c, 46, gi["x_obs"]
    c = O.Conditioning(cond_emb=gi["cond"], cfg=True, text_scale=gi["text_scale"], obs_x0=gi["x_obs"], obs_mask=gi["kf_mask"])
    return O.random_unet_state_dict(seed=11, text=True), c, 45, gi["x_obs"]


@pytest.mark.parametrize("name", ["no_cond", "cfg_impute", "guided", "unet"])
def test_orders_vs_reference_ddim_golden(gold, gi, name):
    sd, c, skip, init = case_args(name, gi)
    tab = O.make_tables("ddim50")
    o1 = S.dpm_solver_sample_loop(sd, tab, SHAPE, c, gi["tape"], 1, skip_timesteps=skip, init_image=init)
    err = maxerr(o1, gold[f"{name}.ddim_ref"])
    print(f"[{name}] |order 1 - reference ddim_sample_loop| = {err:.3e}")
    assert err <= ANCHOR_TOL
    for order in (2, 3):
        got = S.dpm_solver_sample_loop(sd, tab, SHAPE, c, gi["tape"], order, skip_timesteps=skip, init_image=init)
        assert maxerr(got, gold[f"{name}.o{order}"]) <= REGRESSION_TOL, order
        assert maxerr(got, o1) > 1e-3  # the higher orders do change the result


@pytest.mark.parametrize("order", [1, 2, 3])
@pytest.mark.parametrize("t_start", [19, 15, 2])
def test_folded_table_equals_unfolded_formulas(order, t_start):
    tab = O.make_tables("ddim20")
    table = S.coefficient_table(tab, t_start, order)
    assert table.dtype == np.float64 and table.shape == (20, 4)
    assert not table[t_start + 1:].any()
    rng = np.random.default_rng(3)
    for s in range(t_start, -1, -1):
        eff = S.effective_order(order, t_start - s, s)
        x, m0, m1, m2 = rng.standard_normal((4, 64))
        A, B0, B1, B2 = table[s]
        folded = A * x + B0 * m0 + B1 * m1 + B2 * m2
        want = S.unfolded_update(tab, s, eff, x, m0, m1, m2)
        np.testing.assert_allclose(folded, want, rtol=1e-11, atol=1e-12, err_msg=f"s={s} eff={eff}")


def test_effective_order_and_final_step():
    tab = O.make_tables("ddim20")
    assert [S.effective_order(3, k, 19 - k) for k in range(20)] == [1, 2] + [3] * 16 + [2, 1]
    assert [S.effective_order(2, k, 9 - k) for k in range(10)] == [1] + [2] * 8 + [1]
    assert [S.effective_order(3, k, 1 - k) for k in range(2)] == [1, 1]
    for order in (1, 2, 3):
        table = S.coefficient_table(tab, 19, order)
        assert tuple(table[0]) == (0.0, 1.0, 0.0, 0.0)  # the last step lands on abar = 1: x = m0, as DDIM's does
        for s in range(1, 20):
            eff = S.effective_order(order, 19 - s, s)
            assert (table[s, 2] != 0) == (eff >= 2) and (table[s, 3] != 0) == (eff >= 3), (order, s)
    # order 1 is DDIM at eta = 0: x_u = sqrt(abar_u) x0 + sqrt(1 - abar_u) (x - sqrt(abar_s) x0) / sqrt(1 - abar_s)
    t1 = S.coefficient_table(tab, 19, 1)
    ab, abp = tab.alphas_cumprod[1:], tab.alphas_cumprod_prev[1:]
    np.testing.assert_allclose(t1[1:, 0], np.sqrt(1 - abp) / np.sqrt(1 - ab), rtol=1e-13)
    np.testing.assert_allclose(t1[1:, 1], np.sqrt(abp) - np.sqrt(1 - abp) * np.sqrt(ab) / np.sqrt(1 - ab), rtol=1e-10)


def test_convergence_small_transformer():
    """The ODE the three orders discretise, solved at order 1 with the full 1000 steps, against 10 / 20 / 50 steps.  The
    grids are the section respacings "10" / "20" / "50", which keep t = 999 like the 1000-step solution, so every run
    starts from the same x_T at the same noise level.  The weights are random: this measures discretisation error only."""
    Bc, Lc = 1, 60
    sd = O.random_state_dict(seed=3, layers=2)
    g = torch.Generator().manual_seed(8)
    tape = torch.randn(1, Bc, D, 1, Lc, generator=g)
    shape = (Bc, D, 1, Lc)
    ref = S.dpm_solver_sample_loop(sd, O.make_tables(""), shape, O.Conditioning(), tape, 1)
    errs = {}
    for n in (10, 20, 50):
        tab = O.make_tables(str(n))
        assert tab.timestep_map[-1] == 999 and tab.num_timesteps == n
        for order in (1, 2, 3):
            got = S.dpm_solver_sample_loop(sd, tab, shape, O.Conditioning(), tape, order)
            e = (got.double() - ref.double()).abs()
            errs[n, order] = (e.max().item(), e.mean().item())
    print("\nsteps  order  max|x - x_1000|  mean|x - x_1000|")
    for (n, order), (mx, mn) in errs.items():
        print(f"{n:5d}  {order:5d}  {mx:15.3e}  {mn:16.3e}")
    for n in (10, 20, 50):
        for order in (2, 3):
            assert errs[n, order][1] < errs[n, 1][1], (n, order, errs)
            assert errs[n, order][0] < errs[n, 1][0], (n, order, errs)


@pytest.mark.parametrize("order", [0, 4, -1, 1.0, 2.5, True, "2", None])
def test_order_errors(order):
    """raised at the call, before any model or device is touched"""
    d = C.create_gaussian_diffusion(timestep_respacing="ddim50")
    for fn in (d.dpm_solver_sample_loop, d.dpm_solver_sample_loop_progressive):
        with pytest.raises(ValueError):
            fn(None, SHAPE, model_kwargs={"y": {}}, order=order)
    with pytest.raises(ValueError):
        S.check_order(order)


def test_unsupported_arguments():
    d = C.create_gaussian_diffusion(timestep_respacing="ddim50")
    for fn in (d.dpm_solver_sample_loop, d.dpm_solver_sample_loop_progressive):
        with pytest.raises(NotImplementedError):
            fn(None, SHAPE, model_kwargs={"y": {}}, cond_fn=lambda x, t, **kw: x)
        with pytest.raises(NotImplementedError):
            fn(None, SHAPE, model_kwargs={"y": {}}, denoised_fn=lambda x: x)
        with pytest.raises(NotImplementedError):
            fn(None, SHAPE, model_kwargs={"y": {"gmd": True}})
        for kw in ({"eta": 0.0}, {"dump_steps": [1]}):
            with pytest.raises(TypeError):
                fn(None, SHAPE, model_kwargs={"y": {}}, **kw)


@pytest.mark.parametrize("name", ["dpm_solver_sample_loop", "dpm_solver_sample_loop_progressive"])
def test_install_adds_the_dpm_solver_loops(name):
    base = C.create_gaussian_diffusion(timestep_respacing="ddim50")
    stock = StockDiffusion(base.betas, base.timestep_map)
    assert not hasattr(stock, name)
    ref = C.install(stock)
    with pytest.raises(ValueError):
        getattr(ref, name)(None, SHAPE, model_kwargs={"y": {}}, order=4)
    with pytest.raises(NotImplementedError):  # nothing to fall back to: the reference has no such loop
        C.install(StockDiffusion(base.betas, base.timestep_map), fallback_to_reference=True)
        getattr(ref, name)(None, SHAPE, model_kwargs={"y": {}}, cond_fn=lambda x, t, **kw: x)

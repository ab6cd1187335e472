"""CPU: the SDE-DPM-Solver++ restatement in oracle/dpm_solver_sde_oracle.py.

- Order 1 against tests/golden/dpm_solver_sde.* -- the UNMODIFIED reference's p_sample_loop on the same noise tape
  (oracle/make_golden_dpm_solver_sde.py) -- and order 2 against the values stored there.
- The folded coefficient table against the unfolded formulas, order 1 against the DDPM posterior tables, the final step.
- The exact law of the samples on Gaussian data: order 1 converges at rate 1 in the step size, order 2 at rate 2.
- The argument errors of the public loops, and install().
"""
import numpy as np
import pytest
import torch

import condmdi_b200 as C
from oracle import condmdi_oracle as O
from oracle import dpm_solver_sde_oracle as S
from oracle.golden_io import load_golden
from standin import StockDiffusion

B, D, L = 2, 263, 196
SHAPE = (B, D, 1, L)
# The folded fp32 coefficients round differently from the reference's posterior tables and exp(0.5 log variance);
# measured when the fixtures were written (oracle/make_golden_dpm_solver_sde.py states the per-case gaps)
ANCHOR_TOL = 2e-5
# the stored order-2 values come from this same restatement: only thread-count dependent summation order differs
REGRESSION_TOL = 1e-5


@pytest.fixture(scope="module")
def gold(golden_dir):
    return load_golden(golden_dir, "dpm_solver_sde")


@pytest.fixture(scope="module")
def gi(gold):
    gi = O.golden_inputs()
    chk = np.array([float(gi["x"].double().sum()), float(gi["tape"].double().sum()), float(gi["cond"].double().sum())])
    assert np.allclose(chk, gold["inputs.checksum"], rtol=0, atol=1e-9), "seeded inputs differ from the fixtures' inputs"
    return gi


def tape51(gi):
    return gi["tape"][torch.arange(51) % 8]


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
def test_orders_vs_reference_ddpm_golden(gold, gi, name):
    sd, c, skip, init = case_args(name, gi)
    tab = O.make_tables("ddim50")
    tape = tape51(gi)
    o1 = S.dpm_solver_sde_sample_loop(sd, tab, SHAPE, c, tape, 1, skip_timesteps=skip, init_image=init)
    err = maxerr(o1, gold[f"{name}.ddpm_ref"])
    print(f"[{name}] |order 1 - reference p_sample_loop| = {err:.3e}")
    assert err <= ANCHOR_TOL
    o2 = S.dpm_solver_sde_sample_loop(sd, tab, SHAPE, c, tape, 2, skip_timesteps=skip, init_image=init)
    assert maxerr(o2, gold[f"{name}.o2"]) <= REGRESSION_TOL
    assert maxerr(o2, o1) > 1e-3  # order 2 does change the result


@pytest.mark.parametrize("order", [1, 2])
@pytest.mark.parametrize("respacing, t_start", [("ddim10", 9), ("ddim20", 19), ("ddim50", 49), ("ddim20", 12), ("ddim50", 3)])
def test_folded_table_equals_unfolded_formulas(order, respacing, t_start):
    """every step of a whole loop, and of histories started mid-loop (a skip_timesteps call)"""
    tab = O.make_tables(respacing)
    table = S.coefficient_table(tab, t_start, order)
    assert table.dtype == np.float64 and table.shape == (tab.num_timesteps, 4)
    assert not table[t_start + 1:].any()
    rng = np.random.default_rng(5)
    for s in range(t_start, -1, -1):
        eff = S.effective_order(order, t_start - s, s)
        x, m0, m1, z = rng.standard_normal((4, 64))
        A, B0, B1, Cn = table[s]
        folded = A * x + B0 * m0 + B1 * m1 + Cn * z
        want = S.unfolded_update(tab, s, eff, x, m0, m1, z)
        np.testing.assert_allclose(folded, want, rtol=1e-11, atol=1e-12, err_msg=f"s={s} eff={eff}")
        assert (B1 != 0) == (eff >= 2), (s, eff)


@pytest.mark.parametrize("respacing, rtol", [("ddim10", 1e-12), ("ddim20", 1e-12), ("ddim50", 1e-12), ("", 5e-12)])
def test_order1_is_the_ddpm_posterior_step(respacing, rtol):
    """A = posterior_mean_coef2, B0 = posterior_mean_coef1, Cn^2 = posterior_variance for s >= 1; the s = 0 row returns
    x0 with no noise, as p_sample's t = 0 step does.  (On the 1000-step grid h is ~1e-3, and forming it as a difference
    of two logarithms costs about one more digit: 1.2e-12 measured.)"""
    tab = O.make_tables(respacing)
    T = tab.num_timesteps
    for order in (1, 2):
        table = S.coefficient_table(tab, T - 1, order)
        assert tuple(table[0]) == (0.0, 1.0, 0.0, 0.0)
    t1 = S.coefficient_table(tab, T - 1, 1)
    np.testing.assert_allclose(t1[1:, 0], tab.posterior_mean_coef2[1:], rtol=rtol, atol=0)
    np.testing.assert_allclose(t1[1:, 1], tab.posterior_mean_coef1[1:], rtol=rtol, atol=0)
    np.testing.assert_allclose(t1[1:, 3] ** 2, tab.posterior_variance[1:], rtol=rtol, atol=0)
    assert not t1[:, 2].any()


def test_effective_order():
    assert [S.effective_order(2, k, 9 - k) for k in range(10)] == [1] + [2] * 8 + [1]
    assert [S.effective_order(2, k, 1 - k) for k in range(2)] == [1, 1]
    assert [S.effective_order(1, k, 9 - k) for k in range(10)] == [1] * 10


def test_exact_gaussian_law_converges_at_orders_one_and_two():
    """x0 ~ N(0.5, s^2) per element and the exact denoiser: the law of the samples is Gaussian and is propagated exactly
    (oracle gaussian_std_error).  The grids are space_timesteps(1000, [N]).  Fitted over 100-500 steps, |std(x0) - s|
    falls as N^-1 at order 1 and N^-2 at order 2; order 2 with 250 steps beats 1000 ancestral (order-1) steps."""
    ns = [100, 150, 200, 300, 400, 500]
    print("\ndata std  order  slope   err@100   err@500")
    for s in (0.3, 0.5, 1.0):
        for order, (lo, hi) in ((1, (0.85, 1.1)), (2, (1.9, 2.2))):
            errs = [S.gaussian_std_error(O.make_tables([n]), order, s) for n in ns]
            slope = -np.polyfit(np.log(ns), np.log(errs), 1)[0]
            print(f"{s:8.1f}  {order:5d}  {slope:5.3f}  {errs[0]:.3e}  {errs[-1]:.3e}")
            assert lo <= slope <= hi, (s, order, slope)
        ddpm_1000 = S.gaussian_std_error(O.make_tables(""), 1, s)
        o2_250 = S.gaussian_std_error(O.make_tables([250]), 2, s)
        print(f"  s = {s}: order 1 x 1000 {ddpm_1000:.3e}, order 2 x 250 {o2_250:.3e}")
        assert o2_250 < ddpm_1000


@pytest.mark.parametrize("order", [0, 3, -1, 1.0, 2.5, True, "2", None])
def test_order_errors(order):
    """raised at the call, before any model or device is touched"""
    d = C.create_gaussian_diffusion(timestep_respacing="ddim50")
    for fn in (d.dpm_solver_sde_sample_loop, d.dpm_solver_sde_sample_loop_progressive):
        with pytest.raises(ValueError):
            fn(None, SHAPE, model_kwargs={"y": {}}, order=order)
    with pytest.raises(ValueError):
        S.check_order(order)


def test_unsupported_arguments():
    d = C.create_gaussian_diffusion(timestep_respacing="ddim50")
    for fn in (d.dpm_solver_sde_sample_loop, d.dpm_solver_sde_sample_loop_progressive):
        with pytest.raises(NotImplementedError):
            fn(None, SHAPE, model_kwargs={"y": {}}, cond_fn=lambda x, t, **kw: x)
        with pytest.raises(NotImplementedError):
            fn(None, SHAPE, model_kwargs={"y": {}}, denoised_fn=lambda x: x)
        with pytest.raises(NotImplementedError):
            fn(None, SHAPE, model_kwargs={"y": {}}, const_noise=True)
        with pytest.raises(NotImplementedError):
            fn(None, SHAPE, model_kwargs={"y": {"gmd": True}})
        for kw in ({"eta": 0.0}, {"dump_steps": [1]}):
            with pytest.raises(TypeError):
                fn(None, SHAPE, model_kwargs={"y": {}}, **kw)


@pytest.mark.parametrize("name", ["dpm_solver_sde_sample_loop", "dpm_solver_sde_sample_loop_progressive"])
def test_install_adds_the_sde_loops(name):
    base = C.create_gaussian_diffusion(timestep_respacing="ddim50")
    stock = StockDiffusion(base.betas, base.timestep_map)
    assert not hasattr(stock, name)
    ref = C.install(stock)
    with pytest.raises(ValueError):
        getattr(ref, name)(None, SHAPE, model_kwargs={"y": {}}, order=3)
    with pytest.raises(NotImplementedError):  # nothing to fall back to: the reference has no such loop
        ref2 = C.install(StockDiffusion(base.betas, base.timestep_map), fallback_to_reference=True)
        getattr(ref2, name)(None, SHAPE, model_kwargs={"y": {}}, cond_fn=lambda x, t, **kw: x)

"""CPU: the UniPC restatement in oracle/unipc_oracle.py.

- Order 1 without the corrector against tests/golden/unipc.* -- the UNMODIFIED reference's ddim_sample_loop at eta = 0
  (oracle/make_golden_unipc.py) -- and the other orders, variants and corrector settings against the values stored there.
- The folded coefficient table against the unfolded formulas, the order rules and the final step.
- Convergence of the ODE discretisation on Gaussian data, whose exact denoiser and exact solution are known, and the
  local order of one step.
- The argument errors of the public loops, and install().
"""
import numpy as np
import pytest
import torch

import condmdi_b200 as C
from oracle import condmdi_oracle as O
from oracle import dpm_solver_oracle as S
from oracle import unipc_oracle as U
from oracle.golden_io import load_golden
from standin import StockDiffusion

B, D, L = 2, 263, 196
SHAPE = (B, D, 1, L)
# the folded fp32 update rounds differently from the reference's eps form; order 1 without the corrector folds to the
# same rows as DPM-Solver++'s order 1, whose measured distance is 5.5e-6 to 5.6e-5
ANCHOR_TOL = 1e-4
# the stored values come from this same restatement: only thread-count dependent summation order differs
REGRESSION_TOL = 1e-5
# the runs checked here against the stored values (the GPU tests check every stored run)
CPU_KEYS = ["p2_bh1", "c1_bh2", "c2_bh2", "c3_bh1"]


@pytest.fixture(scope="module")
def gold(golden_dir):
    return load_golden(golden_dir, "unipc")


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


def run_key(key):
    """(order, variant, corrector) of a stored run's key: p<order>[_<variant>] or c<order>_<variant>"""
    order = int(key[1])
    return order, key.split("_")[1] if "_" in key else "bh2", key[0] == "c"


@pytest.mark.parametrize("name", ["no_cond", "cfg_impute", "guided", "unet"])
def test_vs_reference_ddim_golden(gold, gi, name):
    sd, c, skip, init = case_args(name, gi)
    tab = O.make_tables("ddim50")
    p1 = U.unipc_sample_loop(sd, tab, SHAPE, c, gi["tape"], 1, "bh2", False, skip_timesteps=skip, init_image=init)
    err = maxerr(p1, gold[f"{name}.ddim_ref"])
    print(f"[{name}] |UniP order 1 - reference ddim_sample_loop| = {err:.3e}")
    assert err <= ANCHOR_TOL
    assert maxerr(p1, gold[f"{name}.p1"]) <= REGRESSION_TOL
    for key in CPU_KEYS:
        order, variant, corrector = run_key(key)
        got = U.unipc_sample_loop(sd, tab, SHAPE, c, gi["tape"], order, variant, corrector, skip_timesteps=skip,
                                  init_image=init)
        assert maxerr(got, gold[f"{name}.{key}"]) <= REGRESSION_TOL, key
        assert maxerr(got, p1) > 1e-3, key  # the higher orders and the corrector do change the result


@pytest.mark.parametrize("respacing", ["ddim10", "ddim20", "ddim50"])
@pytest.mark.parametrize("variant", ["bh1", "bh2"])
@pytest.mark.parametrize("corrector", [False, True])
@pytest.mark.parametrize("order", [1, 2, 3])
def test_folded_table_equals_unfolded_formulas(respacing, variant, corrector, order):
    tab = O.make_tables(respacing)
    T = tab.num_timesteps
    rng = np.random.default_rng(3)
    for t_start in (T - 1, T // 2, 2, 1):
        table = U.coefficient_table(tab, t_start, order, variant, corrector)
        assert table.dtype == np.float64 and table.shape == (T, 12)
        assert not table[t_start + 1:].any() and not table[:, 9:].any()
        for s in range(t_start, -1, -1):
            k = t_start - s
            pe, ce = U.predictor_order(order, k, s), U.corrector_order(order, k, s, corrector)
            x, m0, m1, m2, m3 = rng.standard_normal((5, 64))
            A, B0, B1, B2, Ac, C0, C1, C2, C3 = table[s, :9]
            if s == 0:
                assert tuple(table[0, :4]) == (0.0, 1.0, 0.0, 0.0)
            else:
                folded = A * x + B0 * m0 + B1 * m1 + B2 * m2
                want = U.unfolded_update(tab, s - 1, list(range(s, s + pe)), x, [m0, m1, m2][:pe], variant)
                np.testing.assert_allclose(folded, want, rtol=1e-11, atol=1e-12, err_msg=f"UniP s={s} p={pe}")
                assert all((table[s, j] != 0) == (j <= pe) for j in (2, 3)), (s, pe)
            if ce == 0:
                assert not table[s, 4:9].any()
                continue
            folded = Ac * x + C0 * m0 + C1 * m1 + C2 * m2 + C3 * m3
            want = U.unfolded_update(tab, s, list(range(s + 1, s + 1 + ce)), x, [m1, m2, m3][:ce], variant, m_t=m0)
            np.testing.assert_allclose(folded, want, rtol=1e-11, atol=1e-12, err_msg=f"UniC s={s} p={ce}")
            assert all((table[s, 5 + j] != 0) == (j <= ce) for j in (2, 3)), (s, ce)


def test_order_rules_and_final_step():
    # predictor: DPM-Solver++'s rule; correction at s: the order of the predictor into s, none at k = 0 and s = 0
    assert [U.predictor_order(3, k, 19 - k) for k in range(20)] == [1, 2] + [3] * 16 + [2, 1]
    assert [U.corrector_order(3, k, 19 - k) for k in range(20)] == [0, 1, 2] + [3] * 16 + [0]
    assert [U.corrector_order(2, k, 9 - k) for k in range(10)] == [0, 1] + [2] * 7 + [0]
    assert [U.corrector_order(3, k, 19 - k, corrector=False) for k in range(20)] == [0] * 20
    assert [U.predictor_order(o, k, 19 - k) for o in (1, 2, 3) for k in range(20)] == \
        [S.effective_order(o, k, 19 - k) for o in (1, 2, 3) for k in range(20)]
    tab = O.make_tables("ddim20")
    for variant in U.VARIANTS:
        # order 1 without the corrector is DDIM at eta = 0: the same float64 rows as DPM-Solver++'s order 1
        t = U.coefficient_table(tab, 19, 1, variant, False)
        assert np.array_equal(t[:, :4], S.coefficient_table(tab, 19, 1)) and not t[:, 4:].any()
        # UniC-1 corrects with rhos_c = [0.5]: C0 = -C1 + (DDIM's B0 into s), Ac = DDIM's A into s
        t = U.coefficient_table(tab, 19, 1, variant, True)
        d = S.coefficient_table(tab, 19, 1)
        np.testing.assert_allclose(t[1:19, 4], d[2:20, 0], rtol=1e-14)
        np.testing.assert_allclose(t[1:19, 5] + t[1:19, 6], d[2:20, 1], rtol=1e-12)


def _lambda_grid(n, lam_min=-3.0, lam_max=3.0):
    """n steps uniform in lambda: abar_s = sigmoid(2 lambda_s), s = 0 the least noisy.  (Respaced step grids round
    their strides, so their step sizes are not a smooth refinement and the observed order would wander.)"""
    lam = np.linspace(lam_max, lam_min, n)
    acp = 1.0 / (1.0 + np.exp(-2.0 * lam))
    return O.DiffusionTables(1.0 - acp / np.append(1.0, acp[:-1]), list(range(n)))


CONV_STEPS = (20, 40, 80, 160, 320)
# lower bounds on the fitted slope of log max-error against log steps, 0.15-0.2 below the lower of the two variants'
# values measured on this problem (DESIGN.md section 8): UniP 1.00 / 2.02-2.08 / 2.24-2.29, UniC 2.03-2.10 / 3.03-3.09 / 3.30.  Order 3 observes one
# order less than the steady steps reach: the first step of a history is order 1 (corrected: order 2), and with the
# corrector its error, O(h^3), is what remains at these step counts.
MIN_SLOPE = {(False, 1): 0.85, (False, 2): 1.85, (False, 3): 2.05, (True, 1): 1.85, (True, 2): 2.85, (True, 3): 3.1}


def test_analytic_convergence_gaussian_data():
    """x0 ~ N(mu, s^2) per element.  The exact denoiser is x0(x) = mu + sqrt(abar) s^2 / (abar s^2 + 1 - abar)
    (x - sqrt(abar) mu), and the probability-flow ODE keeps z = (x - sqrt(abar) mu) / sqrt(abar s^2 + 1 - abar)
    constant, so the final x0 of the exact solution is mu + sqrt(abar_0) s^2 z / sqrt(abar_0 s^2 + 1 - abar_0).  Float64
    throughout (the table is not rounded), so the error is the discretisation's alone."""
    rng = np.random.default_rng(0)
    mu, sd, noise = rng.normal(size=256), rng.uniform(0.3, 1.5, 256), rng.normal(size=256)
    errs, slopes = {}, {}
    for variant in U.VARIANTS:
        for corrector in (False, True):
            for order in (1, 2, 3):
                e = []
                for n in CONV_STEPS:
                    tab = _lambda_grid(n)
                    acp = tab.alphas_cumprod

                    def denoise(x, s):
                        a = acp[s]
                        return mu + np.sqrt(a) * sd ** 2 / (a * sd ** 2 + 1 - a) * (x - np.sqrt(a) * mu)
                    a_T, a_0 = acp[n - 1], acp[0]
                    x_T = np.sqrt(a_T) * mu + np.sqrt(1 - a_T) * noise
                    z = (x_T - np.sqrt(a_T) * mu) / np.sqrt(a_T * sd ** 2 + 1 - a_T)
                    exact = mu + np.sqrt(a_0) * sd ** 2 * z / np.sqrt(a_0 * sd ** 2 + 1 - a_0)
                    got = U.unipc_loop(denoise, tab, x_T, n - 1, order, variant, corrector)
                    e.append(np.abs(got - exact).max())
                errs[variant, corrector, order] = e
                slopes[variant, corrector, order] = -np.polyfit(np.log(CONV_STEPS), np.log(e), 1)[0]
    print("\nvariant  UniC  order  slope  " + "  ".join(f"err@{n:<4d}" for n in CONV_STEPS))
    for (variant, corrector, order), e in errs.items():
        print(f"{variant:7s}  {corrector!s:5s} {order:5d}  {slopes[variant, corrector, order]:5.2f}  "
              + "  ".join(f"{v:8.2e}" for v in e))
    for variant in U.VARIANTS:
        for corrector in (False, True):
            sl = [slopes[variant, corrector, o] for o in (1, 2, 3)]
            assert sl[0] < sl[1] < sl[2], (variant, corrector, sl)  # the slope rises with order
            for order in (1, 2, 3):
                assert slopes[variant, corrector, order] >= MIN_SLOPE[corrector, order], (variant, corrector, order, sl)
        for order in (1, 2, 3):
            # UniC-p beats UniP-p at every step count, and observes a higher order
            assert all(c < p for c, p in zip(errs[variant, True, order], errs[variant, False, order])), (variant, order)
            assert slopes[variant, True, order] > slopes[variant, False, order] + 0.8, (variant, order)


def test_local_orders_one_step():
    """One update from the exact trajectory of the Gaussian problem above, with exact x0 history, over steps of h in
    lambda: UniP-p's error falls as h^(p+1), UniC-p's (m_t evaluated at the predicted state) as h^(p+2).  Measured slopes
    (bh1 / bh2): UniP 2.01 / 2.96-2.88 / 4.20, UniC 2.95-2.98 / 3.89-3.87 / 5.08; the bounds sit 0.2 below p + 1 and
    p + 2."""
    rng = np.random.default_rng(1)
    mu, sd, z = rng.normal(size=64), rng.uniform(0.5, 1.5, 64), rng.normal(size=64)

    def exact(a):
        return np.sqrt(a) * mu + z * np.sqrt(a * sd ** 2 + 1 - a)

    def denoise(x, a):
        return mu + np.sqrt(a) * sd ** 2 / (a * sd ** 2 + 1 - a) * (x - np.sqrt(a) * mu)
    hs = [0.16, 0.08, 0.04, 0.02, 0.01]
    for variant in U.VARIANTS:
        for p in (1, 2, 3):
            ep, ec = [], []
            for h in hs:
                lam = 0.2 - h * np.arange(5)
                acp = 1.0 / (1.0 + np.exp(-2.0 * lam))
                tab = O.DiffusionTables(1.0 - acp / np.append(1.0, acp[:-1]), list(range(5)))
                acp = tab.alphas_cumprod
                prev = list(range(1, 1 + p))
                m_prev = [denoise(exact(acp[i]), acp[i]) for i in prev]
                xp = U.unfolded_update(tab, 0, prev, exact(acp[1]), m_prev, variant)
                xc = U.unfolded_update(tab, 0, prev, exact(acp[1]), m_prev, variant, m_t=denoise(xp, acp[0]))
                ep.append(np.abs(xp - exact(acp[0])).max())
                ec.append(np.abs(xc - exact(acp[0])).max())
            sp, sc = (np.polyfit(np.log(hs), np.log(e), 1)[0] for e in (ep, ec))
            print(f"{variant} order {p}: UniP local slope {sp:.2f}, UniC local slope {sc:.2f}")
            assert sp >= p + 0.8 and sc >= p + 1.8, (variant, p, sp, sc)


@pytest.mark.parametrize("kw", [dict(order=0), dict(order=4), dict(order=1.0), dict(order=True), dict(order="2"),
                                dict(order=None), dict(variant="bh3"), dict(variant=None), dict(variant=2),
                                dict(corrector=1), dict(corrector="yes")])
def test_argument_errors(kw):
    """raised at the call, before any model or device is touched"""
    d = C.create_gaussian_diffusion(timestep_respacing="ddim50")
    for fn in (d.unipc_sample_loop, d.unipc_sample_loop_progressive):
        with pytest.raises(ValueError):
            fn(None, SHAPE, model_kwargs={"y": {}}, **kw)
    args = dict(order=2, variant="bh2", corrector=True)
    args.update(kw)
    with pytest.raises(ValueError):
        U.check_args(**args)


def test_unsupported_arguments():
    d = C.create_gaussian_diffusion(timestep_respacing="ddim50")
    for fn in (d.unipc_sample_loop, d.unipc_sample_loop_progressive):
        with pytest.raises(NotImplementedError):
            fn(None, SHAPE, model_kwargs={"y": {}}, cond_fn=lambda x, t, **kw: x)
        with pytest.raises(NotImplementedError):
            fn(None, SHAPE, model_kwargs={"y": {}}, denoised_fn=lambda x: x)
        with pytest.raises(NotImplementedError):
            fn(None, SHAPE, model_kwargs={"y": {"gmd": True}})
        for kw in ({"eta": 0.0}, {"dump_steps": [1]}):
            with pytest.raises(TypeError):
                fn(None, SHAPE, model_kwargs={"y": {}}, **kw)


@pytest.mark.parametrize("name", ["unipc_sample_loop", "unipc_sample_loop_progressive"])
def test_install_adds_the_unipc_loops(name):
    base = C.create_gaussian_diffusion(timestep_respacing="ddim50")
    stock = StockDiffusion(base.betas, base.timestep_map)
    assert not hasattr(stock, name)
    ref = C.install(stock)
    with pytest.raises(ValueError):
        getattr(ref, name)(None, SHAPE, model_kwargs={"y": {}}, order=4)
    with pytest.raises(ValueError):
        getattr(ref, name)(None, SHAPE, model_kwargs={"y": {}}, variant="bh3")
    with pytest.raises(NotImplementedError):  # nothing to fall back to: the reference has no such loop
        C.install(StockDiffusion(base.betas, base.timestep_map), fallback_to_reference=True)
        getattr(ref, name)(None, SHAPE, model_kwargs={"y": {}}, cond_fn=lambda x, t, **kw: x)

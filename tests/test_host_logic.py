"""CPU: host-side logic of the product (no kernel is launched here) and the C-ABI surface."""
import ctypes
import os
import re

import numpy as np
import pytest
import torch

import condmdi_b200 as C
from oracle import condmdi_oracle as O
from oracle.golden_io import load_golden

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
D, L = 263, 196


def test_library_loads_and_exports_every_declared_symbol():
    lib = C.capi.load()
    header = open(os.path.join(ROOT, "include", "condmdi_b200.h")).read()
    declared = re.findall(r"CMDI_API\s+[\w\s\*]+?\b(cmdi_\w+)\s*\(", header)
    assert len(declared) >= 13
    for name in declared:
        assert hasattr(lib, name), f"{name} is declared in include/condmdi_b200.h but not exported"
    assert set(declared) == set(C.capi.EXPORTS)
    assert b"sm_90a" in lib.cmdi_version()


def test_struct_layouts_match_header_field_counts():
    header = open(os.path.join(ROOT, "include", "condmdi_b200.h")).read()
    for cname, cls in (("cmdi_model_cfg", C.capi.ModelCfg), ("cmdi_tensor_desc", C.capi.TensorDesc),
                       ("cmdi_forward_args", C.capi.ForwardArgs), ("cmdi_sample_args", C.capi.SampleArgs)):
        body = re.search(r"typedef struct \{([^}]*)\} " + cname + ";", header).group(1)
        body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
        fields = [re.sub(r"\[\d+\]$", "", f.strip().split()[-1].lstrip("*")) for f in body.split(";") if f.strip()]
        assert fields == [f[0] for f in cls._fields_], cname


def test_no_cpu_fallback():
    with pytest.raises(RuntimeError):
        C.Engine(torch.device("cpu"))
    if not torch.cuda.is_available():
        m = C.MDM()
        with pytest.raises(RuntimeError):
            m(torch.zeros(1, D, 1, L), torch.zeros(1, dtype=torch.long), y={})
        d = C.create_gaussian_diffusion()
        with pytest.raises(Exception):
            d.p_sample_loop(m, (1, D, 1, L), model_kwargs={"y": {}}, device="cpu")


def test_product_never_imports_the_oracle():
    pkg = os.path.join(ROOT, "diffusion-motion-inbetweening_b200")
    for fn in os.listdir(pkg):
        if fn.endswith(".py"):
            src = open(os.path.join(pkg, fn)).read()
            assert "oracle" not in src.replace("no CPU fallback", ""), fn


@pytest.mark.parametrize("resp", ["", "ddim50", "ddim100", "10,15,20"])
def test_diffusion_tables_equal_reference(golden_dir, resp):
    g = load_golden(golden_dir, "schedules")
    name = {"": "full", "10,15,20": "sect"}.get(resp, resp)
    d = C.create_gaussian_diffusion(timestep_respacing=resp)
    assert d.timestep_map == g[f"{name}.timestep_map"].tolist()
    for f in ("betas", "alphas_cumprod", "alphas_cumprod_prev", "sqrt_recip_alphas_cumprod", "sqrt_recipm1_alphas_cumprod",
              "posterior_variance", "posterior_log_variance_clipped", "posterior_mean_coef1", "posterior_mean_coef2"):
        assert np.array_equal(getattr(d, f), g[f"{name}.{f}"]), f
    assert d.num_timesteps == len(d.timestep_map)
    for hook in ("data_transform_fn", "data_inv_transform_fn", "data_get_mean_fn", "log_trajectory_fn"):
        assert getattr(d, hook) is None


def test_space_timesteps_errors():
    assert C.space_timesteps(1000, "ddim100") == set(range(0, 1000, 10))
    with pytest.raises(ValueError):
        C.space_timesteps(1000, "ddim999")
    with pytest.raises(ValueError):
        C.space_timesteps(10, [20])


def test_keyframe_masks_bit_exact_vs_golden(golden_dir):
    g = load_golden(golden_dir, "masks")
    for key in sorted(k[:-5] for k in g if k.endswith(".bits")):
        mode, T, fm = key.split(".")
        lengths = torch.tensor(g[key + ".lengths"])
        m, jm = C.get_keyframes_mask(torch.zeros(len(lengths), D, 1, L), lengths, edit_mode=mode, trans_length=int(T),
                                     feature_mode=fm, get_joint_mask=True)
        assert m.dtype == torch.bool and m.shape == (len(lengths), D, 1, L) and jm.shape == (len(lengths), 22, 1, L)
        assert np.array_equal(np.packbits(m.numpy().reshape(-1)), g[key + ".bits"]), key


def test_keyframe_masks_ragged_and_edge_lengths():
    lengths = torch.tensor([0, 1, 2, 196, 33])
    for T in (1, 3, 7, 196, 500):
        a = C.get_keyframes_mask(torch.zeros(5, D, 1, L), lengths, "benchmark_sparse", trans_length=T)
        b = O.get_keyframes_mask(torch.zeros(5, D, 1, L), lengths, "benchmark_sparse", trans_length=T)
        assert torch.equal(a, b)
    for T in (1, 10, 30):
        lengths = torch.tensor([196, 100, 31, 30, 64])
        a = C.get_keyframes_mask(torch.zeros(5, D, 1, L), lengths, "benchmark_clip", trans_length=T)
        b = O.get_keyframes_mask(torch.zeros(5, D, 1, L), lengths, "benchmark_clip", trans_length=T)
        assert torch.equal(a, b)
    with pytest.raises(ValueError):
        C.get_keyframes_mask(torch.zeros(1, 100, 1, L), torch.tensor([5]))


def test_joint_to_full_mask_single_joints():
    for j in range(22):
        jm = torch.zeros(1, 22, 1, 4, dtype=torch.bool)
        jm[0, j, 0, 2] = True
        for mode in ("pos", "pos_rot", "pos_rot_vel"):
            assert torch.equal(C.joint_to_full_mask(jm, mode), O.joint_to_full_mask(jm, mode))


def test_state_dict_keys_match_reference_key_set():
    sd = O.random_state_dict(seed=0, text=True)  # key set validated against the reference in oracle/make_golden.py
    m = C.MDM(cond_mode="text", cond_mask_prob=0.1)
    assert set(m.state_dict().keys()) == set(sd.keys())
    for k, v in m.state_dict().items():
        assert tuple(v.shape) == tuple(sd[k].shape), k
    missing, unexpected = m.load_state_dict(sd, strict=False)
    assert not missing and not unexpected
    assert torch.equal(m.state_dict()["sequence_pos_encoder.pe"], O.positional_encoding(512))


def test_cfg_wrapper_contract():
    m = C.MDM(cond_mode="text", cond_mask_prob=0.0)
    with pytest.raises(AssertionError):
        C.ClassifierFreeSampleModel(m)  # cfg_sampler.py:11
    m = C.MDM(cond_mode="text", cond_mask_prob=0.1)
    w = C.ClassifierFreeSampleModel(m)
    assert w.njoints == 263 and w.nfeats == 1 and w.cond_mode == "text" and w.keyframe_conditioned is False
    inner, is_cfg = C.resolve_model(w)
    assert inner is m and is_cfg
    with pytest.raises(NotImplementedError):
        C.MDM(arch="trans_dec")


def test_sampler_error_behaviour_mirrors_reference():
    d = C.create_gaussian_diffusion()
    m = C.MDM()
    shape = (1, D, 1, L)
    with pytest.raises(NotImplementedError):
        d.p_sample_loop(m, shape, model_kwargs={"y": {}}, const_noise=True)          # gaussian_diffusion.py:698-699
    with pytest.raises(NotImplementedError):
        d.ddim_sample_loop(m, shape, model_kwargs={"y": {}}, const_noise=True)       # :1480-1481
    with pytest.raises(KeyError):
        d.p_sample_loop(m, shape, model_kwargs={})                                   # :1280 indexes model_kwargs['y']
    with pytest.raises(AssertionError):
        d.p_sample_loop(m, shape, model_kwargs={"y": {}}, cond_fn=lambda *a, **k: 0)  # :685
    with pytest.raises(NotImplementedError):
        d.p_sample_loop(m, shape, model_kwargs={"y": {"gmd": 1}})
    with pytest.raises(AssertionError):
        d.p_sample_loop(m, shape, model_kwargs={"y": {"reconstruction_guidance": True}})  # editing_util.py:329
    eps = C.SpacedDiffusion(C.space_timesteps(1000, [1000]), C.DiffusionConfig(
        betas=C.get_named_beta_schedule("cosine", 1000), model_mean_type=C.ModelMeanType.EPSILON))
    with pytest.raises(NotImplementedError):
        eps.p_sample_loop(m, shape, model_kwargs={"y": {}})


def test_q_sample_matches_oracle_formula():
    d = C.create_gaussian_diffusion()
    x0, nz = torch.randn(3, D, 1, L), torch.randn(3, D, 1, L)
    t = torch.tensor([0, 500, 999])
    tab = O.make_tables("")
    ref = O.extract(tab.sqrt_alphas_cumprod, t, x0.shape) * x0 + O.extract(tab.sqrt_one_minus_alphas_cumprod, t, x0.shape) * nz
    assert torch.equal(d.q_sample(x0, t, nz), ref)


def test_aten_launch_policy_arithmetic():
    """host side of CMDI_RNG_TORCH: ATen's grid / philox-offset bookkeeping for a B200 (148 SMs x 2048 threads)."""
    from condmdi_b200.diffusion import aten_policy
    assert aten_policy(64 * 263 * 196, 148, 2048) == (256 * 1184, 12)   # 3 curand_normal4 calls per thread
    assert aten_policy(4 * 263 * 196, 148, 2048) == (256 * 806, 4)      # fewer blocks than the SMs could hold
    assert aten_policy(1000, 148, 2048) == (1024, 4)
    assert aten_policy(256 * 1184 * 4, 148, 2048) == (256 * 1184, 4)
    assert aten_policy(256 * 1184 * 4 + 1, 148, 2048) == (256 * 1184, 8)


def test_post_processing_has_no_cpu_path():
    import condmdi_b200 as C
    with pytest.raises(RuntimeError):
        C.recover_from_ric(torch.zeros(1, 4, 263), 22)
    with pytest.raises(RuntimeError):
        C.sample_to_joints(torch.zeros(1, 263, 1, 4), torch.zeros(263), torch.ones(263))


def test_rational_erf_of_the_chained_epilogue_is_accurate():
    """gemm_chain.cu::erf_rational (the GELU of the chained FFN1 epilogue), evaluated here in float32 with the same
    coefficients and operation order: max |erf error| 3.7e-7, max |GELU error| 6.4e-7 over [-6, 6]."""
    import math

    import numpy as np
    f = np.float32
    a = [-2.72614225801306e-10, 2.77068142495902e-08, -2.10102402082508e-06, -5.69250639462346e-05, -7.34990630326855e-04,
         -2.95459980854025e-03, -1.60960333262415e-02]
    b = [-1.45660718464996e-05, -2.13374055278905e-04, -1.68282697438203e-03, -7.37332916720468e-03, -1.42647390514189e-02]
    src = open(os.path.join(ROOT, "diffusion-motion-inbetweening_b200", "csrc", "gemm_chain.cu")).read()
    for c in a + b:
        assert f"{c:.14e}".replace("e-0", "e-0") in src or repr(c) in src or f"{c}" in src, c
    x = np.linspace(-6, 6, 200001).astype(f)
    xc = np.clip(x, f(-4), f(4)).astype(f)
    x2 = (xc * xc).astype(f)

    def horner(cs):
        p = np.full_like(x2, f(cs[0]))
        for c in cs[1:]:
            p = (p * x2 + f(c)).astype(f)
        return p

    e = (xc * horner(a) / horner(b)).astype(f)
    ref = np.array([math.erf(float(v)) for v in x])
    assert np.abs(e.astype(np.float64) - ref).max() < 5e-7
    gelu = 0.5 * x.astype(np.float64) * (1 + e.astype(np.float64))
    assert np.abs(gelu - 0.5 * x.astype(np.float64) * (1 + ref)).max() < 1e-6

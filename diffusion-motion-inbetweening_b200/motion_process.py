"""HumanML3D feature vectors <-> joint positions, and the absolute <-> relative representation conversions, on the GPU.

Mirrors `data_loaders/humanml/scripts/motion_process.py:474-489` (`recover_from_ric`, with
`recover_root_rot_pos` :402-441) of the reference and the CPU hop around it in `sample/synthesize.py:153-157`
(`sample.cpu().permute(0, 2, 3, 1)` -> `inv_transform` -> `recover_from_ric` -> `view/permute`).  The work runs in
`cmdi_recover_from_ric` (csrc/elementwise.cu); there is no CPU path.

`joints_to_features`, `abs3d_to_rel` and `rel_to_abs3d` are `extract_features` (motion_process.py:50-187) and the two
conversions the evaluation loop runs per batch (data_loaders/humanml/data/dataset.py:1198-1401), for HumanML3D's
22-joint skeleton.  They run in `cmdi_joints_to_features` / `cmdi_convert_motion` (csrc/motion_features.cu), one launch
per call.  Dataset statistics keep their dtype: float64 statistics (de-)normalise in float64 as the reference's numpy /
torch promotion does, float32 ones in float32.
"""
from __future__ import annotations

import torch

from . import capi
from .engine import _ptr, _stream_ptr


def _check(data: torch.Tensor, what: str = "recover_from_ric"):
    if not data.is_cuda:
        raise RuntimeError(f"condmdi_b200.{what} runs on CUDA tensors only (no CPU fallback)")


def _stats(a, device) -> tuple[torch.Tensor, int]:
    """(float64 copy on `device`, 1 if the statistics are float64): the dtype decides the de-normalisation arithmetic."""
    t = torch.as_tensor(a)
    return t.to(device=device, dtype=torch.float64).contiguous(), int(t.dtype == torch.float64)


def _proj(inv_proj, device):
    if inv_proj is None:
        return None
    p = torch.as_tensor(inv_proj).to(device=device, dtype=torch.float32).contiguous()
    assert p.shape == (263, 263), p.shape
    return p


def joints_to_features(joints: torch.Tensor, feet_thre: float = 0.002) -> torch.Tensor:
    """`extract_features(positions, feet_thre, t2m_raw_offsets, t2m_kinematic_chain, [2, 1, 17, 16], [8, 11], [7, 10])`
    for a batch: `joints` (..., L, 22, 3) fp32 positions -> (..., L - 1, 263) de-normalised relative features."""
    _check(joints, "joints_to_features")
    lead, (L, J, three) = joints.shape[:-3], joints.shape[-3:]
    assert three == 3
    x = joints.to(torch.float32).reshape(-1, L, J, 3).contiguous()
    out = torch.empty(x.shape[0], max(L - 1, 0), 263, dtype=torch.float32, device=x.device)
    with torch.cuda.device(x.device):
        capi.check(capi.load().cmdi_joints_to_features(_ptr(x), L * J * 3, J * 3, x.shape[0], L, J, float(feet_thre), _ptr(out),
                                                       (L - 1) * 263, 263, 1, _stream_ptr(x.device)),
                   "cmdi_joints_to_features")
    return out.reshape(*lead, L - 1, 263)


def _convert(direction: int, sample: torch.Tensor, mean_in, std_in, mean_out, std_out, inv_proj, what: str) -> torch.Tensor:
    _check(sample, what)
    B, C, one, L = sample.shape
    assert one == 1
    dev = sample.device
    x = sample.to(torch.float32).contiguous()
    m_in, f64_in = _stats(mean_in, dev)
    s_in, _ = _stats(std_in, dev)
    m_out, f64_out = _stats(mean_out, dev)
    s_out, _ = _stats(std_out, dev)
    p = _proj(inv_proj, dev)
    out = torch.empty(B, C, 1, L, dtype=torch.float32, device=dev)
    with torch.cuda.device(dev):
        capi.check(capi.load().cmdi_convert_motion(direction, _ptr(x), C * L, L, 1, B, L, C, _ptr(p),
                                                   _ptr(m_in), _ptr(s_in), f64_in, _ptr(m_out), _ptr(s_out), f64_out, 0.002,
                                                   _ptr(out), C * L, L, 1, _stream_ptr(dev)),
                   "cmdi_convert_motion")
    return out


def abs3d_to_rel(sample_abs: torch.Tensor, mean_abs, std_abs, mean_rel, std_rel, inv_proj=None) -> torch.Tensor:
    """dataset.py:1327-1361 `abs3d_to_rel` with `motion_to_rel_data` (:1198-1250): a normalised absolute-representation
    batch (B, 263, 1, L) -> the relative representation (B, 263, 1, L) normalised with (mean_rel, std_rel).
    (mean_abs, std_abs) are the statistics of `t2m_dataset.inv_transform`; `inv_proj` its inverse random projection
    (the `proj*` cards' `inv_rand_proj.npy`) or None."""
    return _convert(capi.MOTION_ABS3D_TO_REL, sample_abs, mean_abs, std_abs, mean_rel, std_rel, inv_proj, "abs3d_to_rel")


def rel_to_abs3d(sample_rel: torch.Tensor, mean, std, mean_abs, std_abs, inv_proj=None) -> torch.Tensor:
    """dataset.py:1364-1401 `rel_to_abs3d` with `motion_to_abs_data` (:1253-1288): a normalised relative-representation
    batch (B, 263, 1, L), de-normalised with (mean, std) (and `inv_proj`), -> the absolute representation (B, 263, 1, L)
    normalised with (mean_abs, std_abs)."""
    return _convert(capi.MOTION_REL_TO_ABS3D, sample_rel, mean, std, mean_abs, std_abs, inv_proj, "rel_to_abs3d")


def recover_from_ric(data: torch.Tensor, joints_num: int, abs_3d: bool = False) -> torch.Tensor:
    """Same contract as the reference function: `data` (..., nframes, nfeats) de-normalised HumanML3D vectors ->
    (..., nframes, joints_num, 3) positions (root first)."""
    _check(data)
    lead, (L, C) = data.shape[:-2], data.shape[-2:]
    x = data.to(torch.float32).reshape(-1, L, C).contiguous()
    out = torch.empty(x.shape[0], L, joints_num, 3, dtype=torch.float32, device=x.device)
    with torch.cuda.device(x.device):
        capi.check(capi.load().cmdi_recover_from_ric(_ptr(x), L * C, C, 1, None, None, x.shape[0], L, C, joints_num, int(abs_3d),
                                                     _ptr(out), L * joints_num * 3, joints_num * 3, 3, 1, _stream_ptr(x.device)),
                   "cmdi_recover_from_ric")
    return out.reshape(*lead, L, joints_num, 3)


def sample_to_joints(sample: torch.Tensor, mean, std, joints_num: int = 22, abs_3d: bool = False, inv_proj=None) -> torch.Tensor:
    """What sample/synthesize.py:153-157 computes from the sampler output, without leaving the GPU:
    `sample` (B, nfeats, 1, nframes) normalised -> (B, joints_num, 3, nframes) positions, with
    `mean`/`std` (nfeats,) the dataset statistics of `t2m_dataset.inv_transform`.

    With `inv_proj` (263, 263), the `proj*` cards' inverse random projection, the sample is first multiplied by it
    (inv_transform with use_rand_proj, dataset.py:378-382, :536-539; sample_to_motion, :1301-1324); that path is
    HumanML3D only (22 joints, 2 <= nframes <= 224) and de-normalises in the statistics' dtype."""
    _check(sample)
    B, C, one, L = sample.shape
    assert one == 1
    if inv_proj is not None:
        if joints_num != 22:
            raise RuntimeError(f"sample_to_joints with inv_proj needs joints_num == 22 (HumanML3D), got {joints_num}")
        dev = sample.device
        x = sample.to(torch.float32).contiguous()
        m, f64 = _stats(mean, dev)
        s, _ = _stats(std, dev)
        p = _proj(inv_proj, dev)
        out = torch.empty(B, joints_num, 3, L, dtype=torch.float32, device=dev)
        direction = capi.MOTION_ABS3D_TO_JOINTS if abs_3d else capi.MOTION_REL_TO_JOINTS
        with torch.cuda.device(dev):
            capi.check(capi.load().cmdi_convert_motion(direction, _ptr(x), C * L, L, 1, B, L, C, _ptr(p), _ptr(m), _ptr(s), f64,
                                                       None, None, 0, 0.002, _ptr(out), joints_num * 3 * L, L, 1, _stream_ptr(dev)),
                       "cmdi_convert_motion")
        return out
    x = sample.to(torch.float32).contiguous()
    mean_t = torch.as_tensor(mean, dtype=torch.float32).to(x.device).contiguous()
    std_t = torch.as_tensor(std, dtype=torch.float32).to(x.device).contiguous()
    assert mean_t.shape == std_t.shape == (C,)
    out = torch.empty(B, joints_num, 3, L, dtype=torch.float32, device=x.device)
    with torch.cuda.device(x.device):
        capi.check(capi.load().cmdi_recover_from_ric(_ptr(x), C * L, 1, L, _ptr(mean_t), _ptr(std_t), B, L, C, joints_num, int(abs_3d),
                                                     _ptr(out), joints_num * 3 * L, 1, 3 * L, L, _stream_ptr(x.device)),
                   "cmdi_recover_from_ric")
    return out

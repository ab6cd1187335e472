"""CPU restatement of the reference's HumanML3D representation conversions (the checker of csrc/motion_features.cu).

Written from the behaviour of the reference (setarehc/diffusion-motion-inbetweening), batched over sequences:
  * extract_features             data_loaders/humanml/scripts/motion_process.py:50-187, with
                                 Skeleton.inverse_kinematics_np (common/skeleton.py:55-101, smooth_forward=True) and the
                                 quaternion helpers of common/quaternion.py (qmul :33-51, qrot :54-73, qbetween :387-397,
                                 quaternion_to_matrix / _cont6d :274-311)
  * inv_transform                data_loaders/humanml/data/dataset.py:378-382 (+ inv_random_projection :536-539)
  * abs3d_to_rel / rel_to_abs3d  dataset.py:1327-1401 with motion_to_rel_data / motion_to_abs_data (:1198-1288) and
                                 recover_root_rot_pos (motion_process.py:402-441); rot2xyz is the identity for pose_rep='xyz'

Dtypes follow the reference: its *_np quaternion helpers cast to float32 torch tensors, numpy's cross with an int64 axis
and gaussian_filter1d run in float64, the foot threshold compares in float64, and dataset statistics keep their dtype
(float64 statistics promote the (de-)normalisation to float64).  `oracle/make_golden_features.py` checks this module
against the unmodified reference functions.
"""
from __future__ import annotations

import numpy as np
import torch
from scipy.ndimage import gaussian_filter1d

from oracle import condmdi_oracle as O

# data_loaders/humanml/utils/paramUtil.py:32-55 (HumanML3D's 22-joint skeleton)
T2M_RAW_OFFSETS = np.array([[0, 0, 0], [1, 0, 0], [-1, 0, 0], [0, 1, 0], [0, -1, 0], [0, -1, 0], [0, 1, 0], [0, -1, 0],
                            [0, -1, 0], [0, 1, 0], [0, 0, 1], [0, 0, 1], [0, 1, 0], [1, 0, 0], [-1, 0, 0], [0, 0, 1],
                            [0, -1, 0], [0, -1, 0], [0, -1, 0], [0, -1, 0], [0, -1, 0], [0, -1, 0]])
T2M_KINEMATIC_CHAIN = [[0, 2, 5, 8, 11], [0, 1, 4, 7, 10], [0, 3, 6, 9, 12, 15], [9, 14, 17, 19, 21], [9, 13, 16, 18, 20]]
FACE_JOINTS = (2, 1, 17, 16)      # motion_process.py:18 (passed as l_hip, r_hip, sdr_r, sdr_l to the IK)
FID_R, FID_L = (8, 11), (7, 10)   # :16
FEET_THRE = 0.002


def qmul(q: torch.Tensor, r: torch.Tensor) -> torch.Tensor:
    """Hamilton product q * r, each component summed left to right over the products r_i q_j."""
    t = lambda i, j: r[..., i] * q[..., j]  # noqa: E731
    w = t(0, 0) - t(1, 1) - t(2, 2) - t(3, 3)
    x = t(0, 1) + t(1, 0) - t(2, 3) + t(3, 2)
    y = t(0, 2) + t(1, 3) + t(2, 0) - t(3, 1)
    z = t(0, 3) - t(1, 2) + t(2, 1) + t(3, 0)
    return torch.stack((w, x, y, z), -1)


def qinv(q: torch.Tensor) -> torch.Tensor:
    return torch.cat((q[..., :1], -q[..., 1:]), -1)


def qrot(q: torch.Tensor, v: torch.Tensor) -> torch.Tensor:
    qv = q[..., 1:]
    uv = torch.cross(qv, v, dim=-1)
    uuv = torch.cross(qv, uv, dim=-1)
    return v + 2 * (q[..., :1] * uv + uuv)


def qbetween(v0: torch.Tensor, v1: torch.Tensor) -> torch.Tensor:
    v = torch.cross(v0, v1, dim=-1)
    w = torch.sqrt((v0 ** 2).sum(-1, keepdim=True) * (v1 ** 2).sum(-1, keepdim=True)) + (v0 * v1).sum(-1, keepdim=True)
    q = torch.cat((w, v), -1)
    return q / torch.norm(q, dim=-1, keepdim=True)


def quat_to_cont6d(q: torch.Tensor) -> torch.Tensor:
    """The first two columns of the rotation matrix of q, column-major: (m00, m10, m20, m01, m11, m21)."""
    r, i, j, k = torch.unbind(q, -1)
    two_s = 2.0 / (q * q).sum(-1)
    col0 = (1 - two_s * (j * j + k * k), two_s * (i * j + k * r), two_s * (i * k - j * r))
    col1 = (two_s * (i * j - k * r), 1 - two_s * (i * i + k * k), two_s * (j * k + i * r))
    return torch.stack(col0 + col1, -1)


def _unit_np(v: np.ndarray) -> np.ndarray:
    return v / np.sqrt((v ** 2).sum(axis=-1))[..., None]


def root_quaternions(positions: np.ndarray) -> torch.Tensor:
    """(B, L, 22, 3) float32 -> (B, L, 4): qbetween(smoothed forward, +z), frame 0 forced to identity (skeleton.py:81)."""
    l_hip, r_hip, sdr_r, sdr_l = FACE_JOINTS
    across = _unit_np((positions[:, :, r_hip] - positions[:, :, l_hip]) + (positions[:, :, sdr_r] - positions[:, :, sdr_l]))
    forward = np.cross(np.array([[0, 1, 0]]), across, axis=-1)                 # float64
    forward = gaussian_filter1d(forward, 20, axis=1, mode="nearest")           # sigma 20, radius 80, float64
    forward = forward / np.sqrt((forward ** 2).sum(axis=-1))[..., None]
    target = torch.tensor([0.0, 0.0, 1.0]).expand(forward.shape)
    rq = qbetween(torch.from_numpy(forward).float(), target)
    rq[:, 0] = torch.tensor([1.0, 0.0, 0.0, 0.0])
    return rq


def extract_features(positions, feet_thre: float = FEET_THRE) -> torch.Tensor:
    """(B, L, 22, 3) or (L, 22, 3) float32 joint positions -> (B, L - 1, 263) de-normalised features (float32 values)."""
    pos = np.asarray(positions, dtype=np.float32)
    single = pos.ndim == 3
    if single:
        pos = pos[None]
    B, L = pos.shape[:2]
    rq = root_quaternions(pos)
    # inverse kinematics: R restarts at the root quaternion on every chain (skeleton.py:84-99)
    quat = torch.zeros(B, L, 22, 4)
    quat[:, :, 0] = rq
    for chain in T2M_KINEMATIC_CHAIN:
        R = rq
        for j0, j1 in zip(chain[:-1], chain[1:]):
            u = torch.from_numpy(T2M_RAW_OFFSETS[j1]).float().expand(B, L, 3)
            v = torch.from_numpy(_unit_np(pos[:, :, j1] - pos[:, :, j0]))
            r_loc = qmul(qinv(R), qbetween(u, v))
            quat[:, :, j1] = r_loc
            R = qmul(R, r_loc)
    cont6d = quat_to_cont6d(quat)
    P = torch.from_numpy(pos)
    velocity = qrot(rq[:, 1:], P[:, 1:, 0] - P[:, :-1, 0])                      # root linear velocity
    r_velocity = qmul(rq[:, 1:], qinv(rq[:, :-1]))                              # root angular velocity
    local = P.clone()                                                           # RIFKE: root xz removed, facing +z
    local[..., 0] -= P[:, :, 0:1, 0]
    local[..., 2] -= P[:, :, 0:1, 2]
    local = qrot(rq[:, :, None].expand(B, L, 22, 4), local)
    root_data = torch.cat((torch.from_numpy(np.arcsin(r_velocity[..., 2:3].numpy())), velocity[..., [0, 2]],
                           local[:, :-1, 0, 1:2]), -1)
    local_vel = qrot(rq[:, :-1, None].expand(B, L - 1, 22, 4), P[:, 1:] - P[:, :-1])

    def contacts(fid):
        d = pos[:, 1:, list(fid)] - pos[:, :-1, list(fid)]
        s = d[..., 0] ** 2 + d[..., 1] ** 2 + d[..., 2] ** 2
        return torch.from_numpy((s < np.array([feet_thre, feet_thre])).astype(np.float32))

    data = torch.cat((root_data, local[:, :-1, 1:].reshape(B, L - 1, -1), cont6d[:, :-1, 1:].reshape(B, L - 1, -1),
                      local_vel.reshape(B, L - 1, -1), contacts(FID_L), contacts(FID_R)), -1)
    return data[0] if single else data


def inv_transform(sample: torch.Tensor, mean, std, inv_proj=None) -> torch.Tensor:
    """(B, 263, 1, L) normalised -> (B, 1, L, 263) float32: [np.matmul(x, inv_proj)] then x * std + mean in the
    statistics' dtype, then .float() (dataset.py:1334-1335)."""
    x = sample.float().permute(0, 2, 3, 1)
    if inv_proj is not None:
        x = torch.from_numpy(np.matmul(x.numpy(), np.asarray(inv_proj)))
    return (x * torch.as_tensor(std) + torch.as_tensor(mean)).float()


def _normalise(feats: torch.Tensor, mean, std) -> torch.Tensor:
    """(B, L, 263) -> (B, 263, 1, L): (x - mean) / std in the statistics' dtype."""
    return ((feats - torch.as_tensor(mean)) / torch.as_tensor(std)).permute(0, 2, 1)[:, :, None, :]


def _features_dup(joints: torch.Tensor) -> torch.Tensor:
    """(B, L, 22, 3) -> (B, L, 263): features with the last row duplicated (dataset.py:1213-1215)."""
    f = extract_features(joints.numpy())
    return torch.cat((f, f[:, -1:]), 1)


def abs3d_to_rel(sample_abs: torch.Tensor, mean_abs, std_abs, mean_rel, std_rel, inv_proj=None) -> torch.Tensor:
    joints = O.recover_from_ric(inv_transform(sample_abs, mean_abs, std_abs, inv_proj), 22, abs_3d=True)[:, 0]
    return _normalise(_features_dup(joints), mean_rel, std_rel)


def root_abs(feats: torch.Tensor):
    """recover_root_rot_pos(abs_3d=False) of (B, L, 263) rows: (rot_ang (B, L), r_pos (B, L, 3))."""
    ang = torch.zeros_like(feats[..., 0])
    ang[..., 1:] = feats[..., :-1, 0]
    ang = torch.cumsum(ang, dim=-1)
    q = torch.zeros(feats.shape[:-1] + (4,))
    q[..., 0], q[..., 2] = torch.cos(ang), torch.sin(ang)
    r_pos = torch.zeros(feats.shape[:-1] + (3,))
    r_pos[..., 1:, 0], r_pos[..., 1:, 2] = feats[..., :-1, 1], feats[..., :-1, 2]
    r_pos = torch.cumsum(qrot(qinv(q), r_pos), dim=-2)
    r_pos[..., 1] = feats[..., 3]
    return ang, r_pos


def rel_to_abs3d(sample_rel: torch.Tensor, mean, std, mean_abs, std_abs, inv_proj=None) -> torch.Tensor:
    joints = O.recover_from_ric(inv_transform(sample_rel, mean, std, inv_proj), 22, abs_3d=False)[:, 0]
    feats = _features_dup(joints)
    ang, r_pos = root_abs(feats)
    feats = feats.clone()
    feats[..., 0] = ang
    feats[..., 1], feats[..., 2] = r_pos[..., 0], r_pos[..., 2]
    return _normalise(feats, mean_abs, std_abs)


def sample_to_joints(sample: torch.Tensor, mean, std, abs_3d: bool, inv_proj=None) -> torch.Tensor:
    """sample_to_motion (dataset.py:1301-1324) for a HumanML3D batch: (B, 263, 1, L) -> (B, 22, 3, L)."""
    pos = O.recover_from_ric(inv_transform(sample, mean, std, inv_proj), 22, abs_3d)
    return pos.reshape(-1, *pos.shape[2:]).permute(0, 2, 3, 1)


def ping_pong(joints: np.ndarray, L: int) -> np.ndarray:
    """Extend a (T, 22, 3) motion to L frames by playing it forwards and backwards (a continuous path)."""
    T = len(joints)
    idx = np.arange(L) % (2 * T - 2)
    idx = np.where(idx < T, idx, 2 * T - 2 - idx)
    return joints[idx]


def fixture_joints(motion: np.ndarray) -> dict:
    """The extract_features inputs of tests/golden/motion_features.*: the bundled motion (dataset/000021.npy, first
    22 joints, float32), two seeded perturbations of it, a copy with a standing-still stretch and its first 2 frames."""
    real = np.asarray(motion, dtype=np.float32)[:, :22]
    rng = np.random.default_rng(21)
    still = real.copy()
    still[40:90] = still[40]
    return {"real": real,
            "pert1": (real + rng.normal(0, 0.01, real.shape)).astype(np.float32),
            "pert2": (real + rng.normal(0, 0.03, real.shape)).astype(np.float32),
            "still": still,
            "two": real[:2].copy()}

"""Shared cases and gates of the SMPL-X body model tests (tests/test_body_model.py, tests/test_body_model_gpu.py).

Gates (metres).  The float32 restatement (oracle/smplx_oracle.py, the arithmetic of the `smplx` package) differs from
its float64 twin by at most ~5e-7 m on joints and ~1e-6 m on vertices of the full-size synthetic model (measured by
test_body_model.py::test_float32_floor_and_gates, DESIGN.md section 2); the gates are at least 4x that floor.
"""
import functools

import numpy as np
import torch

from synthetic_models import SMPLX_FULL_VERTS, SMPLX_SMALL_VERTS, smplx_arrays

JOINT_GATE = 1e-5           # max |joint - float64 joint|
VERTEX_GATE = 1e-5          # max |vertex - float64 vertex|
VELOCITY_GATE = 30 * JOINT_GATE    # 1 / (2 dt) = 15 amplifies each endpoint's position error
ROTATION_GATE = 2e-6


@functools.lru_cache(maxsize=None)
def small_arrays():
    return smplx_arrays(SMPLX_SMALL_VERTS)


@functools.lru_cache(maxsize=None)
def full_arrays():
    return smplx_arrays(SMPLX_FULL_VERTS)


def random_tree(rng, n=55):
    """A random valid 55-joint tree: parent[i] < i."""
    return tuple([-1] + [int(rng.integers(0, i)) for i in range(1, n)])


def random_poses(rng, rows, scale=0.6):
    """(rows, 165) float64 axis-angle with exact zero vectors, angles near 0 (1e-7 rad) and near pi."""
    p = rng.normal(0.0, scale, (rows, 55, 3))
    p[:, 3] = 0.0
    p[:, 11] = rng.normal(0.0, 1e-7, (rows, 3))
    axis = rng.normal(size=(rows, 3))
    p[:, 18] = axis / np.linalg.norm(axis, axis=-1, keepdims=True) * (np.pi - 1e-4)
    p[::3, 40] = 0.0
    return p.reshape(rows, 165)


def masked(poses, mask):
    """poses (..., 165) with the joints whose mask bit is clear set to zero (the FK kernel's joint mask)."""
    keep = torch.tensor([(mask >> j) & 1 for j in range(55)], dtype=poses.dtype, device=poses.device)
    return (poses.reshape(*poses.shape[:-1], 55, 3) * keep[:, None]).reshape(poses.shape)

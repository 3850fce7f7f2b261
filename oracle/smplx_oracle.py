"""Torch restatement of the SMPL-X forward pass (TEST / MEASUREMENT INFRASTRUCTURE; never imported by the product).

Restated from the published SMPL-X model and the `smplx` package conventions the reference depends on
(smplx.create(model_type='smplx', num_betas=300, num_expression_coeffs=100, use_pca=False), flat_hand_mean False):

    full_pose = [global_orient, body 21, jaw, leye, reye, left hand 15, right hand 15] + pose_mean (the hand means)
    v_shaped  = v_template + shapedirs[..., :300] . betas + shapedirs[..., 300:400] . expression
    J         = J_regressor @ v_shaped                                           (55 joints)
    R_j       = I + sin K + (1 - cos) K K, angle = |r + 1e-8|, K the cross matrix of r / angle
    v_posed   = v_shaped + (R[1:] - I).flatten() @ posedirs.reshape(-1, 486).T
    G_i       = G_parent(i) [R_i | J_i - J_parent(i)],  A_i = G_i - [0 | G_i (J_i, 0)]
    vertex    = (sum_j w_vj A_j) (v_posed, 1) + transl,  joints = G_i[:3, 3] + transl

`dtype` selects the arithmetic: float64 for the parity gates, float32 to measure the float32 floor (and to stand in for
the `smplx` package, which also runs in float32).  Joints 55-126 (vertex-selected tips and face landmarks) are NaN: they
are out of scope, and any use of them fails loudly.
"""
from __future__ import annotations

import os

import numpy as np
import torch

N_JOINTS, N_BETAS, N_EXPR = 55, 300, 100
N_OUT_JOINTS = 127


def load_arrays(path):
    """The arrays of an SMPL-X npz; a pickled scipy.sparse J_regressor is densified (smplx accepts both)."""
    raw = np.load(path, allow_pickle=True)
    out = {k: raw[k] for k in raw.files}
    jr = out.get("J_regressor")
    if jr is not None and jr.dtype == object:
        jr = jr.item()
        out["J_regressor"] = np.asarray(jr.toarray() if hasattr(jr, "toarray") else jr)
    return out


def rodrigues(r):
    """(n, 3) axis-angle -> (n, 3, 3), smplx batch_rodrigues order of operations."""
    angle = torch.norm(r + 1e-8, dim=1, keepdim=True)
    k = r / angle
    cos, sin = torch.cos(angle)[:, :, None], torch.sin(angle)[:, :, None]
    kx, ky, kz = k[:, 0], k[:, 1], k[:, 2]
    zero = torch.zeros_like(kx)
    K = torch.stack([zero, -kz, ky, kz, zero, -kx, -ky, kx, zero], dim=1).view(-1, 3, 3)
    eye = torch.eye(3, dtype=r.dtype, device=r.device)[None]
    return eye + sin * K + (1 - cos) * torch.bmm(K, K)


def rigid_transform(rot, J, parents):
    """FK with a Python loop over the joints, as smplx does: returns posed joints (n, 55, 3) and A (n, 55, 4, 4)."""
    n = rot.shape[0]
    rel = J.clone()
    rel[:, 1:] = J[:, 1:] - J[:, parents[1:]]
    bottom = torch.zeros(n, rot.shape[1], 1, 4, dtype=rot.dtype, device=rot.device)
    bottom[..., 3] = 1
    local = torch.cat([torch.cat([rot, rel[..., None]], dim=3), bottom], dim=2)
    chain = [local[:, 0]]
    for i in range(1, len(parents)):
        chain.append(torch.matmul(chain[int(parents[i])], local[:, i]))
    G = torch.stack(chain, dim=1)
    posed = G[:, :, :3, 3]
    jh = torch.cat([J, torch.zeros_like(J[..., :1])], dim=2)[..., None]
    A = G - torch.nn.functional.pad(torch.matmul(G, jh), [3, 0])
    return posed, A


class SmplxRestatement(torch.nn.Module):
    """smplx.SMPLX-like module: forward(betas=, expression=, transl=, global_orient=, body_pose=, jaw_pose=, leye_pose=,
    reye_pose=, left_hand_pose=, right_hand_pose=, return_joints=, return_verts=) -> {"joints", "vertices"}.
    Absent arguments are zeros of the batch size of the given ones."""

    def __init__(self, arrays, dtype=torch.float64):
        super().__init__()
        t = lambda a: torch.as_tensor(np.asarray(a, dtype=np.float64)).to(dtype)
        parents = np.asarray(arrays["kintree_table"][0], dtype=np.int64).copy()
        parents[0] = -1
        self.parents = parents
        self.register_buffer("v_template", t(arrays["v_template"]))
        self.register_buffer("shapedirs", t(arrays["shapedirs"][:, :, :N_BETAS + N_EXPR]))
        self.register_buffer("posedirs", t(arrays["posedirs"].reshape(-1, arrays["posedirs"].shape[-1]).T))
        self.register_buffer("J_regressor", t(arrays["J_regressor"]))
        self.register_buffer("lbs_weights", t(arrays["weights"]))
        mean = np.zeros(3 * N_JOINTS)
        mean[75:120], mean[120:] = arrays["hands_meanl"], arrays["hands_meanr"]
        self.register_buffer("pose_mean", t(mean))

    def forward(self, betas=None, expression=None, transl=None, global_orient=None, body_pose=None, jaw_pose=None,
                leye_pose=None, reye_pose=None, left_hand_pose=None, right_hand_pose=None, return_joints=True,
                return_verts=True, **_):
        dt, dev = self.v_template.dtype, self.v_template.device
        given = [x for x in (global_orient, body_pose, jaw_pose, leye_pose, reye_pose, left_hand_pose, right_hand_pose,
                             transl, expression) if x is not None]
        n = given[0].shape[0] if given else (1 if betas is None else betas.shape[0])
        z = lambda x, c: torch.zeros(n, c, dtype=dt, device=dev) if x is None else x.to(dt).reshape(n, c)
        full_pose = torch.cat([z(global_orient, 3), z(body_pose, 63), z(jaw_pose, 3), z(leye_pose, 3), z(reye_pose, 3),
                               z(left_hand_pose, 45), z(right_hand_pose, 45)], dim=1) + self.pose_mean
        b = torch.zeros(n, N_BETAS, dtype=dt, device=dev) if betas is None else betas.to(dt)
        if b.shape[0] != n:
            b = b.expand(n // b.shape[0], -1)
        coef = torch.cat([b, z(expression, N_EXPR)], dim=1)
        v_shaped = self.v_template + torch.einsum("bl,mkl->bmk", coef, self.shapedirs)
        J = torch.einsum("bik,ji->bjk", v_shaped, self.J_regressor)
        rot = rodrigues(full_pose.view(-1, 3)).view(n, N_JOINTS, 3, 3)
        eye = torch.eye(3, dtype=dt, device=dev)
        v_posed = v_shaped + torch.matmul((rot[:, 1:] - eye).reshape(n, -1), self.posedirs).view(n, -1, 3)
        posed, A = rigid_transform(rot, J, self.parents)
        tr = z(transl, 3)[:, None]
        out = {}
        if return_joints:
            nan = torch.full((n, N_OUT_JOINTS - N_JOINTS, 3), float("nan"), dtype=dt, device=dev)
            out["joints"] = torch.cat([posed + tr, nan], dim=1)
        if return_verts:
            T = torch.matmul(self.lbs_weights, A.view(n, N_JOINTS, 16)).view(n, -1, 4, 4)
            out["vertices"] = (torch.matmul(T[:, :, :3, :3], v_posed[..., None])[..., 0] + T[:, :, :3, 3]) + tr
        return out


def create(model_path, model_type="smplx", gender="NEUTRAL_2020", ext="npz", dtype=torch.float32, **_):
    """smplx.create(...) stand-in: loads <model_path>/smplx/SMPLX_<GENDER>.<ext> (or model_path itself when it is a
    file) into the restatement.  Keyword arguments of the reference call sites (use_face_contour, num_betas=300,
    num_expression_coeffs=100, use_pca=False, ...) are accepted; the model is fixed to those settings."""
    assert model_type == "smplx", model_type
    path = model_path if os.path.isfile(model_path) else os.path.join(model_path, "smplx", f"SMPLX_{gender.upper()}.{ext}")
    return SmplxRestatement(load_arrays(path), dtype=dtype)


def forward_poses(model, poses, betas=None, expression=None, transl=None, vertices=True):
    """The body model's call convention on the restatement: poses (n, 165), betas (n, 300), expression (n, 100),
    transl (n, 3) -> (joints (n, 55, 3), vertices (n, V, 3) or None)."""
    out = model(betas=betas, expression=expression, transl=transl, global_orient=poses[:, :3], body_pose=poses[:, 3:66],
                jaw_pose=poses[:, 66:69], leye_pose=poses[:, 69:72], reye_pose=poses[:, 72:75],
                left_hand_pose=poses[:, 75:120], right_hand_pose=poses[:, 120:165], return_verts=vertices)
    return out["joints"][:, :N_JOINTS], out.get("vertices")

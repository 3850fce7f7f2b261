"""SMPL-X body model on the GPU: joint positions, mesh vertices and the motion representation of generated poses.

The step every consumer of the generated SMPL-X parameters runs next in the reference (the smplx forward pass in
emage_utils/motion_rep_transfer.py:38-50, emage_utils/motion_io.py:117-140, datasets/foot_contact.py:46-58), with the
conventions of smplx.create(model_type='smplx', num_betas=300, num_expression_coeffs=100, use_pca=False): the hand
means are added to the pose (flat_hand_mean False), joints 0-54 are the forward-kinematics joints.

    model = SmplxBodyModel.from_npz("SMPLX_NEUTRAL_2020.npz", "cuda")
    out = model.forward(pred["motion_axis_angle"], expression=pred["expression"], transl=pred["trans"], vertices=True)

Three launches per call (DESIGN.md section 9): pm_smplx_fk_f32 (rest joints, Rodrigues, FK, and the vertex GEMM's
operand row), the tap-GEMM [betas | expression | pose feature] @ [shapedirs | posedirs]^T + v_template in the engine's
precision (engine.set_precision), and pm_smplx_skin_f32.  No host synchronisation: a call can be captured in a CUDA
graph once the current precision's weights are packed (any eager call packs them).
"""
from __future__ import annotations

import numpy as np
import torch

from . import _lib, ops
from .emage_audio import engine

N_JOINTS, N_BETAS, N_EXPR, N_POSE_FEAT = 55, 300, 100, 486
N_COEF = N_BETAS + N_EXPR + N_POSE_FEAT                   # 886: K of the vertex blend GEMM
ALL_JOINTS = (1 << N_JOINTS) - 1
# get_motion_rep_tensor zeroes global orient (0), jaw (22) and the eyes (23, 24): only body and hands are posed
MOTION_REP_JOINTS = ALL_JOINTS & ~((1 << 0) | (1 << 22) | (1 << 23) | (1 << 24))
_KEYS = ("v_template", "shapedirs", "posedirs", "J_regressor", "weights", "kintree_table", "hands_meanl", "hands_meanr")


def _dense(a, name):
    """A dense float64 array; a pickled scipy.sparse matrix (J_regressor in some SMPL-X files) is densified."""
    if isinstance(a, np.ndarray) and a.dtype == object and a.ndim == 0:
        a = a.item()
    if hasattr(a, "toarray"):
        a = a.toarray()
    try:
        return np.asarray(a, dtype=np.float64)
    except (TypeError, ValueError) as e:
        raise ValueError(f"SMPL-X model: {name} is not a numeric array ({e})") from None


def _levels(parents):
    """Joints ordered by depth and the start of each level in that order."""
    depth = np.zeros(len(parents), dtype=np.int64)
    for i in range(1, len(parents)):
        depth[i] = depth[parents[i]] + 1
    order = np.argsort(depth, kind="stable")
    start = np.searchsorted(depth[order], np.arange(depth.max() + 2))
    return order, start


class SmplxBodyModel:
    """SMPL-X forward pass for (batch, frames) of generated poses.  Build with from_npz()."""

    def __init__(self, arrays, device="cuda"):
        a = {k: arrays[k] for k in _KEYS if k in arrays}
        missing = [k for k in _KEYS if k not in a]
        if missing:
            raise ValueError(f"SMPL-X model: missing key(s) {missing}")
        v_template = _dense(a["v_template"], "v_template")
        if v_template.ndim != 2 or v_template.shape[1] != 3 or v_template.shape[0] < 1:
            raise ValueError(f"SMPL-X model: v_template must be (V, 3), got {v_template.shape}")
        nv = v_template.shape[0]
        shapedirs = _dense(a["shapedirs"], "shapedirs")
        if shapedirs.ndim != 3 or shapedirs.shape[:2] != (nv, 3):
            raise ValueError(f"SMPL-X model: shapedirs must be ({nv}, 3, >= 400), got {shapedirs.shape}")
        if shapedirs.shape[2] < N_BETAS + N_EXPR:
            raise ValueError(f"SMPL-X model: shapedirs has {shapedirs.shape[2]} shape components, "
                             f"{N_BETAS} betas + {N_EXPR} expression coefficients need 400")
        checks = {"posedirs": (nv, 3, N_POSE_FEAT), "J_regressor": (N_JOINTS, nv), "weights": (nv, N_JOINTS),
                  "kintree_table": (2, N_JOINTS), "hands_meanl": (45,), "hands_meanr": (45,)}
        d = {}
        for k, shape in checks.items():
            d[k] = _dense(a[k], k)
            if d[k].shape != shape:
                raise ValueError(f"SMPL-X model: {k} must be {shape}, got {d[k].shape}")
        parents = d["kintree_table"][0].astype(np.int64)
        parents[0] = -1
        bad = [i for i in range(1, N_JOINTS) if not 0 <= parents[i] < i]
        if bad:
            raise ValueError(f"SMPL-X model: kintree_table is not a tree with parent[i] < i (joints {bad})")
        if not all(np.isfinite(x).all() for x in (v_template, shapedirs, *d.values())):
            raise ValueError("SMPL-X model: non-finite values")
        self.n_verts, self.device = nv, torch.device(device)
        self.faces = np.asarray(arrays["f"]) if "f" in arrays else None

        # float64 precompute on the host, float32 on the device
        dirs = shapedirs[:, :, :N_BETAS + N_EXPR]
        jreg = d["J_regressor"]
        f32 = lambda x: torch.as_tensor(np.ascontiguousarray(x), dtype=torch.float32, device=self.device)
        i32 = lambda x: torch.as_tensor(np.ascontiguousarray(x), dtype=torch.int32, device=self.device)
        self.j_template = f32((jreg @ v_template).reshape(-1))                                   # (165,)
        self.j_dirs = f32(np.einsum("jv,vck->kjc", jreg, dirs).reshape(N_BETAS + N_EXPR, -1))    # (400, 165)
        mean = np.zeros(3 * N_JOINTS)
        mean[75:120], mean[120:] = d["hands_meanl"], d["hands_meanr"]
        self.pose_mean = f32(mean)
        order, start = _levels(parents)
        self.parents, self.level_order, self.level_start = i32(parents), i32(order), i32(start)
        self.n_levels = len(start) - 1
        # vertex blend GEMM: out (rows, 3V) = [betas | expression | pose feature] @ W^T + v_template, W (3V, 886)
        w = np.concatenate([dirs.reshape(3 * nv, -1), d["posedirs"].reshape(3 * nv, -1)], axis=1)
        self.blend = engine._Linear(None, w=f32(w), b=f32(v_template.reshape(-1)))
        wt = d["weights"]
        nz = wt != 0
        self.skin_csr = (i32(np.concatenate([[0], np.cumsum(nz.sum(1))])), i32(np.nonzero(nz)[1]), f32(wt[nz]))
        self._tables = (self.j_template, self.j_dirs, self.pose_mean, self.parents, self.level_order, self.level_start)

    @classmethod
    def from_npz(cls, path, device="cuda"):
        """Load and validate an SMPL-X model file (SMPLX_NEUTRAL_2020.npz layout).  Raises ValueError naming the problem."""
        raw = np.load(path, allow_pickle=True)
        return cls({k: raw[k] for k in raw.files}, device)

    # ------------------------------------------------------------------------------------------------------------
    def _check(self, x, name, shape):
        if not torch.is_tensor(x):
            raise ValueError(f"{name} must be a tensor, got {type(x).__name__}")
        if not x.is_cuda:
            raise _lib.PmError(f"{name}: the body model needs CUDA tensors (no CPU fallback)")
        if x.device != self.device and not (self.device.index is None and x.device.index == torch.cuda.current_device()):
            raise ValueError(f"{name} is on {x.device}, the body model on {self.device}")
        if tuple(x.shape) != shape or x.dtype != torch.float32:
            raise ValueError(f"{name} must be a {shape} float32 tensor, got {tuple(x.shape)} {x.dtype}")
        if x.stride(-1) != 1:
            raise ValueError(f"{name}: the last dimension must be dense")
        return x

    def _poses(self, poses):
        if not torch.is_tensor(poses) or poses.dim() != 3:
            raise ValueError(f"poses must be a (batch, frames, 165) tensor, got "
                             f"{tuple(poses.shape) if torch.is_tensor(poses) else type(poses).__name__}")
        batch, t = poses.shape[:2]
        self._check(poses, "poses", (batch, t, 3 * N_JOINTS))
        if batch * t == 0:
            raise ValueError("poses has no frames")
        return batch, t

    def _fk(self, poses, betas, expression, transl, mask, vertices):
        """pm_smplx_fk_f32: (joints (rows, 55, 3), A (rows, 55, 12) | None, GEMM operand Planes | fp32 (rows, 888) | None)."""
        batch, t = poses.shape[:2]
        rows = batch * t
        joints = torch.empty(rows, N_JOINTS, 3, device=poses.device, dtype=torch.float32)
        rel = feat = planes = None
        if vertices:
            rel = torch.empty(rows, N_JOINTS, 12, device=poses.device, dtype=torch.float32)
            ns = engine._ns()
            if ns:
                planes = ops._new_planes(ns, (1, rows), N_COEF, poses.device)
            else:
                feat = torch.empty(rows, ops._round_up(N_COEF, 8), device=poses.device, dtype=torch.float32)
        ops.smplx_fk(poses, betas, expression, transl, mask, self._tables, joints, rel, feat, planes)
        return joints, rel, (planes if planes is not None else feat)

    def _blend(self, operand, rows):
        """v_posed (rows, ld) fp32, ld = 3V rounded up to 4 (aligned epilogue stores): the vertex blend GEMM."""
        n3 = 3 * self.n_verts
        buf = torch.empty(rows, ops._round_up(n3, 4), device=self.device, dtype=torch.float32)
        out = buf[:, :n3].unsqueeze(0)
        if isinstance(operand, ops.Planes):
            ops.tapgemm_tc(operand, self.blend.packed(operand.nsplit), self.blend.b, rows_out=rows, out=out)
        else:
            ops.tapgemm(operand[:, :N_COEF].unsqueeze(0), self.blend.w, self.blend.b, out=out)
        return buf

    @torch.no_grad()
    def forward(self, poses, betas=None, expression=None, transl=None, vertices=False):
        """poses (B, T, 165) axis-angle in BEAT / motion_axis_angle joint order, betas (B, 300) per clip, expression
        (B, T, 100), transl (B, T, 3); float32 CUDA tensors, any clip / frame strides with a dense last dimension (the
        outputs of CapturedPipeline / generate() are read in place).  Returns {"joints": (B, T, 55, 3)} and, with
        vertices=True, "vertices": (B, T, V, 3) (a view with rows 3V rounded up to 4 apart)."""
        batch, t = self._poses(poses)
        if betas is not None:
            self._check(betas, "betas", (batch, N_BETAS))
        if expression is not None:
            self._check(expression, "expression", (batch, t, N_EXPR))
        if transl is not None:
            self._check(transl, "transl", (batch, t, 3))
        if not vertices:
            joints, _, _ = self._fk(poses, betas, expression, transl, ALL_JOINTS, False)
            return {"joints": joints.view(batch, t, N_JOINTS, 3)}
        joints, verts = self._vertices(poses, betas, expression, transl, ALL_JOINTS)
        return {"joints": joints.view(batch, t, N_JOINTS, 3), "vertices": verts}

    def _vertices(self, poses, betas, expression, transl, mask):
        """FK, vertex blend GEMM and skinning of validated inputs with the joints of `mask` posed: (joints (rows, 55,
        3), vertices (B, T, V, 3) a view with rows 3V rounded up to 4 apart)."""
        batch, t = poses.shape[:2]
        joints, rel, operand = self._fk(poses, betas, expression, transl, mask, True)
        buf = self._blend(operand, batch * t)
        ops.smplx_skin(buf, self.n_verts, self.skin_csr, rel, transl, t)
        return joints, buf[:, :3 * self.n_verts].view(batch, t, self.n_verts, 3)

    __call__ = forward

    @torch.no_grad()
    def motion_rep(self, poses, pose_fps=30):
        """get_motion_rep_tensor (emage_utils/motion_rep_transfer.py:31-72) for poses (B, T >= 2, 165): joints of the
        body and hands only (global orient, jaw, eyes, expression, betas and transl zero, as in the reference, whose
        betas argument is ignored), velocities one-sided at the clip ends and central inside, rot6d by the quaternion
        route.  Returns position / velocity (B, T, 55, 3), rotation (B, T, 55, 6), angular_velocity (B, T, 55, 3) as
        views of rep15d (B, T, 825), and axis_angle (the poses given)."""
        batch, t = self._poses(poses)
        if t < 2:
            raise ValueError(f"motion_rep needs at least 2 frames per clip (velocities), got {t}")
        joints, _, _ = self._fk(poses, None, None, None, MOTION_REP_JOINTS, False)
        rep = torch.empty(batch, t, N_JOINTS * 15, device=poses.device, dtype=torch.float32)
        dt = 1 / pose_fps
        ops.motion_rep(poses, joints, np.float32(dt), np.float32(2 * dt), rep)
        v = rep.view(batch, t, N_JOINTS, 15)
        return {"position": v[..., 0:3], "velocity": v[..., 3:6], "rotation": v[..., 6:12], "axis_angle": poses,
                "angular_velocity": v[..., 12:15], "rep15d": rep}

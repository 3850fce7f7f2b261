"""SMPL-X mesh frames on the GPU: the reference's face, body and prediction-beside-ground-truth views of poses.

emage_utils/fast_render.py renders every frame of the SMPL-X mesh with pyrender in one of three layouts, all drawn here
with three kernels per chunk of frames, each taking the view count (include/pm_emage.h pm_mesh_vertex_f32 /
pm_mesh_raster / pm_mesh_shade_u8, DESIGN.md section 10):
  - render_sequence: render_one_sequence_with_face (:286-321), a face close-up (only the jaw posed, the mesh scaled x7
    and moved down by 10) left of the full body, 960 x 720;
  - render_body: render_one_sequence_no_gt (:363-391), the full body alone, 480 x 720 (CaMN and DisCo output, upsampled
    to 30 fps as the npz writer does);
  - render_pair: render_one_sequence (:323-361), the prediction left of the ground truth, 960 x 720.

    renderer = MeshRenderer(SmplxBodyModel.from_npz("SMPLX_NEUTRAL_2020.npz"))
    frames = renderer.render_sequence(pred["motion_axis_angle"], pred["expression"], pred["trans"])  # (B, T', 720, 960, 3)
    frames = renderer.render_body(camn["motion_axis_angle"], trans, upsample=2)                   # (B, T', 720, 480, 3)

Geometry, framing, layout and frame count follow the reference; the shading is Lambert with its directional light (not
pyrender's PBR shader, so pixel parity with pyrender is not claimed).  No host synchronisation: a call can be captured
in a CUDA graph after one eager call.
"""
from __future__ import annotations

import numbers

import numpy as np
import torch

from . import ops
from .body_model import ALL_JOINTS

W, H, VIEWS = 480, 720, 2              # one view (fast_render.py args); two-view frames are VIEWS views side by side
FPS = 30                               # render_video_fps: render_sequence draws whole seconds, T // 30 * 30 frames
CHUNK = 8                              # frames per launch group: 8 x 2 visibility buffers of 2.8 MB stay in the 50 MB L2
JAW_ONLY = 1 << 22                     # the face view poses the jaw alone (zeroed joints keep the hand means)
FACE_VIEW = (7.0, (0.0, -10.0, 0.0))   # (scale, offset): v * 7 - (0, 10, 0), fast_render.py:312-315
BODY_VIEW = (1.0, (0.0, 0.0, 0.0))


class MeshRenderer:
    """Renders the triangle list of an SmplxBodyModel (its model file's `f`).  Raises ValueError on malformed faces."""

    def __init__(self, body_model):
        nv, faces = body_model.n_verts, body_model.faces
        if faces is None:
            raise ValueError("SMPL-X model: no faces (key 'f') in the model file: nothing to render")
        faces = np.asarray(faces)
        if faces.ndim != 2 or faces.shape[1] != 3 or faces.shape[0] < 1:
            raise ValueError(f"SMPL-X model: faces must be (F, 3), got {faces.shape}")
        if faces.dtype.kind not in "iu":
            raise ValueError(f"SMPL-X model: faces must be integer vertex indices, got {faces.dtype}")
        if faces.min() < 0 or faces.max() >= nv:
            raise ValueError(f"SMPL-X model: face indices must lie in [0, {nv}), got [{faces.min()}, {faces.max()}]")
        faces = faces.astype(np.int64)
        n_faces = faces.shape[0]
        # vertex -> incident faces in ascending face index (each face once): the normal sum's fixed order
        pairs = np.unique(faces * n_faces + np.arange(n_faces)[:, None])
        vf_ptr = np.searchsorted(pairs // n_faces, np.arange(nv + 1))
        dev = body_model.device
        i32 = lambda x: torch.as_tensor(np.ascontiguousarray(x), dtype=torch.int32, device=dev)
        self.body_model, self.n_verts, self.n_faces, self.device = body_model, nv, n_faces, dev
        self.faces = i32(faces)
        self.vf_csr = (i32(vf_ptr), i32(pairs % n_faces))

    def _frames(self, v, name):
        if not torch.is_tensor(v):
            raise ValueError(f"{name} must be a tensor, got {type(v).__name__}")
        if v.dim() == 4:
            v = v.view(-1, *v.shape[2:])
        if v.dim() != 3 or tuple(v.shape[1:]) != (self.n_verts, 3) or v.dtype != torch.float32:
            raise ValueError(f"{name} must be (N, {self.n_verts}, 3) or (B, T, {self.n_verts}, 3) float32, got "
                             f"{tuple(v.shape)} {v.dtype}")
        if v.stride(2) != 1 or v.stride(1) != 3:
            raise ValueError(f"{name}: each frame's vertices must be dense")
        return v

    @torch.no_grad()
    def render(self, vertices, views=None, out=None):
        """Draw N frames of one or two views.  vertices: one tensor, or (left, right), each (N, V, 3) or (B, T, V, 3)
        float32 CUDA with dense frames any stride apart (body model output is read in place); views: the affine transform
        p * scale + offset of each view, (scale, (ox, oy, oz)) for one view or a pair of them (default: BODY_VIEW for
        one view, (FACE_VIEW, BODY_VIEW) for two).  Returns out (N, 720, 480 * views, 3) uint8 (each frame dense)."""
        if torch.is_tensor(vertices):
            vertices = (vertices,)
        if views is None:
            views = (FACE_VIEW, BODY_VIEW)[-len(vertices):]
        elif len(views) == 2 and isinstance(views[0], (int, float)):
            views = (views,)                                   # one (scale, offset) transform
        nv = len(vertices)
        if nv not in (1, VIEWS) or len(views) != nv:
            raise ValueError(f"render draws 1 or {VIEWS} views: give as many vertex tensors as transforms, got "
                             f"{nv} and {len(views)}")
        verts = [self._frames(v, f"vertices[{i}]") for i, v in enumerate(vertices)]
        n = verts[0].shape[0]
        if any(v.shape[0] != n for v in verts):
            raise ValueError(f"the views have {[v.shape[0] for v in verts]} frames")
        if out is None:
            out = torch.empty(n, H, nv * W, 3, dtype=torch.uint8, device=verts[0].device)
        elif tuple(out.shape) != (n, H, nv * W, 3) or out.dtype != torch.uint8 or (n and not out[0].is_contiguous()):
            raise ValueError(f"out must be ({n}, {H}, {nv * W}, 3) uint8 with dense frames")
        c = min(n, CHUNK)
        if c == 0:
            return out
        dev = verts[0].device
        xy = torch.empty(c, nv, self.n_verts, 2, dtype=torch.int32, device=dev)
        depth = torch.empty(c, nv, self.n_verts, device=dev)
        normal = torch.empty(c, nv, self.n_verts, 3, device=dev)
        vis = torch.empty(c, nv, H, W, dtype=torch.int64, device=dev)
        for s in range(0, n, CHUNK):
            k = min(CHUNK, n - s)
            ops.mesh_vertex([v[s:s + k] for v in verts], views, self.faces, self.vf_csr, xy[:k], depth[:k], normal[:k])
            ops.mesh_raster(xy[:k], depth[:k], self.faces, vis[:k])
            ops.mesh_shade(vis[:k], xy[:k], normal[:k], self.faces, out[s:s + k])
        return out

    @torch.no_grad()
    def render_sequence(self, poses, expression, trans, betas=None, out=None):
        """render_one_sequence_with_face (fast_render.py:286-321) for clips of generated poses: poses (B, T, 165),
        expression (B, T, 100), trans (B, T, 3), betas (B, 300) or None, float32 CUDA tensors as generate() /
        CapturedPipeline return them (read in place).  Every frame uses frame 0's trans (remove_transl=True); the face
        view poses only the jaw.  Returns out (B, T // 30 * 30, 720, 960, 3) uint8: face view left, body view right."""
        bm = self.body_model
        batch, t = bm._poses(poses)
        bm._check(expression, "expression", (batch, t, 100))
        bm._check(trans, "trans", (batch, t, 3))
        if betas is not None:
            bm._check(betas, "betas", (batch, 300))
        n = t // FPS * FPS
        return self._draw([(poses, betas, expression, trans, JAW_ONLY), (poses, betas, expression, trans, ALL_JOINTS)],
                          (FACE_VIEW, BODY_VIEW), n, out)

    def _draw(self, sides, views, n, out):
        """Frames [0, n) of every clip, one image view per side (poses, betas, expression or None, trans, joint mask),
        each side posed with its clip's frame-0 translation (remove_transl=True) and drawn with the transform(s)
        `views`.  out: None or a contiguous (B, n, 720, 480 * len(sides), 3) uint8 tensor; returns it."""
        batch, dev = sides[0][0].shape[0], sides[0][0].device
        shape = (batch, n, H, len(sides) * W, 3)
        if out is None:
            out = torch.empty(shape, dtype=torch.uint8, device=dev)
        elif tuple(out.shape) != shape or out.dtype != torch.uint8 or not out.is_contiguous():
            raise ValueError(f"out must be a contiguous {shape} uint8 tensor")
        if n == 0:
            return out
        verts = [self.body_model._vertices(p[:, :n], b, None if e is None else e[:, :n], tr[:, :1].expand(batch, n, 3),
                                           mask)[1] for p, b, e, tr, mask in sides]
        self.render(verts, views, out.view(batch * n, *shape[2:]))
        return out

    @torch.no_grad()
    def render_body(self, poses, trans, expression=None, betas=None, upsample=1, out=None):
        """render_one_sequence_no_gt (fast_render.py:363-391) of the npz the reference writer saves with upsample=k
        (test_camn_audio.py / test_disco_audio.py: k = 30 // pose_fps).  poses (B, t, 165), trans (B, t, 3) (only frame
        0 is used: remove_transl=True), expression (B, t, 100) or None (zeros, as the writer stores for CaMN and DisCo),
        betas (B, 300) or None; float32 CUDA tensors, read in place.  With upsample = k > 1, poses and expression are
        upsampled to k*t frames first (ops.time_upsample: motion_io.time_upsample_numpy as the renderer reads it back);
        frame 0 of trans is unchanged by it.  Returns out (B, k*t // 30 * 30, 720, 480, 3) uint8: one body view."""
        bm = self.body_model
        batch, t = bm._poses(poses)
        bm._check(trans, "trans", (batch, t, 3))
        if expression is not None:
            bm._check(expression, "expression", (batch, t, 100))
        if betas is not None:
            bm._check(betas, "betas", (batch, 300))
        if not isinstance(upsample, numbers.Integral) or isinstance(upsample, bool) or upsample < 1:
            raise ValueError(f"upsample must be a positive int, got {upsample!r}")
        upsample = int(upsample)
        n = upsample * t // FPS * FPS
        if upsample > 1 and n:
            poses = ops.time_upsample(poses, upsample)
            expression = None if expression is None else ops.time_upsample(expression, upsample)
        return self._draw([(poses, betas, expression, trans, ALL_JOINTS)], BODY_VIEW, n, out)

    @torch.no_grad()
    def render_pair(self, poses, trans, gt_poses, gt_trans, expression=None, betas=None, gt_expression=None,
                    gt_betas=None, out=None):
        """render_one_sequence (fast_render.py:323-361): the prediction beside the ground truth, as the reference's
        training scripts inspect results.  poses (B, t, 165), trans (B, t, 3), expression (B, t, 100) or None, betas
        (B, 300) or None for the prediction; gt_* the same for the ground truth with its own length t_gt >= n =
        t // 30 * 30, of which frames [0, n) are drawn.  Each side uses its own betas, expression and frame-0
        translation, all joints posed.  Float32 CUDA tensors, read in place.  Returns out (B, n, 720, 960, 3) uint8:
        prediction left, ground truth right.  Raises ValueError when the ground truth is shorter than n frames."""
        bm = self.body_model
        batch, t = bm._poses(poses)
        gb, gt_t = bm._poses(gt_poses)
        if gb != batch:
            raise ValueError(f"gt_poses has {gb} clips, poses {batch}")
        n = t // FPS * FPS
        if gt_t < n:
            raise ValueError(f"the ground truth has {gt_t} frames, fewer than the {n} frames drawn of the prediction")
        sides = []
        for p, tr, e, b, tag, tt in ((poses, trans, expression, betas, "", t),
                                     (gt_poses, gt_trans, gt_expression, gt_betas, "gt_", gt_t)):
            bm._check(tr, tag + "trans", (batch, tt, 3))
            if e is not None:
                bm._check(e, tag + "expression", (batch, tt, 100))
            if b is not None:
                bm._check(b, tag + "betas", (batch, 300))
            sides.append((p, b, e, tr, ALL_JOINTS))
        return self._draw(sides, (BODY_VIEW, BODY_VIEW), n, out)

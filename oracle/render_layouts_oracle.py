"""CPU restatement of the body-only and prediction-beside-ground-truth render layouts (TEST / MEASUREMENT
INFRASTRUCTURE; never imported by the product).

Follows emage_utils/fast_render.py where cited, next to render_oracle.sequence_vertices (render_one_sequence_with_face):
  - render_one_sequence_no_gt (:363-391): the body alone, all joints posed, one 480 x 720 view per frame (:71-79
    do_render_one_frame_no_gt, :95-106 write_images_from_queue_no_gt);
  - render_one_sequence (:323-361): the prediction's body left of the ground truth's (:58-69, :80-92), the ground truth
    read over the prediction's frames, each side with its own betas, expression and frame-0 trans.
Both draw T // 30 * 30 frames, every frame at frame 0's trans (remove_transl=True).  The frames themselves are
render_oracle.render_views with one view ([BODY_VIEW]) or two ([BODY_VIEW, BODY_VIEW]).
"""
from __future__ import annotations

import torch

from oracle.render_oracle import FPS


def _body(model, poses, expression, trans, betas, n):
    """All joints posed, frame 0's trans on every frame, the first n frames: (n, V, 3) in the model's dtype."""
    dt = model.v_template.dtype
    pose = torch.as_tensor(poses[:n]).to(dt)
    expr = None if expression is None else torch.as_tensor(expression[:n]).to(dt)
    kw = dict(betas=None if betas is None else torch.as_tensor(betas).to(dt)[None].repeat(n, 1),
              transl=torch.as_tensor(trans).to(dt)[0:1].repeat(n, 1), expression=expr, jaw_pose=pose[:, 66:69],
              return_verts=True)
    return model(global_orient=pose[:, :3], body_pose=pose[:, 3:66], left_hand_pose=pose[:, 75:120],
                 right_hand_pose=pose[:, 120:165], leye_pose=pose[:, 69:72], reye_pose=pose[:, 72:75], **kw)["vertices"]


def body_vertices(model, poses, expression, trans, betas=None):
    """render_one_sequence_no_gt's vertices (fast_render.py:366-386) of the npz contents on an smplx-like model
    (oracle/smplx_oracle.py SmplxRestatement): poses (T, 165), expression (T, 100) or None (zeros), trans (T, 3), betas
    (300,) or None.  Returns (T // 30 * 30, V, 3): the body view, every frame at frame 0's trans."""
    return _body(model, poses, expression, trans, betas, poses.shape[0] // FPS * FPS)


def pair_vertices(model, pred, gt):
    """render_one_sequence's vertices (fast_render.py:326-356): pred and gt are (poses, expression, trans, betas) as in
    body_vertices.  Both sides draw n = T_pred // 30 * 30 frames, the ground truth its first n, each with its own betas,
    expression and frame-0 trans.  Returns (pred_body, gt_body), each (n, V, 3)."""
    n = pred[0].shape[0] // FPS * FPS
    if gt[0].shape[0] < n:
        raise ValueError(f"the ground truth has {gt[0].shape[0]} frames, fewer than {n}")
    return _body(model, *pred, n), _body(model, *gt, n)

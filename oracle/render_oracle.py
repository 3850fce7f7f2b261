"""CPU restatement of the SMPL-X mesh render (TEST / MEASUREMENT INFRASTRUCTURE; never imported by the product).

Restates include/pm_emage.h pm_mesh_vertex_f32 / pm_mesh_raster / pm_mesh_shade_u8, one or two views per frame, and the
scene of emage_utils/fast_render.py, which it follows line by line where cited:
  - viewport 480 x 720 per view (fast_render.py:17-24 args, :106-108 OffscreenRenderer(width, height)), the views side
    by side with the face view left (:80-92 np.hstack((fig1, fig2)), :164-176 distribute_frames, :318
    generate_silent_videos(..., vertices1_all, vertices_all, ...));
  - OrthographicCamera(xmag=1, ymag=1) at create_pose_camera(-2) (:30-36, :53-54), DirectionalLight at
    create_pose_light(-30) (:38-44, :55-56), uniform colour 220 (:59), smooth shading (:49);
  - the composition of render_one_sequence_with_face (:286-321): frame 0's trans on every frame, the face view with only
    the jaw posed, scaled x7 and moved by -(0, 10, 0), and T // 30 * 30 frames.
Assumed from pyrender, which is not available to check: znear 0.05, zfar 100, and an orthographic projection that
ignores the aspect ratio (x_ndc = x / xmag, y_ndc = y / ymag).  The shading is Lambert (shade()), not pyrender's PBR.

Vertex stage and shading in float64 (the view's affine transform in float32 first, as the kernel defines it).
Rasterisation from given snapped coordinates and fp32 depths with the kernel's int64 edge functions, fill rule, fp64
depth formula and key, so its visibility buffer equals the kernel's bit for bit.
"""
from __future__ import annotations

import numpy as np
import torch

W, H, VIEWS, FPS = 480, 720, 2, 30
SUB = 256
GUARD = 2.0 ** 20
BAD = -(2 ** 31)
XMAG = YMAG = 1.0
ZNEAR, ZFAR = np.float32(0.05), np.float32(100.0)
COLOR = 220.0
FACE_SCALE, FACE_SHIFT = 7.0, (0.0, -10.0, 0.0)
JAW = 22
EMPTY = np.uint64(0xFFFFFFFFFFFFFFFF)


def rot_x_pose(deg, ty, tz):
    """create_pose_camera / create_pose_light (fast_render.py:30-44): rotation about x, translation (0, ty, tz)."""
    a = np.deg2rad(deg)
    return np.array([[1.0, 0.0, 0.0, 0.0], [0.0, np.cos(a), -np.sin(a), ty], [0.0, np.sin(a), np.cos(a), tz],
                     [0.0, 0.0, 0.0, 1.0]])


CAMERA_POSE = rot_x_pose(-2, 1.0, 5.0)
LIGHT_POSE = rot_x_pose(-30, 0.0, 3.0)
LIGHT_DIR = LIGHT_POSE[:3, 2]          # light travels along the pose's -z axis: toward the light is +z


def incident_faces(faces, n_verts):
    """(vf_ptr, vf_face): each vertex's faces in ascending face index, each face once."""
    faces = np.asarray(faces, dtype=np.int64)
    nf = faces.shape[0]
    pairs = np.unique(faces * nf + np.arange(nf)[:, None])
    return np.searchsorted(pairs // nf, np.arange(n_verts + 1)), pairs % nf


def vertex_stage(verts, scale, offset, faces):
    """One view of one frame: verts (V, 3) float32 -> (xy (V, 2) int64 snapped or BAD, unsnapped pixel coordinates
    (V, 2) float64, depth (V,) float64, normal (V, 3) float64)."""
    p = np.asarray(verts, np.float32) * np.float32(scale) + np.asarray(offset, np.float32)     # float32, as the kernel
    p = p.astype(np.float64)
    view = p - CAMERA_POSE[:3, 3]
    view = view @ CAMERA_POSE[:3, :3]                   # R^T (p - t), row vectors
    s = np.stack([(view[:, 0] / XMAG + 1.0) * (W / 2), (1.0 - view[:, 1] / YMAG) * (H / 2)], axis=1)
    ok = (np.abs(s) <= GUARD).all(1) & np.isfinite(view[:, 2])
    xy = np.full(s.shape, BAD, dtype=np.int64)
    xy[ok] = np.rint(s[ok] * SUB).astype(np.int64)
    f = np.asarray(faces, dtype=np.int64)
    cr = np.cross(p[f[:, 1]] - p[f[:, 0]], p[f[:, 2]] - p[f[:, 0]])
    vf_ptr, vf_face = incident_faces(f, len(p))
    owner = np.repeat(np.arange(len(p)), np.diff(vf_ptr))
    n = np.zeros_like(p)
    np.add.at(n, owner, cr[vf_face])
    ln = np.linalg.norm(n, axis=1, keepdims=True)
    return xy, s, -view[:, 2], np.divide(n, ln, out=np.zeros_like(n), where=ln > 0)


def _setup(xy, faces):
    """Corner ids after the winding swap, their coordinates and area2, and which triangles are drawn."""
    f = torch.as_tensor(np.asarray(faces, dtype=np.int64))
    xy = torch.as_tensor(np.asarray(xy, dtype=np.int64))
    X, Y = xy[f, 0], xy[f, 1]
    area = (X[:, 1] - X[:, 0]) * (Y[:, 2] - Y[:, 0]) - (Y[:, 1] - Y[:, 0]) * (X[:, 2] - X[:, 0])
    ok = (X != BAD).all(1) & (area != 0)
    swap = area < 0
    perm = torch.tensor([0, 1, 2]).repeat(len(f), 1)
    perm[swap] = torch.tensor([0, 2, 1])
    ids = torch.gather(f, 1, perm)
    return ids, torch.gather(X, 1, perm), torch.gather(Y, 1, perm), area.abs(), ok


def _edges(X, Y):
    """Per edge k (corner k+1 -> k+2): dx, dy (tri, 3)."""
    p, q = [1, 2, 0], [2, 0, 1]
    return X[:, q] - X[:, p], Y[:, q] - Y[:, p], X[:, p], Y[:, p]


def raster(xy, depth, faces):
    """Visibility keys (H, W) uint64 of one view, all ones where nothing is drawn: the kernel's rules exactly, evaluated
    per triangle row as a pixel span solved from the edge inequalities (work proportional to the covered pixels)."""
    ids, X, Y, area, ok = _setup(xy, faces)
    d = torch.as_tensor(np.asarray(depth, np.float32)).double()
    half = SUB // 2
    px0 = (-((half - X.min(1).values) // SUB)).clamp(min=0)
    px1 = ((X.max(1).values - half) // SUB).clamp(max=W - 1)
    py0 = (-((half - Y.min(1).values) // SUB)).clamp(min=0)
    py1 = ((Y.max(1).values - half) // SUB).clamp(max=H - 1)
    ok &= (px0 <= px1) & (py0 <= py1)
    tri = torch.nonzero(ok)[:, 0]
    dx, dy, xp, yp = _edges(X[tri], Y[tri])
    bias = torch.where((dy < 0) | ((dy == 0) & (dx > 0)), 0, 1)
    vis = torch.full((H * W,), torch.iinfo(torch.int64).max, dtype=torch.int64)
    rows = (py1 - py0 + 1)[tri]
    # (triangle, row) pairs in blocks
    start = 0
    while start < len(tri):
        csum = torch.cumsum(rows[start:], 0)
        stop = start + max(1, int(torch.searchsorted(csum, 1 << 20, right=True)))
        sl = slice(start, stop)
        start = stop
        t = torch.repeat_interleave(torch.arange(sl.start, sl.stop), rows[sl])
        py = py0[tri[t]] + (torch.arange(len(t)) - torch.repeat_interleave(torch.cumsum(rows[sl], 0) - rows[sl], rows[sl]))
        cy = py * SUB + half
        # w_k(px) = c_k + s_k px with s_k = -256 dy; covered where s_k px >= bias_k - c_k for every k
        c = dx[t] * (cy[:, None] - yp[t]) - dy[t] * (half - xp[t])
        s = -SUB * dy[t]
        r = bias[t] - c
        lo, hi = px0[tri[t]].clone(), px1[tri[t]].clone()
        for k in range(3):
            sk, rk = s[:, k], r[:, k]
            pos, neg = sk > 0, sk < 0
            lo[pos] = torch.maximum(lo[pos], -((-rk[pos]) // sk[pos]))
            hi[neg] = torch.minimum(hi[neg], rk[neg] // sk[neg])
            hi[(sk == 0) & (rk > 0)] = -1
        n = (hi - lo + 1).clamp(min=0)
        keep = n > 0
        t, py, lo, n = t[keep], py[keep], lo[keep], n[keep]
        for a in range(0, len(t), 1 << 14):
            b = slice(a, a + (1 << 14))
            if int(n[b].sum()) == 0:
                continue
            _span_keys(vis, tri, t[b], py[b], lo[b], n[b], ids, X, Y, area, d)
    out = vis.numpy().view(np.uint64).copy()
    out[vis.numpy() == torch.iinfo(torch.int64).max] = EMPTY
    return out.reshape(H, W)


def _span_keys(vis, tri, t, py, lo, n, ids, X, Y, area, d):
    """Depth keys of the pixels of the given spans, min-reduced into vis."""
    tt = torch.repeat_interleave(t, n)
    px = torch.repeat_interleave(lo, n) + (torch.arange(len(tt)) - torch.repeat_interleave(torch.cumsum(n, 0) - n, n))
    py = torch.repeat_interleave(py, n)
    g = tri[tt]
    cx, cy = px * SUB + SUB // 2, py * SUB + SUB // 2
    Xg, Yg = X[g], Y[g]
    w0 = (Xg[:, 2] - Xg[:, 1]) * (cy - Yg[:, 1]) - (Yg[:, 2] - Yg[:, 1]) * (cx - Xg[:, 1])
    w1 = (Xg[:, 0] - Xg[:, 2]) * (cy - Yg[:, 2]) - (Yg[:, 0] - Yg[:, 2]) * (cx - Xg[:, 2])
    w2 = area[g] - w0 - w1                    # the three edge functions sum to area2 exactly
    dd = d[ids[g]]
    z = ((w0.double() * dd[:, 0] + w1.double() * dd[:, 1]) + w2.double() * dd[:, 2]) / area[g].double()
    zf = z.float()
    keep = (zf >= float(ZNEAR)) & (zf <= float(ZFAR))
    key = (zf.view(torch.int32).long() << 32) | g
    vis.scatter_reduce_(0, (py * W + px)[keep], key[keep], "amin")


def shade(n):
    """The shading rule: 220 max(0, n.l / |n|) rounded to nearest (0 where n = 0), for R, G and B alike."""
    n = np.asarray(n, np.float64)
    ln = np.linalg.norm(n, axis=-1)
    d = np.divide(n @ LIGHT_DIR, ln, out=np.zeros(n.shape[:-1]), where=ln > 0)
    return np.rint(COLOR * np.maximum(0.0, d))


def shade_view(vis, xy, normal, faces):
    """float64 shaded values (H, W) of one view from its visibility keys: barycentric weights of the visible triangle
    at the pixel centre interpolate the vertex normals.  Background is 0."""
    vis = np.asarray(vis)
    out = np.zeros(vis.shape)
    hit = vis != EMPTY
    ids, X, Y, area, _ = _setup(xy, faces)
    g = torch.as_tensor((vis[hit] & np.uint64(0xFFFFFFFF)).astype(np.int64))
    py, px = (torch.as_tensor(a) for a in np.nonzero(hit))
    cx, cy = px * SUB + SUB // 2, py * SUB + SUB // 2
    dx, dy, xp, yp = _edges(X[g], Y[g])
    w = dx * (cy[:, None] - yp) - dy * (cx[:, None] - xp)
    b = (w.double() / area[g, None].double()).numpy()
    nrm = np.asarray(normal, np.float64)[ids[g].numpy()]
    out[hit] = shade((b[:, :, None] * nrm).sum(1))
    return out


def render_views(vertices, views, faces, depth=None, xy=None):
    """One output frame (H, 2W) float64 of shaded values from per-view vertices (V, 3) and (scale, offset) views.
    xy / depth: per-view snapped coordinates and fp32 depths to rasterise instead of the oracle's own (a kernel's)."""
    cols = []
    for k, (v, (scale, off)) in enumerate(zip(vertices, views)):
        sxy, _, dep, nrm = vertex_stage(v, scale, off, faces)
        sxy = sxy if xy is None else xy[k]
        dep = np.float32(dep) if depth is None else depth[k]
        cols.append(shade_view(raster(sxy, dep, faces), sxy, nrm, faces))
    return np.concatenate(cols, axis=1)


def sequence_vertices(model, poses, expression, trans, betas=None):
    """render_one_sequence_with_face's vertices (fast_render.py:290-315) on an smplx-like model (oracle/smplx_oracle.py
    SmplxRestatement): poses (T, 165), expression (T, 100), trans (T, 3), betas (300,) or None.  Returns (face, body)
    (T // 30 * 30, V, 3): the face view with only the jaw posed, x7 and -(0, 10, 0); every frame at frame 0's trans."""
    n = poses.shape[0]
    dt = model.v_template.dtype
    pose = torch.as_tensor(poses).to(dt)
    kw = dict(betas=None if betas is None else torch.as_tensor(betas).to(dt)[None].repeat(n, 1),
              transl=torch.as_tensor(trans).to(dt)[0:1].repeat(n, 1), expression=torch.as_tensor(expression).to(dt),
              jaw_pose=pose[:, 66:69], return_verts=True)
    body = model(global_orient=pose[:, :3], body_pose=pose[:, 3:66], left_hand_pose=pose[:, 75:120],
                 right_hand_pose=pose[:, 120:165], leye_pose=pose[:, 69:72], reye_pose=pose[:, 72:75], **kw)["vertices"]
    face = model(**kw)["vertices"] * FACE_SCALE + torch.tensor(FACE_SHIFT, dtype=dt)
    m = n // FPS * FPS
    return face[:m], body[:m]

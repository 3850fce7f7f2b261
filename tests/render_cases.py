"""Shared cases of the mesh render GPU tests (tests/test_render_gpu.py, tests/test_render_layouts_gpu.py): a renderer
over a bare triangle list, the three kernels on one chunk, and the test meshes."""
import types

import numpy as np
import torch

from body_cases import random_poses
from pantomatrix_b200 import ops
from pantomatrix_b200.body_model import SmplxBodyModel
from pantomatrix_b200.render import H, W, MeshRenderer

DEV = "cuda"


def renderer(v, faces):
    return MeshRenderer(types.SimpleNamespace(n_verts=v, faces=faces, device=torch.device(DEV)))


def run_chunk(r, verts, views):
    """The three kernels on one chunk of len(verts) views: (xy, depth, normal, vis, rgb) on the host."""
    k, nv, nviews = verts[0].shape[0], r.n_verts, len(verts)
    xy = torch.empty(k, nviews, nv, 2, dtype=torch.int32, device=DEV)
    depth = torch.empty(k, nviews, nv, device=DEV)
    normal = torch.empty(k, nviews, nv, 3, device=DEV)
    vis = torch.empty(k, nviews, H, W, dtype=torch.int64, device=DEV)
    rgb = torch.empty(k, H, nviews * W, 3, dtype=torch.uint8, device=DEV)
    ops.mesh_vertex(verts, views, r.faces, r.vf_csr, xy, depth, normal)
    ops.mesh_raster(xy, depth, r.faces, vis)
    ops.mesh_shade(vis, xy, normal, r.faces, rgb)
    torch.cuda.synchronize()
    return xy.cpu().numpy(), depth.cpu().numpy(), normal.cpu().numpy(), vis.cpu().numpy().view(np.uint64), rgb.cpu().numpy()


def world(x, frames=1):
    return torch.as_tensor(np.asarray(x, np.float32), device=DEV).expand(frames, *np.shape(x)).contiguous()


def sphere(rings=24, segs=40):
    v = [(0.0, 0.0, -1.0)]
    for r in range(1, rings):
        th = np.pi * r / rings
        v += [(np.sin(th) * np.cos(p), np.sin(th) * np.sin(p), -np.cos(th)) for p in 2 * np.pi * np.arange(segs) / segs]
    v.append((0.0, 0.0, 1.0))
    ring = lambda r, s: 1 + r * segs + s % segs
    f = []
    for s in range(segs):
        f += [(0, ring(0, s + 1), ring(0, s)), (len(v) - 1, ring(rings - 2, s), ring(rings - 2, s + 1))]
        for r in range(rings - 2):
            f += [(ring(r, s), ring(r + 1, s + 1), ring(r + 1, s)), (ring(r, s), ring(r, s + 1), ring(r + 1, s + 1))]
    return np.array(v), np.array(f)


def posed(arrays, frames, seed, scale=0.3):
    rng = np.random.default_rng(seed)
    bm = SmplxBodyModel(arrays, DEV)
    poses = torch.as_tensor(random_poses(rng, frames, scale).astype(np.float32), device=DEV).view(1, frames, 165)
    trans = torch.as_tensor(rng.normal(0, 0.05, (1, frames, 3)) + (0, 1.0, 0), dtype=torch.float32, device=DEV)
    body = bm(poses, transl=trans, vertices=True)["vertices"][0]
    face = bm._vertices(poses, None, None, trans, 1 << 22)[1][0]
    return bm, face, body

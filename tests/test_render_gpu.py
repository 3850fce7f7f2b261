"""SMPL-X mesh render on the H100 against the CPU restatement (oracle/render_oracle.py): vertex stage against float64,
visibility bit for bit, shaded values within 1, determinism, CUDA graph capture and render_sequence end to end on EMAGE
generate() output."""
import numpy as np
import pytest
import torch

from body_cases import random_poses
from oracle import render_oracle as R
from oracle.smplx_oracle import SmplxRestatement
from pantomatrix_b200.body_model import SmplxBodyModel
from pantomatrix_b200.render import BODY_VIEW, FACE_VIEW, H, W, MeshRenderer
from render_cases import DEV, posed, renderer, run_chunk, sphere, world
from synthetic_models import SMPLX_FULL_VERTS, smplx_arrays, smplx_surface_arrays

pytestmark = pytest.mark.gpu
VIEWS = (FACE_VIEW, BODY_VIEW)


def _check(verts, views, faces, normal_cond=0.0):
    """Every claim of the kernels on one chunk against the oracle.  normal_cond: normals are gated only where the float64
    sum of the face normals keeps at least that fraction of the sum of their lengths (random soups cancel)."""
    r = renderer(verts[0].shape[1], faces)
    xy, depth, normal, vis, rgb = run_chunk(r, verts, views)
    f = np.asarray(faces, np.int64)
    covered = 0
    for k in range(verts[0].shape[0]):
        for view in range(2):
            v = verts[view][k].cpu().numpy()
            oxy, s, _, onrm = R.vertex_stage(v, *views[view], faces)
            ok = oxy[:, 0] != R.BAD
            near_guard = (np.abs(s) > R.GUARD - 1).any(1)
            assert np.array_equal((xy[k, view, :, 0] != R.BAD)[~near_guard], ok[~near_guard])
            assert np.abs(xy[k, view][ok] - oxy[ok]).max(initial=0) <= 1
            p = (np.float32(v) * np.float32(views[view][0]) + np.float32(views[view][1])).astype(np.float64)
            cr = np.cross(p[f[:, 1]] - p[f[:, 0]], p[f[:, 2]] - p[f[:, 0]])
            total = np.zeros(len(v))
            for c in range(3):
                np.add.at(total, f[:, c], np.linalg.norm(cr, axis=1))
            ptr, fl = R.incident_faces(f, len(v))
            summed = np.zeros_like(p)
            np.add.at(summed, np.repeat(np.arange(len(v)), np.diff(ptr)), cr[fl])
            good = np.linalg.norm(summed, axis=1) > normal_cond * total
            assert np.abs(normal[k, view][good] - onrm[good]).max(initial=0) <= 1e-5
            ovis = R.raster(xy[k, view], depth[k, view], faces)
            assert np.array_equal(vis[k, view], ovis), (k, view, int((vis[k, view] != ovis).sum()))
            img = R.shade_view(ovis, xy[k, view], onrm, faces)
            got = rgb[k, :, view * W:(view + 1) * W]
            assert (got[..., 0] == got[..., 1]).all() and (got[..., 0] == got[..., 2]).all()
            hit = ovis != R.EMPTY
            assert (got[~hit] == 0).all()
            assert np.abs(got[..., 0][hit].astype(np.float64) - img[hit]).max(initial=0) <= 1
            covered += int(hit.sum())
    return covered


def test_structured_meshes_against_the_oracle():
    rng = np.random.default_rng(0)
    v, f = sphere()
    spheres = [world(v * 0.4 + (0.1, 1.2, 0.3)), world(v * 0.6 + (0.0, 1.0, 0.0))]
    assert _check(spheres, ((1.0, (0, 0, 0)), BODY_VIEW), f) > 50000
    # a jittered grid of shared edges, and two equal-depth overlapping triangles plus an interpenetrating one
    n = 30
    gx, gy = np.meshgrid(np.linspace(-0.9, 0.9, n), np.linspace(0.1, 1.9, n))
    grid = np.stack([gx, gy, rng.normal(0, 0.05, gx.shape)], -1).reshape(-1, 3) + rng.normal(0, 2e-3, (n * n, 3))
    idx = np.arange(n * n).reshape(n, n)
    gf = np.concatenate([np.stack([idx[:-1, :-1], idx[1:, :-1], idx[1:, 1:]], -1).reshape(-1, 3),
                         np.stack([idx[:-1, :-1], idx[1:, 1:], idx[:-1, 1:]], -1).reshape(-1, 3)])
    tie = np.array([[-0.5, 0.5, 0.2], [0.5, 0.6, 0.2], [0.0, 1.5, 0.2], [-0.4, 0.4, 0.2], [0.6, 0.9, 0.2],
                    [-0.2, 1.6, 0.2], [-0.8, 0.8, -0.3], [0.8, 0.8, 0.7], [0.0, 1.2, 0.2]])
    verts = np.concatenate([grid, tie])
    faces = np.concatenate([gf, n * n + np.array([[3, 4, 5], [0, 1, 2], [6, 7, 8]])])
    assert _check([world(verts, 2), world(verts, 2)], (BODY_VIEW, (1.0, (0.01, 0.003, -0.2))), faces) > 100000


def test_depth_clipping_against_the_oracle():
    # triangles reaching behind znear (depth < 0.05: z > 4.95) and beyond zfar (depth > 100: z < -95)
    v = np.array([[-0.9, 0.2, 4.99], [0.9, 0.3, 4.9], [0.0, 1.8, 3.0], [-0.9, 1.9, -150.0], [0.9, 1.8, 0.0],
                  [0.2, 0.1, -20.0]])
    faces = np.array([[0, 1, 2], [3, 4, 5]])
    assert _check([world(v), world(v)], (BODY_VIEW, (1.0, (0.0, 0.0, 0.02))), faces) > 10000


@pytest.mark.parametrize("kind", ["surface", "soup"])
def test_full_size_models_in_both_views(kind):
    arrays = smplx_surface_arrays() if kind == "surface" else smplx_arrays(SMPLX_FULL_VERTS)
    bm, face, body = posed(arrays, 2 if kind == "surface" else 1, 5)       # the soup's oracle takes ~25 s a frame
    assert _check([face, body], VIEWS, arrays["f"], normal_cond=0.0 if kind == "surface" else 0.05) > 20000


def test_two_calls_are_identical_and_a_captured_replay_equals_the_eager_call():
    arrays = smplx_surface_arrays()
    bm = SmplxBodyModel(arrays, DEV)
    r = MeshRenderer(bm)
    rng = np.random.default_rng(7)
    poses = torch.as_tensor(random_poses(rng, 2 * 45, 0.3).astype(np.float32), device=DEV).view(2, 45, 165)
    expr = torch.as_tensor(rng.normal(0, 0.5, (2, 45, 100)), dtype=torch.float32, device=DEV)
    trans = torch.as_tensor(rng.normal(0, 0.05, (2, 45, 3)) + (0, 1.0, 0), dtype=torch.float32, device=DEV)
    a = r.render_sequence(poses, expr, trans)
    b = r.render_sequence(poses, expr, trans)
    assert a.shape == (2, 30, H, 2 * W, 3) and torch.equal(a, b)
    out = torch.zeros_like(a)
    g = torch.cuda.CUDAGraph()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        r.render_sequence(poses, expr, trans, out=out)
        with torch.cuda.graph(g, stream=s):
            r.render_sequence(poses, expr, trans, out=out)
    torch.cuda.current_stream().wait_stream(s)
    out.zero_()
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(out, a)
    poses.mul_(0.5)                                     # the graph reads the static inputs in place
    g.replay()
    want = r.render_sequence(poses, expr, trans)
    torch.cuda.synchronize()
    assert torch.equal(out, want) and not torch.equal(want, a)


def test_render_sequence_on_generate_output_end_to_end():
    from oracle.weights import synth_audio
    from pantomatrix_b200.pipeline import generate
    from synthetic_models import build_product
    model, vqm = build_product(seed=0, device=DEV)
    _, pred = generate(model, vqm, torch.from_numpy(synth_audio(2, 34000, 99)).to(DEV))
    poses, expr, trans = pred["motion_axis_angle"], pred["expression"], pred["trans"]
    t = poses.shape[1]
    assert t >= 30
    arrays = smplx_surface_arrays()
    r = MeshRenderer(SmplxBodyModel(arrays, DEV))
    seen = []
    draw = r.render
    r.render = lambda verts, views, out: seen.append([v.clone() for v in verts]) or draw(verts, views, out)
    betas = torch.as_tensor(np.random.default_rng(3).normal(0, 1, (2, 300)), dtype=torch.float32, device=DEV)
    frames = r.render_sequence(poses, expr, trans, betas).cpu().numpy()
    n = t // 30 * 30
    assert frames.shape == (2, n, H, 2 * W, 3)
    m64 = SmplxRestatement(arrays, torch.float64)
    face, body = (x.view(2, n, -1, 3).cpu() for x in seen[0])
    for b in range(2):
        want_face, want_body = R.sequence_vertices(m64, poses[b].cpu(), expr[b].cpu(), trans[b].cpu(), betas[b].cpu())
        # the body model's jaw-only vertices; the kernel applies the view's x7 and -(0, 10, 0)
        got_face = face[b].double().numpy() * FACE_VIEW[0] + np.array(FACE_VIEW[1])
        assert np.abs(got_face - want_face.numpy()).max() <= 7e-5
        assert np.abs(body[b].double().numpy() - want_body.numpy()).max() <= 1e-5
        for k in (0, n - 1):
            img = R.render_views([face[b, k].numpy(), body[b, k].numpy()], VIEWS, arrays["f"])
            diff = np.abs(frames[b, k, ..., 0].astype(np.float64) - img)
            assert (diff <= 1).mean() >= 0.995, float((diff <= 1).mean())

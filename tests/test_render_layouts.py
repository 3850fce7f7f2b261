"""The body-only and prediction-beside-ground-truth render layouts without a GPU: the CPU restatement
(oracle/render_oracle.py, oracle/render_layouts_oracle.py) against the golden made by the reference's own compositions
(tests/golden/case_render_layouts.npz), the npz writer's upsampling, and how MeshRenderer.render_body / render_pair /
single-view render compose body-model calls, views and chunks on stand-in kernels."""
import types

import numpy as np
import pytest
import torch

from oracle import render_layouts_oracle as L
from oracle import render_oracle as R
from oracle.smplx_oracle import SmplxRestatement
from pantomatrix_b200 import motion_io, render
from pantomatrix_b200.body_model import ALL_JOINTS
from synthetic_models import SMPLX_SMALL_VERTS, smplx_arrays, smplx_hash

BODY_GATE = 1e-5          # metres, as for render_sequence's body view


@pytest.fixture(scope="module")
def golden(golden_dir):
    g = dict(np.load(f"{golden_dir}/case_render_layouts.npz"))
    arrays = smplx_arrays(SMPLX_SMALL_VERTS)
    assert str(g["model_sha256"]) == smplx_hash(arrays)
    return g, SmplxRestatement(arrays, torch.float64)


def test_oracle_reproduces_the_body_only_scene(golden):
    g, model = golden
    f32 = lambda k: g[k].astype(np.float32)          # the renderer reads the npz back as float32
    body = L.body_vertices(model, f32("body_poses"), f32("body_expressions"), f32("body_trans"), f32("body_betas"))
    n = g["body_poses"].shape[0] // 30 * 30
    assert g["body_poses"].shape[0] == 2 * g["body_poses15"].shape[0]
    assert int(g["body_frames"]) == n == body.shape[0] == 60
    assert g["body_vertices"].shape[1] == 1
    assert float((body.numpy() - g["body_vertices"][:, 0]).__abs__().max()) <= BODY_GATE
    assert tuple(g["body_viewport"]) == (R.W, R.H) == (render.W, render.H)
    assert tuple(g["body_image_shape"]) == (render.H, render.W, 3)
    # the writer's zero expressions and betas equal passing none
    assert not g["body_expressions"].any() and not g["body_betas"].any()
    none = L.body_vertices(model, f32("body_poses"), None, f32("body_trans"))
    assert torch.equal(none, body)


def test_oracle_reproduces_the_paired_scene(golden):
    g, model = golden
    side = lambda tag: tuple(g[f"pair_{tag}_{k}"] for k in ("poses", "expressions", "trans", "betas"))
    pred, gt = L.pair_vertices(model, side("pred"), side("gt"))
    n = g["pair_pred_poses"].shape[0] // 30 * 30
    assert g["pair_gt_poses"].shape[0] > g["pair_pred_poses"].shape[0]
    assert int(g["pair_frames"]) == n == pred.shape[0] == gt.shape[0] == 30
    # prediction left, ground truth right
    assert float((pred.numpy() - g["pair_vertices"][:, 0]).__abs__().max()) <= BODY_GATE
    assert float((gt.numpy() - g["pair_vertices"][:, 1]).__abs__().max()) <= BODY_GATE
    assert float(np.abs(g["pair_vertices"][:, 0] - g["pair_vertices"][:, 1]).max()) > 0.1
    assert tuple(g["pair_viewport"]) == (R.W, R.H)
    assert tuple(g["pair_image_shape"]) == (render.H, render.VIEWS * render.W, 3)
    short = (g["pair_gt_poses"][:n - 1],) + side("gt")[1:]
    with pytest.raises(ValueError):
        L.pair_vertices(model, side("pred"), short)


def test_time_upsample_reproduces_the_npz_writer(golden):
    g, _ = golden
    up = motion_io.time_upsample_numpy(g["body_poses15"], 2)
    assert up.dtype == np.float64 and np.array_equal(up, g["body_poses"])
    assert np.array_equal(motion_io.time_upsample_numpy(np.zeros((37, 100), np.float32), 2), g["body_expressions"])
    assert np.array_equal(motion_io.time_upsample_numpy(g["body_trans"][::2], 2), g["body_trans"])


class _Body:
    n_verts, faces, device = 5, np.array([[0, 1, 2]]), torch.device("cpu")

    def __init__(self):
        self.calls = []

    def _poses(self, poses):
        return poses.shape[0], poses.shape[1]

    def _check(self, x, name, shape):
        if tuple(x.shape) != shape:
            raise ValueError(name)

    def _vertices(self, p, betas, e, tr, mask):
        self.calls.append(types.SimpleNamespace(p=p, betas=betas, e=e, tr=tr, mask=mask))
        return None, torch.zeros(p.shape[0], p.shape[1], 5, 3)


def _upsample_on_host(x, k, out=None):
    return torch.from_numpy(motion_io.time_upsample_numpy(x.numpy(), k).astype(np.float32))


def test_render_body_composes_the_reference_view(monkeypatch):
    body = _Body()
    r = render.MeshRenderer(body)
    drawn = []
    monkeypatch.setattr(r, "render", lambda verts, views, out: drawn.append((verts, views, out)))
    monkeypatch.setattr(render.ops, "time_upsample", _upsample_on_host)
    for t, k, expr in ((149, 2, True), (149, 2, False), (14, 2, False), (15, 2, True), (61, 1, True), (20, 3, True)):
        body.calls.clear()
        drawn.clear()
        poses, trans = torch.randn(2, t, 165), torch.randn(2, t, 3)
        e = torch.randn(2, t, 100) if expr else None
        betas = torch.randn(2, 300)
        out = r.render_body(poses, trans, e, betas, upsample=k)
        n = k * t // 30 * 30
        assert out.shape == (2, n, render.H, render.W, 3) and out.dtype == torch.uint8 and out.is_contiguous()
        if n == 0:
            assert not body.calls and not drawn
            continue
        (c,), ((verts, views, o),) = body.calls, drawn
        assert c.mask == ALL_JOINTS and c.betas is betas and c.p.shape == (2, n, 165)
        assert torch.equal(c.p, _upsample_on_host(poses, k)[:, :n] if k > 1 else poses[:, :n])
        assert (c.e is None) == (not expr)
        if expr:
            assert torch.equal(c.e, _upsample_on_host(e, k)[:, :n] if k > 1 else e[:, :n])
        assert c.tr.shape == (2, n, 3) and c.tr.stride(1) == 0 and torch.equal(c.tr[:, 0], trans[:, 0])
        assert views == render.BODY_VIEW and o.shape == (2 * n, render.H, render.W, 3)
        assert o.data_ptr() == out.data_ptr()
    assert r.render_body(torch.zeros(1, 149, 165), torch.zeros(1, 149, 3), upsample=2).shape[1] == 270
    for bad in (0, 1.5, True):
        with pytest.raises(ValueError):
            r.render_body(torch.zeros(1, 30, 165), torch.zeros(1, 30, 3), upsample=bad)
    with pytest.raises(ValueError):
        r.render_body(torch.zeros(1, 30, 165), torch.zeros(1, 29, 3))


def test_render_pair_composes_the_reference_views(monkeypatch):
    body = _Body()
    r = render.MeshRenderer(body)
    drawn = []
    monkeypatch.setattr(r, "render", lambda verts, views, out: drawn.append((verts, views, out)))
    for t, gt_t in ((67, 67), (67, 60), (45, 90), (29, 5)):
        body.calls.clear()
        drawn.clear()
        p, tr, e, b = torch.randn(2, t, 165), torch.randn(2, t, 3), torch.randn(2, t, 100), torch.randn(2, 300)
        gp, gtr, ge, gb = torch.randn(2, gt_t, 165), torch.randn(2, gt_t, 3), torch.randn(2, gt_t, 100), torch.randn(2, 300)
        out = r.render_pair(p, tr, gp, gtr, e, b, ge, gb)
        n = t // 30 * 30
        assert out.shape == (2, n, render.H, render.VIEWS * render.W, 3) and out.is_contiguous()
        if n == 0:
            assert not body.calls and not drawn
            continue
        pred, gt = body.calls
        for c, (pp, ptr, pe, pb) in ((pred, (p, tr, e, b)), (gt, (gp, gtr, ge, gb))):
            assert c.mask == ALL_JOINTS and c.betas is pb
            assert torch.equal(c.p, pp[:, :n]) and torch.equal(c.e, pe[:, :n])
            assert c.tr.shape == (2, n, 3) and c.tr.stride(1) == 0 and torch.equal(c.tr[:, 0], ptr[:, 0])
        (verts, views, o), = drawn
        assert views == (render.BODY_VIEW, render.BODY_VIEW) and o.shape == (2 * n, render.H, 2 * render.W, 3)
        assert o.data_ptr() == out.data_ptr()
    # no expressions or betas: none reach the body model
    body.calls.clear()
    r.render_pair(torch.randn(1, 30, 165), torch.randn(1, 30, 3), torch.randn(1, 30, 165), torch.randn(1, 30, 3))
    assert all(c.e is None and c.betas is None for c in body.calls)


def test_render_pair_rejects_a_short_ground_truth(monkeypatch):
    r = render.MeshRenderer(_Body())
    monkeypatch.setattr(r, "render", lambda verts, views, out: None)
    for t, gt_t in ((67, 59), (30, 29), (90, 1)):
        with pytest.raises(ValueError, match="ground truth"):
            r.render_pair(torch.zeros(1, t, 165), torch.zeros(1, t, 3), torch.zeros(1, gt_t, 165),
                          torch.zeros(1, gt_t, 3))
    with pytest.raises(ValueError):
        r.render_pair(torch.zeros(1, 30, 165), torch.zeros(1, 30, 3), torch.zeros(2, 30, 165), torch.zeros(2, 30, 3))


def test_single_view_render_chunks_every_frame_once(monkeypatch):
    chunks = []

    def vertex(verts, views, faces, csr, xy, depth, normal):
        (v,), (view,) = verts, views
        k, nv = v.shape[:2]
        assert xy.shape == (k, 1, nv, 2) and depth.shape == (k, 1, nv) and normal.shape == (k, 1, nv, 3)
        assert view == render.BODY_VIEW
        depth[:, 0, 0] = v[:, 0, 0]
        chunks.append((k, depth))

    def raster(xy, depth, faces, vis):
        assert vis.shape == (xy.shape[0], 1, render.H, render.W)

    def shade(vis, xy, normal, faces, out):
        assert out.shape[1:] == (render.H, render.W, 3) and out[0].is_contiguous()
        out[:, 0, 0, 0] = chunks[-1][1][:out.shape[0], 0, 0].to(torch.uint8)
        out[:, 1, 1, 0] += 1

    monkeypatch.setattr(render.ops, "mesh_vertex", vertex)
    monkeypatch.setattr(render.ops, "mesh_raster", raster)
    monkeypatch.setattr(render.ops, "mesh_shade", shade)
    r = render.MeshRenderer(types.SimpleNamespace(n_verts=5, faces=np.array([[0, 1, 2]]), device=torch.device("cpu")))
    for n in (1, 8, 9, 21):
        chunks.clear()
        marks = torch.arange(n, dtype=torch.float32)
        body = torch.zeros(3, n, 5, 3)[1]
        body[:, 0, 0] = marks
        out = torch.zeros(n, render.H, render.W, 3, dtype=torch.uint8)
        for views in (render.BODY_VIEW, (render.BODY_VIEW,), None):
            out.zero_()
            verts = body if views is not None else [body]
            assert r.render(verts, views, out) is out
            assert [c[0] for c in chunks[-len(range(0, n, render.CHUNK)):]] == [
                min(render.CHUNK, n - s) for s in range(0, n, render.CHUNK)]
            assert torch.equal(out[:, 0, 0, 0], marks.to(torch.uint8)) and bool((out[:, 1, 1, 0] == 1).all())
        assert r.render(body).shape == (n, render.H, render.W, 3)
    with pytest.raises(ValueError):
        r.render(body, (render.BODY_VIEW, render.BODY_VIEW))
    with pytest.raises(ValueError):
        r.render((body, body, body))
    with pytest.raises(ValueError):
        r.render(body, out=torch.zeros(n, render.H, 2 * render.W, 3, dtype=torch.uint8))

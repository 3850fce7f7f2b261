"""SMPL-X mesh render without a GPU: the CPU restatement (oracle/render_oracle.py) against the golden made by the
reference's own render composition (tests/golden/case_render.npz), the fill rule, depth ties, face validation and the
chunking of MeshRenderer on stand-in kernels."""
import types

import numpy as np
import pytest
import torch

from oracle import render_oracle as R
from oracle.smplx_oracle import SmplxRestatement
from pantomatrix_b200 import _lib, render
from pantomatrix_b200.body_model import ALL_JOINTS
from synthetic_models import SMPLX_SMALL_VERTS, smplx_arrays, smplx_hash, smplx_surface_arrays

BODY_GATE, FACE_GATE = 1e-5, 7e-5        # metres: the x7 face view scales the body model's error by 7


def test_oracle_reproduces_the_golden_scene(golden_dir):
    g = np.load(f"{golden_dir}/case_render.npz")
    arrays = smplx_arrays(SMPLX_SMALL_VERTS)
    assert str(g["model_sha256"]) == smplx_hash(arrays)
    face, body = R.sequence_vertices(SmplxRestatement(arrays, torch.float64), g["poses"], g["expressions"], g["trans"],
                                     g["betas"])
    n = g["poses"].shape[0] // 30 * 30
    assert int(g["frames"]) == n == face.shape[0] == g["vertices"].shape[0]
    assert float((face.numpy() - g["vertices"][:, 0]).__abs__().max()) <= FACE_GATE
    assert float((body.numpy() - g["vertices"][:, 1]).__abs__().max()) <= BODY_GATE
    assert np.array_equal(g["faces"], arrays["f"])
    assert bool(g["camera_poses_equal"])
    np.testing.assert_allclose(g["camera_pose"], R.CAMERA_POSE, atol=1e-15)
    np.testing.assert_allclose(g["light_pose"], R.LIGHT_POSE, atol=1e-15)
    np.testing.assert_allclose(g["light_pose"][:3, 2], (0.0, 0.5, np.sqrt(3) / 2), atol=1e-15)
    assert float(g["xmag"]) == R.XMAG and float(g["ymag"]) == R.YMAG
    assert tuple(g["viewport"]) == (R.W, R.H) == (render.W, render.H)
    assert tuple(g["merged_shape"]) == (render.H, render.VIEWS * render.W, 3)
    assert tuple(g["mesh_color"][:3]) == (R.COLOR,) * 3 and bool(g["smooth"])
    # the product's constants are the oracle's
    assert render.FACE_VIEW == (R.FACE_SCALE, R.FACE_SHIFT) and render.BODY_VIEW == (1.0, (0.0, 0.0, 0.0))
    assert render.JAW_ONLY == 1 << R.JAW and render.FPS == R.FPS


def _brute_cover(X, Y):
    """Pixels (H, W) bool covered by one triangle of snapped corners, by the header's rule, with Python integers."""
    x, y = [int(v) for v in X], [int(v) for v in Y]
    area = (x[1] - x[0]) * (y[2] - y[0]) - (y[1] - y[0]) * (x[2] - x[0])
    out = np.zeros((R.H, R.W), bool)
    if area == 0:
        return out
    if area < 0:
        x[1], x[2], y[1], y[2] = x[2], x[1], y[2], y[1]
    edges = [((x[(k + 1) % 3], y[(k + 1) % 3]), (x[(k + 2) % 3], y[(k + 2) % 3])) for k in range(3)]
    for py in range(max(0, min(y) // 256 - 1), min(R.H, max(y) // 256 + 2)):
        for px in range(max(0, min(x) // 256 - 1), min(R.W, max(x) // 256 + 2)):
            cx, cy = px * 256 + 128, py * 256 + 128
            inside = True
            for (xa, ya), (xb, yb) in edges:
                dx, dy = xb - xa, yb - ya
                w = dx * (cy - ya) - dy * (cx - xa)
                inside &= w > 0 or (w == 0 and (dy < 0 or (dy == 0 and dx > 0)))
            out[py, px] = inside
    return out


def _cover(xy, faces):
    """Coverage count per pixel and the set of triangles that cover something, one triangle at a time."""
    count = np.zeros((R.H, R.W), int)
    for f in faces:
        count += R.raster(xy, np.ones(len(xy), np.float32), f[None]) != R.EMPTY
    return count


def test_shared_edges_are_covered_exactly_once():
    rng = np.random.default_rng(0)
    for _ in range(20):
        # a quad split along a random diagonal, corners at random sub-pixel positions, some on pixel centres
        x, y = rng.integers(10, 40, 2) * 256 + 128
        xy = np.array([[x, y], [x + 3000, y + 200], [x + 2500, y + 4000], [x - 300, y + 3500]])
        xy += rng.integers(-2, 3, (4, 2)) * 128 + (rng.random((4, 2)) < 0.5) * rng.integers(-127, 128, (4, 2))
        faces = np.array([[0, 1, 2], [0, 2, 3]])
        count = _cover(xy, faces)
        assert count.max() == 1
        # the union is the quad: every pixel covered by the brute-force rule of either triangle is covered once
        union = _brute_cover(xy[[0, 1, 2], 0], xy[[0, 1, 2], 1]) | _brute_cover(xy[[0, 2, 3], 0], xy[[0, 2, 3], 1])
        assert np.array_equal(count == 1, union)


def _sphere(rings=12, segs=20):
    v = [(0.0, 0.0, -1.0)]
    for r in range(1, rings):
        th = np.pi * r / rings
        for s in range(segs):
            ph = 2 * np.pi * s / segs
            v.append((np.sin(th) * np.cos(ph), np.sin(th) * np.sin(ph), -np.cos(th)))
    v.append((0.0, 0.0, 1.0))
    ring = lambda r, s: 1 + r * segs + s % segs
    f = []
    for s in range(segs):
        f += [(0, ring(0, s + 1), ring(0, s)), (len(v) - 1, ring(rings - 2, s), ring(rings - 2, s + 1))]
        for r in range(rings - 2):
            f += [(ring(r, s), ring(r + 1, s + 1), ring(r + 1, s)), (ring(r, s), ring(r, s + 1), ring(r + 1, s + 1))]
    return np.array(v), np.array(f)


def test_closed_sphere_has_no_cracks_and_no_double_hits():
    rng = np.random.default_rng(1)
    v, f = _sphere()
    for _ in range(3):
        q, _ = np.linalg.qr(rng.normal(size=(3, 3)))
        p = v @ q.T
        xy = np.rint((p[:, :2] * 60 + rng.uniform(60, 200, 2)) * 256).astype(np.int64)
        area = lambda t: ((xy[t[1], 0] - xy[t[0], 0]) * (xy[t[2], 1] - xy[t[0], 1])
                          - (xy[t[1], 1] - xy[t[0], 1]) * (xy[t[2], 0] - xy[t[0], 0]))
        front = np.array([area(t) > 0 for t in f])
        for side in (front, ~front):
            count = _cover(xy, f[side])
            union = np.zeros_like(count, bool)
            for t in f[side]:
                union |= _brute_cover(xy[t, 0], xy[t, 1])
            assert count.max() == 1 and np.array_equal(count == 1, union)
        # each side covers the same silhouette
        assert np.array_equal(_cover(xy, f[front]), _cover(xy, f[~front]))


def test_sliver_is_hit_only_where_the_centre_is_inside():
    rng = np.random.default_rng(2)
    for _ in range(10):
        x0, y0 = rng.integers(20 * 256, 30 * 256, 2)
        xy = np.array([[x0, y0], [x0 + 256, y0 + rng.integers(-64, 64)], [x0 + rng.integers(-300, 300), y0 + 300 * 256]])
        got = R.raster(xy, np.ones(3, np.float32), np.array([[0, 1, 2]])) != R.EMPTY
        assert got.any() and np.array_equal(got, _brute_cover(xy[:, 0], xy[:, 1]))


def test_depth_ties_go_to_the_lower_triangle_id_and_nearer_wins():
    xy = np.array([[10, 10], [300, 20], [40, 500], [300, 300], [20, 40], [250, 480]]) * 256 + 128
    faces = np.array([[3, 4, 5], [0, 1, 2]])
    flat = R.raster(xy, np.full(6, 2.0, np.float32), faces)
    both = (R.raster(xy, np.ones(6, np.float32), faces[:1]) != R.EMPTY) & (
        R.raster(xy, np.ones(6, np.float32), faces[1:]) != R.EMPTY)
    assert both.sum() > 100
    assert ((flat[both] & np.uint64(0xFFFFFFFF)) == 0).all()
    # interpenetrating: triangle 1 rises in depth with x, triangle 0 is flat at 2: each wins where it is nearer
    d = np.array([1.0, 3.0, 1.0, 2.0, 2.0, 2.0], np.float32)
    vis = R.raster(xy, d, faces)
    ids = (vis & np.uint64(0xFFFFFFFF)).astype(np.int64)
    z = (vis >> np.uint64(32)).astype(np.uint32).view(np.float32)
    assert set(np.unique(ids[both])) == {0, 1}
    assert (z[both] <= 2.0).all()


def test_znear_and_zfar_clip_pixels():
    xy = np.array([[0, 0], [480, 0], [0, 720]]) * 256
    for d, want in (((0.01, 0.01, 0.01), False), ((150.0, 150.0, 150.0), False), ((0.05, 0.05, 0.05), True),
                    ((100.0, 100.0, 100.0), True)):
        vis = R.raster(xy, np.array(d, np.float32), np.array([[0, 1, 2]]))
        assert (vis != R.EMPTY).any() == want, d


def test_surface_model_is_closed_and_wound_outward():
    a = smplx_surface_arrays(1100)
    v, f = a["v_template"], a["f"].astype(np.int64)
    assert v.shape == (1100, 3) and a["J_regressor"].shape == (55, 1100) and a["weights"].shape == (1100, 55)
    np.testing.assert_allclose(a["weights"].sum(1), 1.0)
    edges = {tuple(e) for e in np.concatenate([f[:, [0, 1]], f[:, [1, 2]], f[:, [2, 0]]])}
    assert len(edges) == 3 * len(f) and all((b, c) in edges for c, b in edges)        # closed, consistently wound
    assert np.einsum("ij,ij->i", v[f[:, 0]], np.cross(v[f[:, 1]], v[f[:, 2]])).sum() > 0   # outward


def _fake_body(faces, n_verts=50):
    return types.SimpleNamespace(n_verts=n_verts, faces=faces, device=torch.device("cpu"))


@pytest.mark.parametrize("faces", [None, np.zeros((4, 4), np.int32), np.zeros((0, 3), np.int32),
                                   np.zeros((4, 3), np.float32), np.full((4, 3), 50), np.full((4, 3), -1),
                                   np.zeros(12, np.int32)])
def test_renderer_rejects_malformed_faces(faces):
    with pytest.raises(ValueError):
        render.MeshRenderer(_fake_body(faces))


def test_renderer_builds_the_incidence_in_ascending_face_order():
    faces = np.array([[0, 1, 2], [2, 1, 3], [3, 3, 0], [4, 0, 2]])
    r = render.MeshRenderer(_fake_body(faces, 6))
    vf_ptr, vf_face = (x.numpy() for x in r.vf_csr)
    want = R.incident_faces(faces, 6)
    assert np.array_equal(vf_ptr, want[0]) and np.array_equal(vf_face, want[1])
    assert list(vf_face[vf_ptr[3]:vf_ptr[4]]) == [1, 2] and vf_ptr[5] == vf_ptr[6]


class _FakeOps:
    """Stand-in kernels: mesh_vertex copies each view's frame marker (vertex 0's x) into depth, mesh_shade writes the
    markers into pixels (0, 0) and (0, 1) of its frames and counts each frame's visits in pixel (1, 1)."""

    def __init__(self):
        self.chunks = []

    def mesh_vertex(self, verts, views, faces, csr, xy, depth, normal):
        k, nv = verts[0].shape[:2]
        assert xy.shape == (k, 2, nv, 2) and depth.shape == (k, 2, nv) and normal.shape == (k, 2, nv, 3)
        assert views == (render.FACE_VIEW, render.BODY_VIEW)
        depth[:, 0, 0], depth[:, 1, 0] = verts[0][:, 0, 0], verts[1][:, 0, 0]
        self.chunks.append(k)

    def mesh_raster(self, xy, depth, faces, vis):
        assert vis.shape == (xy.shape[0], 2, render.H, render.W) and vis.dtype == torch.int64

    def mesh_shade(self, vis, xy, normal, faces, out):
        assert out.shape[1:] == (render.H, 2 * render.W, 3) and out[0].is_contiguous()
        d = self.depth[:out.shape[0]]
        out[:, 0, 0, 0], out[:, 0, 1, 0] = d[:, 0, 0].to(torch.uint8), d[:, 1, 0].to(torch.uint8)
        out[:, 1, 1, 0] += 1


def test_chunking_covers_every_frame_once(monkeypatch):
    fake = _FakeOps()

    def vertex(verts, views, faces, csr, xy, depth, normal):
        fake.mesh_vertex(verts, views, faces, csr, xy, depth, normal)
        fake.depth = depth

    monkeypatch.setattr(render.ops, "mesh_vertex", vertex)
    monkeypatch.setattr(render.ops, "mesh_raster", fake.mesh_raster)
    monkeypatch.setattr(render.ops, "mesh_shade", fake.mesh_shade)
    r = render.MeshRenderer(_fake_body(np.array([[0, 1, 2]]), 5))
    for n in (1, 8, 9, 21):
        fake.chunks.clear()
        marks = torch.arange(n, dtype=torch.float32)
        body = torch.zeros(3, n, 5, 3)[1]
        body[:, 0, 0] = marks
        face = torch.zeros(n, 8, 3)[:, :5].unflatten(1, (5, 1)).squeeze(2)       # frames 24 floats apart
        face[:, 0, 0] = 100 + marks
        out = torch.zeros(n, render.H, 2 * render.W, 3, dtype=torch.uint8)
        assert r.render((face, body), out=out) is out
        assert fake.chunks == [min(render.CHUNK, n - s) for s in range(0, n, render.CHUNK)]
        assert torch.equal(out[:, 0, 0, 0], (100 + marks).to(torch.uint8))
        assert torch.equal(out[:, 0, 1, 0], marks.to(torch.uint8))
        assert bool((out[:, 1, 1, 0] == 1).all())
        assert r.render((face, body)).shape == (n, render.H, 2 * render.W, 3)


def test_render_sequence_poses_and_draws_the_face_view_then_the_body_view(monkeypatch):
    calls = []

    class Body:
        n_verts, faces, device = 5, np.array([[0, 1, 2]]), torch.device("cpu")

        def _poses(self, poses):
            return poses.shape[0], poses.shape[1]

        def _check(self, x, name, shape):
            assert tuple(x.shape) == shape, name

        def _vertices(self, p, betas, e, tr, mask):
            calls.append((tuple(p.shape), tuple(e.shape), tr.stride(1), torch.equal(tr[:, -1], tr[:, 0]), mask))
            return None, torch.zeros(p.shape[0], p.shape[1], 5, 3)

    r = render.MeshRenderer(Body())
    drawn = []
    monkeypatch.setattr(r, "render", lambda verts, views, out: drawn.append((verts, views, out)))
    for t in (29, 30, 67):
        calls.clear()
        drawn.clear()
        trans = torch.randn(2, t, 3)
        out = r.render_sequence(torch.zeros(2, t, 165), torch.zeros(2, t, 100), trans, torch.zeros(2, 300))
        n = t // 30 * 30
        assert out.shape == (2, n, render.H, 2 * render.W, 3) and out.dtype == torch.uint8 and out.is_contiguous()
        if n == 0:
            assert not calls and not drawn
            continue
        assert [c[4] for c in calls] == [1 << 22, ALL_JOINTS]          # in view order: face left, body right
        assert all(c[:4] == ((2, n, 165), (2, n, 100), 0, True) for c in calls)
        (verts, views, o), = drawn
        assert views == (render.FACE_VIEW, render.BODY_VIEW) and o.shape == (2 * n, render.H, 2 * render.W, 3)
        assert o.data_ptr() == out.data_ptr()


def test_render_refuses_cpu_tensors():
    r = render.MeshRenderer(_fake_body(np.array([[0, 1, 2]]), 5))
    v = torch.zeros(2, 5, 3)
    with pytest.raises(_lib.PmError):
        r.render((v, v))
    with pytest.raises(ValueError):
        r.render((v, torch.zeros(2, 6, 3)))

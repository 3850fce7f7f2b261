"""Single-view mesh render, frame-rate upsampling and the body-only / prediction-beside-ground-truth layouts on the H100,
against the CPU restatement (oracle/render_oracle.py, oracle/render_layouts_oracle.py) and the npz writer
(motion_io.time_upsample_numpy): upsampling bit for bit, single-view chunks under the same gates as the two-view ones,
a one-view chunk bit for bit the right half of the two-view one, both layouts on the golden inputs and on CaMN, DisCo
and EMAGE output, and CUDA graph capture."""
import numpy as np
import pytest
import torch

from body_cases import random_poses
from oracle import render_layouts_oracle as L
from oracle import render_oracle as R
from oracle.smplx_oracle import SmplxRestatement
from pantomatrix_b200 import motion_io, ops
from pantomatrix_b200.body_model import SmplxBodyModel
from pantomatrix_b200.render import BODY_VIEW, FACE_VIEW, H, W, MeshRenderer
from render_cases import DEV, posed, renderer, run_chunk, sphere, world
from synthetic_models import SMPLX_FULL_VERTS, SMPLX_SMALL_VERTS, smplx_arrays, smplx_surface_arrays

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("t", [1, 2, 3, 37, 149])
@pytest.mark.parametrize("k", [1, 2, 3])
def test_time_upsample_is_bit_identical_to_the_npz_writer(t, k):
    rng = np.random.default_rng(t * 10 + k)
    # values across magnitudes and signs, read through clip and frame strides with a dense last dimension
    base = rng.normal(0, 1, (3, 2 * t, 170)) * 10.0 ** rng.uniform(-4, 3, (3, 2 * t, 170))
    x = torch.as_tensor(base.astype(np.float32), device=DEV)[:, ::2, 3:168]
    assert x.stride(1) == 340 and x.stride(-1) == 1
    got = ops.time_upsample(x, k)
    want = np.float32(motion_io.time_upsample_numpy(x.cpu().numpy(), k))
    assert got.shape == (3, k * t, 165) and got.is_contiguous()
    assert np.array_equal(got.cpu().numpy().view(np.uint32), want.view(np.uint32))


def _check_single(verts, view, faces, normal_cond=0.0):
    """One view per frame against the oracle: snapped coordinates within 1, normals, visibility bit for bit, RGB within
    1 on covered pixels and 0 elsewhere.  Returns the number of covered pixels."""
    r = renderer(verts.shape[1], faces)
    xy, depth, normal, vis, rgb = run_chunk(r, [verts], [view])
    assert rgb.shape[2] == W
    f = np.asarray(faces, np.int64)
    covered = 0
    for k in range(verts.shape[0]):
        v = verts[k].cpu().numpy()
        oxy, s, _, onrm = R.vertex_stage(v, *view, faces)
        ok = oxy[:, 0] != R.BAD
        near_guard = (np.abs(s) > R.GUARD - 1).any(1)
        assert np.array_equal((xy[k, 0, :, 0] != R.BAD)[~near_guard], ok[~near_guard])
        assert np.abs(xy[k, 0][ok] - oxy[ok]).max(initial=0) <= 1
        p = (np.float32(v) * np.float32(view[0]) + np.float32(view[1])).astype(np.float64)
        cr = np.cross(p[f[:, 1]] - p[f[:, 0]], p[f[:, 2]] - p[f[:, 0]])
        total = np.zeros(len(v))
        for c in range(3):
            np.add.at(total, f[:, c], np.linalg.norm(cr, axis=1))
        ptr, fl = R.incident_faces(f, len(v))
        summed = np.zeros_like(p)
        np.add.at(summed, np.repeat(np.arange(len(v)), np.diff(ptr)), cr[fl])
        good = np.linalg.norm(summed, axis=1) > normal_cond * total
        assert np.abs(normal[k, 0][good] - onrm[good]).max(initial=0) <= 1e-5
        ovis = R.raster(xy[k, 0], depth[k, 0], faces)
        assert np.array_equal(vis[k, 0], ovis), (k, int((vis[k, 0] != ovis).sum()))
        img = R.shade_view(ovis, xy[k, 0], onrm, faces)
        got = rgb[k]
        assert (got[..., 0] == got[..., 1]).all() and (got[..., 0] == got[..., 2]).all()
        hit = ovis != R.EMPTY
        assert (got[~hit] == 0).all()
        assert np.abs(got[..., 0][hit].astype(np.float64) - img[hit]).max(initial=0) <= 1
        covered += int(hit.sum())
    return covered


def test_single_view_structured_meshes_against_the_oracle():
    rng = np.random.default_rng(0)
    v, f = sphere()
    assert _check_single(world(v * 0.6 + (0.0, 1.0, 0.0), 2), BODY_VIEW, f) > 2 * 50000
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
    assert _check_single(world(verts, 3), (1.0, (0.01, 0.003, -0.2)), faces) > 3 * 100000
    # depth clipping: triangles reaching behind znear and beyond zfar
    v = np.array([[-0.9, 0.2, 4.99], [0.9, 0.3, 4.9], [0.0, 1.8, 3.0], [-0.9, 1.9, -150.0], [0.9, 1.8, 0.0],
                  [0.2, 0.1, -20.0]])
    assert _check_single(world(v), (1.0, (0.0, 0.0, 0.02)), np.array([[0, 1, 2], [3, 4, 5]])) > 10000


@pytest.mark.parametrize("kind", ["surface", "soup"])
def test_single_view_full_size_models(kind):
    arrays = smplx_surface_arrays() if kind == "surface" else smplx_arrays(SMPLX_FULL_VERTS)
    _, _, body = posed(arrays, 2 if kind == "surface" else 1, 6)
    assert _check_single(body, BODY_VIEW, arrays["f"], normal_cond=0.0 if kind == "surface" else 0.05) > 20000


def test_one_view_draws_the_right_half_of_two_views_bit_for_bit():
    arrays = smplx_surface_arrays()
    _, face, body = posed(arrays, 11, 8)
    r = renderer(face.shape[1], arrays["f"])
    for views in ((FACE_VIEW, BODY_VIEW), (BODY_VIEW, (1.0, (0.1, -0.05, 0.2)))):
        two = run_chunk(r, [face, body], views)
        one = run_chunk(r, [body], views[1:])
        for a, b in zip(two[:4], one[:4]):
            assert np.array_equal(a[:, 1:], b)
        assert np.array_equal(two[4][:, :, W:], one[4])
        assert (two[4] > 0).mean() > 0.05


def _spy(r):
    """Records the vertex tensors each render() call draws."""
    seen, draw = [], r.render
    r.render = lambda verts, views, out: seen.append(
        ([v.clone() for v in verts] if isinstance(verts, (list, tuple)) else [verts.clone()], views)) or draw(verts, views, out)
    return seen


def _images_agree(frames, verts, views, faces):
    img = R.render_views(verts, views, faces)
    diff = np.abs(frames[..., 0].astype(np.float64) - img)
    assert (diff <= 1).mean() >= 0.995, float((diff <= 1).mean())


def test_both_layouts_on_the_golden_inputs(golden_dir):
    g = np.load(f"{golden_dir}/case_render_layouts.npz")
    arrays = smplx_arrays(SMPLX_SMALL_VERTS)
    r = MeshRenderer(SmplxBodyModel(arrays, DEV))
    m64 = SmplxRestatement(arrays, torch.float64)
    cuda = lambda a: torch.as_tensor(np.asarray(a, np.float32), device=DEV)[None]
    seen = _spy(r)
    # body only: the 15 fps poses, upsampled on the GPU as the writer upsampled them
    p15 = cuda(g["body_poses15"])
    assert torch.equal(ops.time_upsample(p15, 2)[0].cpu(), torch.from_numpy(g["body_poses"].astype(np.float32)))
    frames = r.render_body(p15, cuda(g["body_trans"][:37]), upsample=2).cpu().numpy()
    n = int(g["body_frames"])
    assert frames.shape == (1, n, H, W, 3) and tuple(frames.shape[2:]) == tuple(g["body_image_shape"])
    (got,), views = seen[0]
    assert views == BODY_VIEW
    want = L.body_vertices(m64, g["body_poses"].astype(np.float32), None, g["body_trans"].astype(np.float32))
    got = got.view(n, -1, 3).cpu()
    assert np.abs(got.double().numpy() - want.numpy()).max() <= 1e-5
    assert np.abs(got.numpy() - g["body_vertices"][:, 0]).max() <= 2e-5
    for k in (0, n - 1):
        _images_agree(frames[0, k], [got[k].numpy()], [BODY_VIEW], arrays["f"])
    # prediction beside a longer ground truth
    side = lambda tag: [cuda(g[f"pair_{tag}_{k}"]) for k in ("poses", "trans", "expressions")] + [
        torch.as_tensor(g[f"pair_{tag}_betas"], device=DEV)[None]]
    (p, tr, e, b), (gp, gtr, ge, gb) = side("pred"), side("gt")
    frames = r.render_pair(p, tr, gp, gtr, e, b, ge, gb).cpu().numpy()
    n = int(g["pair_frames"])
    assert frames.shape == (1, n, H, 2 * W, 3) and tuple(frames.shape[2:]) == tuple(g["pair_image_shape"])
    (lv, rv), views = seen[1]
    assert views == (BODY_VIEW, BODY_VIEW)
    lv, rv = lv.view(n, -1, 3).cpu(), rv.view(n, -1, 3).cpu()
    want = L.pair_vertices(m64, *[tuple(g[f"pair_{t}_{k}"] for k in ("poses", "expressions", "trans", "betas"))
                                  for t in ("pred", "gt")])
    for got, w, gold in ((lv, want[0], g["pair_vertices"][:, 0]), (rv, want[1], g["pair_vertices"][:, 1])):
        assert np.abs(got.double().numpy() - w.numpy()).max() <= 1e-5
        assert np.abs(got.numpy() - gold).max() <= 2e-5
    for k in (0, n - 1):
        _images_agree(frames[0, k], [lv[k].numpy(), rv[k].numpy()], [BODY_VIEW, BODY_VIEW], arrays["f"])


@pytest.mark.parametrize("kind", ["camn", "disco"])
def test_render_body_on_lstm_output_end_to_end(kind):
    from oracle.weights import synth_audio
    from synthetic_models import build_lstm_product
    model = build_lstm_product(kind, device=DEV)
    assert model.cfg.pose_fps == 15
    audio = torch.from_numpy(synth_audio(2, 48000, 21)).to(DEV)
    poses = model(audio, torch.zeros(2, 1, dtype=torch.long, device=DEV), seed_frames=4)["motion_axis_angle"]
    poses = poses.reshape(2, poses.shape[1], 165)
    t = poses.shape[1]
    arrays = smplx_surface_arrays()
    bm = SmplxBodyModel(arrays, DEV)
    pelvis = torch.as_tensor(motion_io.pelvis_translation(bm, np.zeros(300, np.float32)), device=DEV)
    trans = pelvis.expand(2, t, 3)
    r = MeshRenderer(bm)
    seen = _spy(r)
    frames = r.render_body(poses, trans, upsample=2).cpu().numpy()
    n = 2 * t // 30 * 30
    assert n >= 30 and frames.shape == (2, n, H, W, 3)
    body = seen[0][0][0].view(2, n, -1, 3).cpu()
    m64 = SmplxRestatement(arrays, torch.float64)
    for b in range(2):
        up = np.float32(motion_io.time_upsample_numpy(poses[b].cpu().numpy(), 2))
        want = L.body_vertices(m64, up, None, trans[b].cpu().numpy())
        assert np.abs(body[b].double().numpy() - want.numpy()).max() <= 1e-5
        for k in (0, n - 1):
            _images_agree(frames[b, k], [body[b, k].numpy()], [BODY_VIEW], arrays["f"])


def test_render_pair_on_generate_output_end_to_end():
    from oracle.weights import synth_audio
    from pantomatrix_b200.pipeline import generate
    from synthetic_models import build_product
    model, vqm = build_product(seed=0, device=DEV)
    _, pred = generate(model, vqm, torch.from_numpy(synth_audio(2, 34000, 99)).to(DEV))
    _, gt = generate(model, vqm, torch.from_numpy(synth_audio(2, 40000, 98)).to(DEV))
    keys = ("motion_axis_angle", "trans", "expression")
    (p, tr, e), (gp, gtr, ge) = ([x[k] for k in keys] for x in (pred, gt))
    t, n = p.shape[1], p.shape[1] // 30 * 30
    assert n >= 30 and gp.shape[1] > t
    rng = np.random.default_rng(4)
    b, gb = (torch.as_tensor(rng.normal(0, 1, (2, 300)), dtype=torch.float32, device=DEV) for _ in range(2))
    arrays = smplx_surface_arrays()
    r = MeshRenderer(SmplxBodyModel(arrays, DEV))
    seen = _spy(r)
    frames = r.render_pair(p, tr, gp, gtr, e, b, ge, gb).cpu().numpy()
    assert frames.shape == (2, n, H, 2 * W, 3)
    lv, rv = (x.view(2, n, -1, 3).cpu() for x in seen[0][0])
    m64 = SmplxRestatement(arrays, torch.float64)
    for c in range(2):
        side = lambda x, y, z, w: (x[c].cpu().numpy(), z[c].cpu().numpy(), y[c].cpu().numpy(), w[c].cpu().numpy())
        want = L.pair_vertices(m64, side(p, tr, e, b), side(gp, gtr, ge, gb))
        assert np.abs(lv[c].double().numpy() - want[0].numpy()).max() <= 1e-5
        assert np.abs(rv[c].double().numpy() - want[1].numpy()).max() <= 1e-5
        for k in (0, n - 1):
            _images_agree(frames[c, k], [lv[c, k].numpy(), rv[c, k].numpy()], [BODY_VIEW, BODY_VIEW], arrays["f"])


def _capture_matches_eager(call, inputs):
    a, b = call(None), call(None)
    torch.cuda.synchronize()
    assert torch.equal(a, b) and bool((a > 0).any())
    out = torch.zeros_like(a)
    g = torch.cuda.CUDAGraph()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        call(out)
        with torch.cuda.graph(g, stream=s):
            call(out)
    torch.cuda.current_stream().wait_stream(s)
    out.zero_()
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(out, a)
    for x in inputs:                                    # the graph reads the static inputs in place
        x.mul_(0.5)
    g.replay()
    want = call(None)
    torch.cuda.synchronize()
    assert torch.equal(out, want) and not torch.equal(want, a)


def test_both_layouts_are_deterministic_and_capturable():
    arrays = smplx_surface_arrays()
    r = MeshRenderer(SmplxBodyModel(arrays, DEV))
    rng = np.random.default_rng(9)
    cuda = lambda a: torch.as_tensor(np.asarray(a), dtype=torch.float32, device=DEV)
    poses = cuda(random_poses(rng, 2 * 31, 0.3)).view(2, 31, 165)        # 62 frames upsampled, 60 drawn; 30 paired
    expr = cuda(rng.normal(0, 0.5, (2, 31, 100)))
    trans = cuda(rng.normal(0, 0.05, (2, 31, 3)) + (0, 1.0, 0))
    betas = cuda(rng.normal(0, 1, (2, 300)))
    _capture_matches_eager(lambda out: r.render_body(poses, trans, expr, betas, upsample=2, out=out), [poses])
    gp = cuda(random_poses(rng, 2 * 40, 0.3)).view(2, 40, 165)
    ge = cuda(rng.normal(0, 0.5, (2, 40, 100)))
    gtr = cuda(rng.normal(0, 0.05, (2, 40, 3)) + (0, 1.0, 0))
    _capture_matches_eager(lambda out: r.render_pair(poses, trans, gp, gtr, expr, betas, ge, None, out=out), [poses, gp])

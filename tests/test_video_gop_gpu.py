"""H.264 GOP encoding on the H100 (pantomatrix_b200/video.py, gop > 1): the samples are byte for byte the CPU
restatement's (tests/h264_ref.py) on the CPU cases, every qp, random clips and rendered EMAGE and CaMN GOPs at qp 0,
20 and 51; each GOP encodes as it does alone at the same parity in (B, T, ...) and (N, ...) batches; calls are
deterministic and capture in a CUDA graph; pm_h264_encode_gop at gop 1 is pm_h264_encode; a 300-frame gop 30
write_mp4 file decodes to the restatement's reconstruction; bad gop values raise ValueError."""
import numpy as np
import pytest
import torch

import h264_ref as R
from oracle.weights import synth_audio
from pantomatrix_b200 import _lib, ops, video
from pantomatrix_b200.body_model import SmplxBodyModel
from pantomatrix_b200.pipeline import generate
from pantomatrix_b200.render import MeshRenderer
from synthetic_models import build_lstm_product, build_product, smplx_surface_arrays
from test_video import decode
from test_video_gop import GOPS, gop_cases, gop_of

pytestmark = pytest.mark.gpu
DEV = "cuda"


def samples(frames, qp=20, gop=1):
    data, nbytes = video.encode(frames, qp=qp, gop=gop)
    data, nbytes = data.cpu().numpy(), nbytes.cpu().numpy()
    assert all(not data[i, k:].any() for i, k in enumerate(nbytes))
    return [data[i, :k].tobytes() for i, k in enumerate(nbytes)]


@pytest.fixture(scope="module")
def rendered_gop():
    """The first 10 frames of an EMAGE render_sequence clip (960 x 720) and of two CaMN render_body(upsample=2) clips
    (480 x 720), on the full-size synthetic surface model."""
    model, vqm = build_product(seed=0, device=DEV)
    _, pred = generate(model, vqm, torch.from_numpy(synth_audio(1, 160000, 5)).to(DEV))
    r = MeshRenderer(SmplxBodyModel(smplx_surface_arrays(), DEV))
    emage = r.render_sequence(pred["motion_axis_angle"], pred["expression"], pred["trans"])
    camn = build_lstm_product("camn", device=DEV)
    poses = camn(torch.from_numpy(synth_audio(2, 160000, 6)).to(DEV),
                 torch.zeros(2, 1, dtype=torch.long, device=DEV))["motion_axis_angle"]
    poses = poses.reshape(2, poses.shape[1], 165)[:, :15]           # upsample 2 draws whole seconds: 30 frames
    body = r.render_body(poses, torch.zeros(2, 15, 3, device=DEV), upsample=2)[:, :10].contiguous()
    torch.cuda.synchronize()
    assert emage.shape == (1, 300, 720, 960, 3) and body.shape == (2, 10, 720, 480, 3)
    return emage, body


@pytest.mark.parametrize("g", GOPS, ids=[str(g) for g in GOPS])
@pytest.mark.parametrize("name,frames,qp", gop_cases(), ids=[c[0] for c in gop_cases()])
def test_gop_cases_are_byte_identical_to_the_restatement(name, frames, qp, g):
    gop = gop_of(g, len(frames))
    got = samples(torch.as_tensor(np.stack(frames), device=DEV), qp, gop)
    assert got == [e[0] for e in R.encode_clip(frames, qp, gop)]


def test_every_qp_is_byte_identical_to_the_restatement():
    rng = np.random.default_rng(5)
    a = rng.integers(0, 256, (32, 48, 3), dtype=np.uint8)
    a[16:] = a[16:] // 32 * 32
    b = a.copy()
    b[4:20, 6:30] = np.clip(b[4:20, 6:30].astype(int) + rng.integers(-12, 13, (16, 24, 3)), 0, 255)
    t = torch.as_tensor(np.stack([a, b]), device=DEV)
    for qp in range(52):
        assert samples(t, qp, 2) == [e[0] for e in R.encode_clip([a, b], qp, 2)], qp


def test_random_clips_are_byte_identical_to_the_restatement():
    rng = np.random.default_rng(11)
    for h, w in ((16, 32), (48, 64), (96, 160)):
        base = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
        clip = [base]
        for t in range(1, 6):
            f = clip[-1].copy()
            y, x = rng.integers(0, h - 8), rng.integers(0, w - 8)
            f[y:y + 8, x:x + 8] = rng.integers(0, 256, (8, 8, 3))
            if t == 3:
                f = np.clip(f.astype(int) + rng.integers(-5, 6, f.shape), 0, 255).astype(np.uint8)
            clip.append(f)
        for qp, gop in ((0, 3), (12, 4), (30, 6), (45, 2)):
            got = samples(torch.as_tensor(np.stack(clip), device=DEV), qp, gop)
            want = R.encode_clip(clip, qp, gop)
            for i, (b, e) in enumerate(zip(got, want)):
                assert b == e[0], (h, w, qp, gop, i)
                assert len(b) <= video.max_bytes(h, w, gop)


@pytest.mark.parametrize("qp", [0, 20, 51])
def test_rendered_gops_are_byte_identical_to_the_restatement(rendered_gop, qp):
    emage, body = rendered_gop
    for clip, gop in ((emage[0, :10], 5), (body[1], 10)):
        got = samples(clip, qp, gop)
        assert got == [e[0] for e in R.encode_clip(list(clip.cpu().numpy()), qp, gop)], qp


def test_batch_encodes_each_gop_as_alone_at_the_same_parity(rendered_gop):
    _, body = rendered_gop
    clips = body[:, :9].contiguous()                     # (2, 9, ...): GOPs t = 0..3, 4..7, 8 at gop 4
    both = samples(clips, 20, 4)
    for b in range(2):
        for t0 in (0, 4, 8):
            t1 = min(t0 + 4, 9)
            alone = samples(clips[b, t0:t1], 20, 4)
            if (t0 // 4) % 2:                            # parity 1: the GOP after a GOP of the same frames
                alone = samples(torch.cat([clips[b, t0:t1], clips[b, t0:t1]]), 20, t1 - t0)[t1 - t0:]
            assert alone == both[9 * b + t0:9 * b + t1], (b, t0)
    # (N, ...) input is one clip: the same bytes as its (1, N, ...) view
    assert samples(clips[0], 20, 4) == samples(clips[:1], 20, 4) == both[:9]


def test_deterministic_and_captured_replay_equals_eager(rendered_gop):
    emage, _ = rendered_gop
    frames = emage[0, :10]
    a, na = video.encode(frames, gop=4)
    b, nb = video.encode(frames, gop=4)
    assert torch.equal(a, b) and torch.equal(na, nb)
    out = (torch.full_like(a, 0xAB), torch.zeros_like(na))
    video.encode(frames, out=out, gop=4)
    torch.cuda.synchronize()
    out[0].fill_(0xCD)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        video.encode(frames, out=out, gop=4)
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(out[0], a) and torch.equal(out[1], na)


def test_encode_gop_at_gop_1_is_encode(rendered_gop):
    _, body = rendered_gop
    frames = body.reshape(-1, 720, 480, 3)
    n, h, w, _ = frames.shape
    sc = video.slice_bytes(w)
    res = []
    for name in ("pm_h264_encode", "pm_h264_encode_gop"):
        scratch = torch.zeros(n, h // 16, sc, dtype=torch.uint8, device=DEV)
        sizes = torch.zeros(n, h // 16, dtype=torch.int32, device=DEV)
        args = [frames.data_ptr(), 3 * h * w, n, 10, h, w, 20, scratch.data_ptr(), sc, sizes.data_ptr()]
        if name == "pm_h264_encode_gop":
            args += [1, 0, 0]
        _lib.call(name, *args, ops._stream())
        torch.cuda.synchronize()
        res.append((scratch, sizes))
    assert torch.equal(res[0][0], res[1][0]) and torch.equal(res[0][1], res[1][1])


def test_write_mp4_gop_30_of_a_300_frame_render_decodes_to_the_reconstruction(rendered_gop, tmp_path):
    emage, _ = rendered_gop
    path = video.write_mp4(emage[0], str(tmp_path / "clip.mp4"), fps=30, gop=30)
    lumas, _, fps = decode(path)
    assert len(lumas) == 300 and fps == 30
    host = emage[0].cpu().numpy()
    for t0 in (0, 270):
        for i, e in enumerate(R.encode_clip(list(host[t0:t0 + 3]), 20, 30)):
            assert np.array_equal(lumas[t0 + i].reshape(-1)[:720 * 960].reshape(720, 960), e[1][0]), t0 + i


def test_gop_past_the_clip_length_gives_the_gop_t_samples(rendered_gop, tmp_path):
    """gop = T + 1, 2^31 - 1 (past a 32-bit T + gop - 1) and 2^32 + 2 (a C int would read 2) give the gop = T bytes,
    in batches and in a write_mp4 file."""
    _, body = rendered_gop
    want = samples(body, 20, 10)
    for gop in (11, 2 ** 31 - 1, 2 ** 32 + 2):
        assert samples(body, 20, gop) == want, gop
    one = video.write_mp4(body[0], str(tmp_path / "t.mp4"), gop=10)
    big = video.write_mp4(body[0], str(tmp_path / "big.mp4"), gop=2 ** 32 + 2)
    assert open(one, "rb").read() == open(big, "rb").read()


def test_bad_gop_raises_value_error(tmp_path):
    f = torch.zeros(2, 16, 32, 3, dtype=torch.uint8, device=DEV)
    for gop in (0, -3, 2.0, True, None):
        with pytest.raises(ValueError):
            video.encode(f, gop=gop)
        with pytest.raises(ValueError):
            video.write_mp4(f, str(tmp_path / "x.mp4"), gop=gop)
    cap = (video.max_bytes(16, 960, 2) - 1) // 4 * 4     # a multiple of 4 short of the gop 2 bound
    assert cap >= video.slot_bytes(16, 960)
    g = torch.zeros(2, 16, 960, 3, dtype=torch.uint8, device=DEV)
    small = (torch.zeros(2, cap, dtype=torch.uint8, device=DEV), torch.zeros(2, dtype=torch.int64, device=DEV))
    video.encode(g, out=small)
    with pytest.raises(ValueError):
        video.encode(g, out=small, gop=2)

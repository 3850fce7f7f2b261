"""H.264 motion search on the H100 (pantomatrix_b200/video.py, gop > 1 and search > 0): the samples are byte for byte
the CPU restatement's (tests/h264_ref.py) on the CPU cases, random clips and the first frames of rendered EMAGE and
CaMN clips at qp 0, 20 and 51; a rendered frame shifted by (5, -3) pixels gets vector (20, -12) on at least 80 % of
the body's moving macroblocks; each GOP encodes as it does alone at the same parity; calls are deterministic and
capture in a CUDA graph; search 0 is pm_h264_encode_gop; gop T + 1 gives the gop T samples; a 300-frame gop 30 search
16 write_mp4 file decodes to the restatement's reconstruction."""
import numpy as np
import pytest
import torch

import h264_ref as R
from test_video import decode
from test_video_gop_gpu import rendered_gop, samples  # noqa: F401  (the module fixture)
from test_video_me import GOPS, gop_of, me_cases
from pantomatrix_b200 import video

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _samples(frames, qp, gop, search):
    data, nbytes = video.encode(frames, qp=qp, gop=gop, search=search)
    data, nbytes = data.cpu().numpy(), nbytes.cpu().numpy()
    assert all(not data[i, k:].any() for i, k in enumerate(nbytes))
    return [data[i, :k].tobytes() for i, k in enumerate(nbytes)]


@pytest.mark.parametrize("g", GOPS, ids=[str(g) for g in GOPS])
@pytest.mark.parametrize("name,frames,qp,search,truth", me_cases(), ids=[c[0] for c in me_cases()])
def test_me_cases_are_byte_identical_to_the_restatement(name, frames, qp, search, truth, g):
    gop = gop_of(g, len(frames))
    got = _samples(torch.as_tensor(np.stack(frames), device=DEV), qp, gop, search)
    assert got == [e[0] for e in R.encode_clip(frames, qp, gop, search)]


def test_random_clips_are_byte_identical_to_the_restatement():
    rng = np.random.default_rng(12)
    for h, w in ((16, 32), (48, 64), (96, 160)):
        base = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
        clip = [base]
        for t in range(1, 5):
            f = np.roll(clip[-1], (int(rng.integers(-3, 4)), int(rng.integers(-5, 6))), (0, 1))
            y, x = rng.integers(0, h - 8), rng.integers(0, w - 8)
            f[y:y + 8, x:x + 8] = rng.integers(0, 256, (8, 8, 3))
            clip.append(f)
        for qp, gop, search in ((0, 3, 32), (12, 4, 1), (30, 5, 7), (45, 2, 16)):
            got = _samples(torch.as_tensor(np.stack(clip), device=DEV), qp, gop, search)
            want = R.encode_clip(clip, qp, gop, search)
            for i, (b, e) in enumerate(zip(got, want)):
                assert b == e[0], (h, w, qp, gop, search, i)
                assert len(b) <= video.max_bytes(h, w, gop)


@pytest.mark.parametrize("qp", [0, 20, 51])
def test_rendered_clips_are_byte_identical_to_the_restatement(rendered_gop, qp):
    emage, body = rendered_gop
    for clip, gop, search in ((emage[0, :4], 4, 16), (body[1, :4], 4, 16)):
        got = _samples(clip, qp, gop, search)
        assert got == [e[0] for e in R.encode_clip(list(clip.cpu().numpy()), qp, gop, search)], qp


def test_a_shifted_render_gets_the_shift_as_vector(rendered_gop):
    emage, _ = rendered_gop
    a = emage[0, 0]
    b = torch.zeros_like(a)
    b[3:, :-5] = a[:-3, 5:]                               # each sample of b is a's 5 to the right and 3 up
    enc = R.encode_clip([a.cpu().numpy(), b.cpu().numpy()], 20, 2, 8)
    got = _samples(torch.stack([a, b]), 20, 2, 8)
    assert got == [e[0] for e in enc]
    types, mv = enc[1].types, enc[1].mv
    body = (types == "P") & (mv != 0).any(-1)
    hit = (mv[body] == (20, -12)).all(-1)
    # the others match another vector at no higher J: flat shading, where a shorter vector costs fewer bits
    assert body.sum() >= 20 and hit.mean() >= 0.8, (int(body.sum()), float(hit.mean()))


def test_batch_encodes_each_gop_as_alone_at_the_same_parity(rendered_gop):
    _, body = rendered_gop
    clips = body[:, :9].contiguous()                     # (2, 9, ...): GOPs t = 0..3, 4..7, 8 at gop 4
    both = _samples(clips, 20, 4, 16)
    for b in range(2):
        for t0 in (0, 4, 8):
            t1 = min(t0 + 4, 9)
            alone = _samples(clips[b, t0:t1], 20, 4, 16)
            if (t0 // 4) % 2:                            # parity 1: the GOP after a GOP of the same frames
                alone = _samples(torch.cat([clips[b, t0:t1], clips[b, t0:t1]]), 20, t1 - t0, 16)[t1 - t0:]
            assert alone == both[9 * b + t0:9 * b + t1], (b, t0)
    assert _samples(clips[0], 20, 4, 16) == _samples(clips[:1], 20, 4, 16) == both[:9]


def test_deterministic_and_captured_replay_equals_eager(rendered_gop):
    emage, _ = rendered_gop
    frames = emage[0, :6]
    a, na = video.encode(frames, gop=3, search=16)
    b, nb = video.encode(frames, gop=3, search=16)
    assert torch.equal(a, b) and torch.equal(na, nb)
    out = (torch.full_like(a, 0xAB), torch.zeros_like(na))
    video.encode(frames, out=out, gop=3, search=16)
    torch.cuda.synchronize()
    out[0].fill_(0xCD)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        video.encode(frames, out=out, gop=3, search=16)
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(out[0], a) and torch.equal(out[1], na)


def test_search_0_is_encode_gop_and_gop_past_t_is_gop_t(rendered_gop):
    _, body = rendered_gop
    assert _samples(body, 20, 4, 0) == samples(body, 20, 4)
    assert _samples(body, 20, 11, 16) == _samples(body, 20, 10, 16)
    assert _samples(body, 20, 1, 16) == samples(body, 20, 1)


def test_write_mp4_gop_30_search_16_of_a_300_frame_render_decodes_to_the_reconstruction(rendered_gop, tmp_path):
    emage, _ = rendered_gop
    path = video.write_mp4(emage[0], str(tmp_path / "clip.mp4"), fps=30, gop=30, search=16)
    lumas, _, fps = decode(path)
    assert len(lumas) == 300 and fps == 30
    host = emage[0].cpu().numpy()
    for t0 in (0, 270):
        for i, e in enumerate(R.encode_clip(list(host[t0:t0 + 3]), 20, 30, 16)):
            assert np.array_equal(lumas[t0 + i].reshape(-1)[:720 * 960].reshape(720, 960), e[1][0]), t0 + i

"""H.264 encoding on the H100 (pantomatrix_b200/video.py): the samples are byte for byte the CPU restatement's
(oracle/h264_oracle.py) on the CPU cases, random frames and rendered EMAGE and CaMN frames at qp 0, 20 and 51; a batch
encodes each frame as it does alone at the same index parity; calls are deterministic and capture in a CUDA graph; a
300-frame write_mp4 file decodes to the oracle's reconstruction; bad inputs raise ValueError."""
import numpy as np
import pytest
import torch

from oracle import h264_oracle as O
from oracle.weights import synth_audio
from pantomatrix_b200 import video
from pantomatrix_b200.body_model import SmplxBodyModel
from pantomatrix_b200.pipeline import generate
from pantomatrix_b200.render import MeshRenderer
from synthetic_models import build_lstm_product, build_product, smplx_surface_arrays
from test_video import cases, decode

pytestmark = pytest.mark.gpu
DEV = "cuda"


def samples(frames, qp=20):
    data, nbytes = video.encode(frames, qp=qp)
    data, nbytes = data.cpu().numpy(), nbytes.cpu().numpy()
    assert all(not data[i, k:].any() for i, k in enumerate(nbytes))
    return [data[i, :k].tobytes() for i, k in enumerate(nbytes)]


@pytest.fixture(scope="module")
def rendered():
    """EMAGE generate() output drawn by render_sequence (1 x 300 frames, 960 x 720) and CaMN forward() output drawn by
    render_body(upsample=2) (2 clips, 480 x 720), on the full-size synthetic surface model."""
    model, vqm = build_product(seed=0, device=DEV)
    _, pred = generate(model, vqm, torch.from_numpy(synth_audio(1, 160000, 5)).to(DEV))
    r = MeshRenderer(SmplxBodyModel(smplx_surface_arrays(), DEV))
    emage = r.render_sequence(pred["motion_axis_angle"], pred["expression"], pred["trans"])
    camn = build_lstm_product("camn", device=DEV)
    poses = camn(torch.from_numpy(synth_audio(2, 160000, 6)).to(DEV),
                 torch.zeros(2, 1, dtype=torch.long, device=DEV))["motion_axis_angle"]
    poses = poses.reshape(2, poses.shape[1], 165)
    body = r.render_body(poses, torch.zeros(2, poses.shape[1], 3, device=DEV), upsample=2)
    torch.cuda.synchronize()
    return emage, body


@pytest.mark.parametrize("name,frames,qp", cases(), ids=[c[0] for c in cases()])
def test_cases_are_byte_identical_to_the_oracle(name, frames, qp):
    got = samples(torch.as_tensor(np.stack(frames), device=DEV), qp)
    for i, f in enumerate(frames):
        assert got[i] == O.encode(f, qp, i)[0], i


def test_every_qp_is_byte_identical_to_the_oracle():
    rng = np.random.default_rng(9)
    f = rng.integers(0, 256, (32, 48, 3), dtype=np.uint8)
    f[16:] = f[16:] // 32 * 32
    t = torch.as_tensor(f, device=DEV)[None]
    for qp in range(52):
        assert samples(t, qp)[0] == O.encode(f, qp, 0)[0], qp


def test_random_frames_are_byte_identical_to_the_oracle():
    rng = np.random.default_rng(11)
    for h, w in ((16, 32), (48, 64), (96, 160)):
        fr = rng.integers(0, 256, (4, h, w, 3), dtype=np.uint8)
        fr[1] = fr[1] // 64 * 64
        fr[2] = np.repeat(fr[2][:, :1], w, 1)
        fr[3] = np.repeat(np.repeat(fr[3][:h // 8, :w // 8], 8, 0), 8, 1)
        for qp in (0, 12, 30):
            for i, b in enumerate(samples(torch.as_tensor(fr, device=DEV), qp)):
                assert b == O.encode(fr[i], qp, i)[0], (h, w, qp, i)
                assert len(b) <= video.max_bytes(h, w)


@pytest.mark.parametrize("qp", [0, 20, 51])
def test_rendered_frames_are_byte_identical_to_the_oracle(rendered, qp):
    emage, body = rendered
    for clip, picks in ((emage, (0, 151)), (body, (3,))):
        got = samples(clip, qp)
        flat = clip.view(-1, *clip.shape[2:])
        t = clip.shape[1]
        for i in picks:
            assert got[i] == O.encode(flat[i].cpu().numpy(), qp, i % t)[0], (qp, i)


def test_batch_encodes_each_frame_as_alone_at_the_same_parity(rendered):
    _, body = rendered
    frames = body.view(-1, 720, 480, 3)[::37][:8]
    both = samples(frames)
    for i in range(frames.shape[0]):
        alone = samples(frames[i:i + 1]) if i % 2 == 0 else samples(frames[i - 1:i + 1])[1:]
        assert alone[0] == both[i], i
    # (B, T, ...) input: the index is t, so both clips' frame t is coded alike
    pair = samples(torch.stack([frames[:4], frames[:4]]))
    assert pair[:4] == pair[4:] == both[:4]


def test_deterministic_and_captured_replay_equals_eager(rendered):
    emage, _ = rendered
    frames = emage[0, :16]
    a, na = video.encode(frames)
    b, nb = video.encode(frames)
    assert torch.equal(a, b) and torch.equal(na, nb)
    out = (torch.full_like(a, 0xAB), torch.zeros_like(na))
    video.encode(frames, out=out)                        # eager call before capture
    torch.cuda.synchronize()
    out[0].fill_(0xCD)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        video.encode(frames, out=out)
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(out[0], a) and torch.equal(out[1], na)


def test_write_mp4_of_a_300_frame_render_decodes_to_the_reconstruction(rendered, tmp_path):
    emage, _ = rendered
    assert emage.shape == (1, 300, 720, 960, 3)
    path = video.write_mp4(emage[0], str(tmp_path / "clip.mp4"), fps=30)
    lumas, _, fps = decode(path)
    assert len(lumas) == 300 and fps == 30
    host = emage[0].cpu().numpy()
    for i in (0, 1, 299):
        _, (ry, _, _), _ = O.encode(host[i], 20, i)
        assert np.array_equal(lumas[i].reshape(-1)[:720 * 960].reshape(720, 960), ry), i


def test_errors_raise_value_error(tmp_path):
    f = torch.zeros(2, 16, 32, 3, dtype=torch.uint8, device=DEV)
    bad = [torch.zeros(2, 16, 32, 3, dtype=torch.uint8),                       # CPU
           f.float(),                                                          # dtype
           f[..., :2], f[0], torch.zeros(2, 16, 0, 3, dtype=torch.uint8, device=DEV),   # shapes
           torch.zeros(2, 24, 32, 3, dtype=torch.uint8, device=DEV),           # H not a multiple of 16
           torch.zeros(2, 16, 40, 3, dtype=torch.uint8, device=DEV),           # W not a multiple of 16
           torch.zeros(1, 16, 16 * 544, 3, dtype=torch.uint8, device=DEV),     # wider than level 5.1 allows
           f[:, :, ::2]]                                                       # not dense
    for x in bad:
        with pytest.raises(ValueError):
            video.encode(x)
    for qp in (-1, 52, 20.0):
        with pytest.raises(ValueError):
            video.encode(f, qp=qp)
    for fps in (0, -30):
        with pytest.raises(ValueError):
            video.write_mp4(f, str(tmp_path / "x.mp4"), fps=fps)
    cap = video.slot_bytes(16, 32)
    for out in ((torch.zeros(2, cap - 4, dtype=torch.uint8, device=DEV), torch.zeros(2, dtype=torch.int64, device=DEV)),
                (torch.zeros(2, cap + 2, dtype=torch.uint8, device=DEV), torch.zeros(2, dtype=torch.int64, device=DEV)),
                (torch.zeros(2, cap, dtype=torch.uint8, device=DEV), torch.zeros(2, dtype=torch.int32, device=DEV)),
                (torch.zeros(1, cap, dtype=torch.uint8, device=DEV), torch.zeros(2, dtype=torch.int64, device=DEV))):
        with pytest.raises(ValueError):
            video.encode(f, out=out)

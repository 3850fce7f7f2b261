"""PNG encoding on the H100 (pantomatrix_b200/png.py): the files are byte for byte the CPU restatement's
(oracle/png_oracle.py) on the edge cases, random frames and rendered EMAGE and CaMN frames; every frame of a 300-frame
render decodes back to it; a batch encodes each frame as it does alone; calls are deterministic and capture in a CUDA
graph; write_frames' files open in Pillow as the frames; bad inputs raise ValueError."""
import zlib

import numpy as np
import pytest
import torch
from PIL import Image

from oracle import png_oracle as P
from oracle.weights import synth_audio
from pantomatrix_b200 import png
from pantomatrix_b200.body_model import SmplxBodyModel
from pantomatrix_b200.pipeline import generate
from pantomatrix_b200.render import MeshRenderer
from synthetic_models import build_lstm_product, build_product, smplx_surface_arrays
from test_png import cases, check_file

pytestmark = pytest.mark.gpu
DEV = "cuda"


def files(frames):
    data, nbytes = png.encode(frames)
    data, nbytes = data.cpu().numpy(), nbytes.cpu().numpy()
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


@pytest.mark.parametrize("name,frame", cases(), ids=[c[0] for c in cases()])
def test_edge_cases_are_byte_identical_to_the_oracle(name, frame):
    got = files(torch.as_tensor(frame, device=DEV)[None])[0]
    assert got == P.encode(frame)


def test_random_frames_are_byte_identical_to_the_oracle():
    rng = np.random.default_rng(11)
    for h, w in ((1, 2), (7, 13), (48, 64), (90, 120)):
        # noise, and noise quantised to a few levels so matches of every distance occur
        fr = rng.integers(0, 256, (3, h, w, 3), dtype=np.uint8)
        fr[1] = fr[1] // 64 * 64
        fr[2] = np.repeat(fr[2][:, :1], w, 1) if w > 1 else fr[2]
        for f, b in zip(fr, files(torch.as_tensor(fr, device=DEV))):
            assert b == P.encode(f)
            assert len(b) <= png.max_bytes(h, w)


def test_rendered_frames_are_byte_identical_to_the_oracle(rendered):
    emage, body = rendered
    for clip, picks in ((emage, (0, 150, 299)), (body, (0, 269))):
        frames = clip.view(-1, *clip.shape[2:])
        got = files(frames)
        for i in picks:
            want = P.encode(frames[i].cpu().numpy())
            assert got[i] == want, i


def test_every_frame_of_a_300_frame_render_decodes_back(rendered):
    emage, _ = rendered
    assert emage.shape == (1, 300, 720, 960, 3)
    data, nbytes = png.encode(emage)                     # (B, T, H, W, 3) read in place
    host, sizes = data.cpu().numpy(), nbytes.cpu().numpy()
    frames = emage[0].cpu().numpy()
    for i in range(300):
        b = host[i, :sizes[i]]
        assert not host[i, sizes[i]:].any()
        if i % 50 == 0:
            check_file(b.tobytes(), frames[i])
        z = b[41:-16].tobytes()
        assert zlib.crc32(b[37:-16].tobytes()) == int.from_bytes(b[-16:-12].tobytes(), "big")
        raw = np.frombuffer(zlib.decompress(z), np.uint8).reshape(720, 2881)
        pix = raw[:, 1:].astype(np.int64)
        pix = np.cumsum(pix.reshape(720, 960, 3), axis=1) & 0xFF         # undo Sub: running sums per channel
        assert np.array_equal(pix.astype(np.uint8), frames[i]), i


def test_batch_encodes_each_frame_as_alone(rendered):
    _, body = rendered
    frames = body.view(-1, 720, 480, 3)[::37]
    both = files(frames)
    for i in range(frames.shape[0]):
        assert files(frames[i:i + 1])[0] == both[i]


def test_deterministic_and_captured_replay_equals_eager(rendered):
    emage, _ = rendered
    frames = emage[0, :16]
    a, na = png.encode(frames)
    b, nb = png.encode(frames)
    assert torch.equal(a, b) and torch.equal(na, nb)
    out = (torch.full_like(a, 0xAB), torch.zeros_like(na))
    png.encode(frames, out=out)                          # eager call before capture
    torch.cuda.synchronize()
    out[0].fill_(0xCD)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        png.encode(frames, out=out)
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(out[0], a) and torch.equal(out[1], na)


def test_write_frames_files_open_as_the_frames(rendered, tmp_path):
    _, body = rendered
    frames = body[1, :12]
    paths = png.write_frames(frames, str(tmp_path / "f"))
    assert [p.rsplit("/", 1)[1] for p in paths] == [f"frame_{i:05d}.png" for i in range(12)]
    want = frames.cpu().numpy()
    for i, p in enumerate(paths):
        assert np.array_equal(np.asarray(Image.open(p)), want[i])


def test_errors_raise_value_error():
    f = torch.zeros(2, 8, 8, 3, dtype=torch.uint8, device=DEV)
    bad = [torch.zeros(2, 8, 8, 3, dtype=torch.uint8),                         # CPU
           f.float(),                                                          # dtype
           f[..., :2], f[0], torch.zeros(2, 8, 0, 3, dtype=torch.uint8, device=DEV),   # shapes
           f[:, :, ::2],                                                       # not dense
           torch.empty(1, 16000, 40000, 3, dtype=torch.uint8, device=DEV)]     # bound past 2^31 bytes
    for x in bad:
        with pytest.raises(ValueError):
            png.encode(x)
    cap = png.slot_bytes(8, 8)
    for out in ((torch.zeros(2, cap - 4, dtype=torch.uint8, device=DEV), torch.zeros(2, dtype=torch.int64, device=DEV)),
                (torch.zeros(2, cap + 2, dtype=torch.uint8, device=DEV), torch.zeros(2, dtype=torch.int64, device=DEV)),
                (torch.zeros(2, cap, dtype=torch.uint8, device=DEV), torch.zeros(2, dtype=torch.int32, device=DEV)),
                (torch.zeros(1, cap, dtype=torch.uint8, device=DEV), torch.zeros(2, dtype=torch.int64, device=DEV))):
        with pytest.raises(ValueError):
            png.encode(f, out=out)

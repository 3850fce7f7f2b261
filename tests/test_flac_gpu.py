"""FLAC encoding on the H100 (pantomatrix_b200/flac.py): the frames are byte for byte the CPU restatement's
(oracle/flac_oracle.py) on the CPU cases and on random clips; a clip in a batch encodes as it does alone; calls are
deterministic and capture in a CUDA graph; a write_mp4 file of rendered frames with 10 s of 48 kHz stereo decodes
through FFmpeg to the trimmed input, sample for sample; bad inputs raise ValueError."""
import numpy as np
import pytest
import torch

from oracle import flac_oracle as O
from pantomatrix_b200 import flac, video
from pantomatrix_b200.body_model import SmplxBodyModel
from pantomatrix_b200.render import MeshRenderer
from synthetic_models import smplx_surface_arrays
from test_flac import cases, decode_audio, speech

pytestmark = pytest.mark.gpu
DEV = "cuda"


def frames(pcm, rate):
    """The GPU's frames of a host clip (n, C), or of each clip of (B, n, C), as lists of bytes."""
    data, nbytes = flac.encode(torch.as_tensor(pcm, device=DEV), rate)
    data, nbytes = data.cpu().numpy(), nbytes.cpu().numpy()
    assert all(not data[i, k:].any() for i, k in enumerate(nbytes))
    out = [data[i, :k].tobytes() for i, k in enumerate(nbytes)]
    if pcm.ndim == 3:
        f = flac.frames_of(pcm.shape[1])
        return [out[b * f:(b + 1) * f] for b in range(pcm.shape[0])]
    return out


@pytest.mark.parametrize("name,pcm,rate", cases(), ids=[c[0] for c in cases()])
def test_cases_are_byte_identical_to_the_oracle(name, pcm, rate):
    assert frames(pcm, rate) == O.encode(pcm, rate)[0]


def test_random_clips_are_byte_identical_to_the_oracle():
    rng = np.random.default_rng(21)
    for trial in range(12):
        c = int(rng.integers(1, 9))
        n = int(rng.integers(1, 3 * 4096))
        scale = int(rng.choice([0, 3, 300, 30000]))
        walk = np.cumsum(rng.integers(-scale, scale + 1, (n, c)), 0)
        if trial % 2:
            pcm = np.clip(walk * 40, -(1 << 23), (1 << 23) - 1).astype(np.int32)
        else:
            pcm = np.clip(walk, -32768, 32767).astype(np.int16)
        rate = int(rng.choice([8000, 16000, 44100, 48000, 37800]))
        got = frames(pcm, rate)
        assert got == O.encode(pcm, rate)[0], (trial, n, c, scale)
        bps = O.check(pcm, rate)
        assert all(len(f) <= flac.max_frame_bytes(c, bps, min(4096, n)) for f in got)


def test_a_clip_in_a_batch_encodes_as_alone():
    clips = np.stack([speech(9000, 16000, s) for s in range(3)])              # (3, 9000, 1)
    clips[1] = 0
    both = frames(clips, 16000)
    for b in range(3):
        assert both[b] == frames(clips[b], 16000), b
    # clips any stride apart: every other clip of a larger batch
    wide = torch.as_tensor(np.concatenate([clips, clips]), device=DEV)[::2]
    data, nbytes = flac.encode(wide, 16000)
    f = flac.frames_of(9000)
    got = [bytes(data[i, :int(nbytes[i])].cpu().numpy()) for i in range(3 * f)]
    want = [x for c in (0, 2, 1) for x in both[c]]
    assert got == want


def test_deterministic_and_captured_replay_equals_eager():
    pcm = torch.as_tensor(np.concatenate([speech(30000, 48000, 1), speech(30000, 48000, 2)], 1), device=DEV)
    a, na = flac.encode(pcm, 48000)
    b, nb = flac.encode(pcm, 48000)
    assert torch.equal(a, b) and torch.equal(na, nb)
    out = (torch.full_like(a, 0xAB), torch.zeros_like(na))
    flac.encode(pcm, 48000, out=out)                   # eager call before capture
    torch.cuda.synchronize()
    out[0].fill_(0xCD)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        flac.encode(pcm, 48000, out=out)
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(out[0], a) and torch.equal(out[1], na)


def test_write_mp4_with_audio_decodes_to_the_trimmed_input(tmp_path):
    """300 rendered frames at 30 fps beside 10.5 s of 48 kHz stereo: the file holds the first 10 s, exactly."""
    r = MeshRenderer(SmplxBodyModel(smplx_surface_arrays(), DEV))
    t = torch.arange(300, device=DEV, dtype=torch.float32)[:, None]
    poses = torch.zeros(1, 300, 165, device=DEV)
    poses[0, :, 3:6] = 0.3 * torch.sin(t / 20)
    clip = r.render_body(poses, torch.zeros(1, 300, 3, device=DEV))[0]
    n = 48000 * 21 // 2
    pcm = np.concatenate([speech(n, 48000, 4), speech(n, 48000, 5) // 2], 1)
    path = video.write_mp4(clip, str(tmp_path / "clip.mp4"), fps=30, audio=(torch.as_tensor(pcm, device=DEV), 48000))
    got, rate = decode_audio(path)
    assert rate == 48000 and np.array_equal(got, pcm[:480000].astype(np.int64))
    silent = video.write_mp4(clip, str(tmp_path / "silent.mp4"), fps=30)
    a, b = open(path, "rb").read(), open(silent, "rb").read()
    assert len(a) > len(b)
    from test_video import decode
    assert [np.array_equal(x, y) for x, y in zip(decode(path)[0], decode(silent)[0])] == [True] * 300


def test_out_of_range_24_bit_samples_are_flagged():
    pcm = torch.zeros(9000, 2, dtype=torch.int32, device=DEV)
    pcm[5000, 1] = 1 << 23
    _, nbytes = flac.encode(pcm, 48000)
    assert nbytes.tolist()[0] > 0 and nbytes.tolist()[1] == -1 and nbytes.tolist()[2] > 0
    f = torch.zeros(30, 16, 16, 3, dtype=torch.uint8, device=DEV)
    with pytest.raises(ValueError):
        video.write_mp4(f, "/nonexistent/x.mp4", audio=(pcm, 48000))


def test_errors_raise_value_error():
    p = torch.zeros(100, 2, dtype=torch.int16, device=DEV)
    bad = [torch.zeros(100, 2, dtype=torch.int16),                          # CPU
           p.float(), p.to(torch.int64),                                   # dtype
           p[0], torch.zeros(0, 2, dtype=torch.int16, device=DEV),         # shapes
           torch.zeros(100, 9, dtype=torch.int16, device=DEV),             # channels
           torch.zeros(2, 100, 4, dtype=torch.int16, device=DEV)[..., ::2],    # not dense
           torch.zeros(100, 2, 1, dtype=torch.int16, device=DEV).expand(100, 2, 3)]
    for x in bad:
        with pytest.raises(ValueError):
            flac.encode(x, 16000)
    for rate in (0, 65536, 16000.0, True):
        with pytest.raises(ValueError):
            flac.encode(p, rate)
    cap = flac.slot_bytes(2, 16, 100)
    for out in ((torch.zeros(1, cap - 4, dtype=torch.uint8, device=DEV), torch.zeros(1, dtype=torch.int64, device=DEV)),
                (torch.zeros(1, cap + 2, dtype=torch.uint8, device=DEV), torch.zeros(1, dtype=torch.int64, device=DEV)),
                (torch.zeros(1, cap, dtype=torch.uint8, device=DEV), torch.zeros(1, dtype=torch.int32, device=DEV)),
                (torch.zeros(2, cap, dtype=torch.uint8, device=DEV), torch.zeros(1, dtype=torch.int64, device=DEV))):
        with pytest.raises(ValueError):
            flac.encode(p, 16000, out=out)
    f = torch.zeros(3, 16, 16, 3, dtype=torch.uint8, device=DEV)
    for audio in ((p, 0), (p[None], 16000), (p.cpu(), 16000), (p[:, :1], 9)):        # 3 frames hold no 9 Hz sample
        with pytest.raises(ValueError):
            video.write_mp4(f, "/nonexistent/x.mp4", audio=audio)

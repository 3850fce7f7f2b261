"""The H.264 encoding rule on the CPU (oracle/h264_oracle.py, DESIGN.md section 12): its MP4 files decode with
OpenCV's FFmpeg to the oracle's reconstruction, luma bit for bit; the colour rule, the size bound, the fallbacks and
the parameter sets; the muxer's box tree; and the ops wrapper's ctypes arguments.  The GPU's bytes are compared with
these in tests/test_video_gpu.py."""
import ctypes
import struct

import numpy as np
import pytest
import torch

from oracle import h264_oracle as O
from pantomatrix_b200 import video

def encode_clip(frames, qp=20):
    """The oracle's samples, reconstructions and macroblock types of a list of frames (index = position)."""
    return [O.encode(f, qp, i) for i, f in enumerate(frames)]


def decode(path):
    """(luma planes, BGR frames, fps) of an MP4 file, by OpenCV's FFmpeg."""
    cv2 = pytest.importorskip("cv2")
    out = []
    for convert in (0, 1):
        cap = cv2.VideoCapture(path, cv2.CAP_FFMPEG)
        assert cap.isOpened()
        cap.set(cv2.CAP_PROP_CONVERT_RGB, convert)
        fps, frames = cap.get(cv2.CAP_PROP_FPS), []
        while True:
            ok, fr = cap.read()
            if not ok:
                break
            frames.append(np.asarray(fr))
        cap.release()
        out.append(frames)
    return out[0], out[1], fps


def check_clip(enc, h, w, tmp_path, fps=30):
    """The oracle's MP4 decodes to its reconstruction: frame count, size, fps, luma exact, BGR within 3."""
    cv2 = pytest.importorskip("cv2")
    path = str(tmp_path / "clip.mp4")
    with open(path, "wb") as f:
        f.write(video.mp4_bytes([e[0] for e in enc], h, w, fps))
    lumas, bgrs, got_fps = decode(path)
    assert len(lumas) == len(enc) == len(bgrs)
    assert abs(got_fps - fps) < 1e-6
    for e, y, bgr in zip(enc, lumas, bgrs):
        ry, rcb, rcr = e[1]
        assert y.reshape(-1)[:h * w].reshape(h, w).tolist() == ry.tolist()
        i420 = np.concatenate([ry.reshape(-1), rcb.reshape(-1), rcr.reshape(-1)]).astype(np.uint8)
        want = cv2.cvtColor(i420.reshape(h * 3 // 2, w), cv2.COLOR_YUV2BGR_I420)
        assert bgr.shape == (h, w, 3)
        # FFmpeg's converter and cvtColor treat samples outside the nominal range (noise at high qp can reconstruct
        # to Y = 0) differently: compare where the pixel's Y, Cb and Cr are nominal
        c = lambda p: np.repeat(np.repeat(p, 2, 0), 2, 1)
        nominal = (ry >= 16) & (ry <= 235) & (c(rcb) >= 16) & (c(rcb) <= 240) & (c(rcr) >= 16) & (c(rcr) <= 240)
        assert nominal.mean() > 0.99
        assert np.abs(bgr.astype(int) - want.astype(int))[nominal].max(initial=0) <= 3
        assert len(e[0]) <= video.max_bytes(h, w)


def _grad(h, w):
    g = np.zeros((h, w, 3), np.uint8)
    g[..., 0] = (np.arange(w)[None] * 255 // max(w - 1, 1))
    g[..., 1] = (np.arange(h)[:, None] * 255 // max(h - 1, 1))
    g[..., 2] = (np.arange(h)[:, None] + np.arange(w)[None]) * 3 % 256
    return g


def _blocks(h, w):
    """High-contrast 4x4 checker blocks: large transform levels that take level escapes at qp 0."""
    yy, xx = np.mgrid[:h, :w]
    v = np.where(((yy // 4) + (xx // 4)) % 2 == 0, 255, 0).astype(np.uint8)
    v[(yy % 16 < 2)] = 0
    return np.stack([v, 255 - v, v], -1)


def cases():
    """(name, frames, qp) cases, shared with the GPU test."""
    rng = np.random.default_rng(7)
    noise = lambda h, w: rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
    smooth = np.repeat(np.repeat(noise(6, 8), 8, 0), 8, 1)
    return [("16x16", [noise(16, 16)], 20),
            ("one_row", [noise(16, 80), noise(16, 80)], 20),
            ("one_column", [noise(64, 16)], 26),
            ("black", [np.zeros((32, 48, 3), np.uint8)], 20),
            ("white", [np.full((32, 48, 3), 255, np.uint8)], 20),
            ("grey", [np.full((32, 48, 3), 128, np.uint8)], 20),
            ("gradient", [_grad(48, 64), _grad(48, 64)[::-1].copy()], 20),
            ("gradient_qp0", [_grad(48, 64)], 0),
            ("blocky", [smooth], 10),
            ("noise_qp0", [noise(32, 48)], 0),
            ("noise_qp36", [noise(32, 48), noise(32, 48), noise(32, 48)], 36),
            ("contrast_qp0", [_blocks(32, 64)], 0)]


@pytest.mark.parametrize("name,frames,qp", cases(), ids=[c[0] for c in cases()])
def test_oracle_clips_decode_to_the_reconstruction(name, frames, qp, tmp_path):
    h, w, _ = frames[0].shape
    check_clip(encode_clip(frames, qp), h, w, tmp_path)


def test_every_qp_decodes_to_the_reconstruction(tmp_path):
    rng = np.random.default_rng(5)
    f = rng.integers(0, 256, (32, 32, 3), dtype=np.uint8)
    f[:16] = _grad(16, 32)
    for qp in range(52):
        enc = [O.encode(f, qp, 0)]
        check_clip(enc, 32, 32, tmp_path)


def test_noise_at_qp0_falls_back_to_pcm_with_source_luma():
    f = np.random.default_rng(1).integers(0, 256, (32, 48, 3), dtype=np.uint8)
    _, (ry, rcb, rcr), types = O.encode(f, 0)
    assert (types == O.PCM).all()
    y, cb, cr = O.colour(f)
    assert np.array_equal(ry, y) and np.array_equal(rcb, cb) and np.array_equal(rcr, cr)


def test_high_contrast_blocks_at_qp0_use_level_escapes():
    """The contrast case codes Intra16x16 macroblocks whose levels need level_prefix 14 or 15 (the escapes)."""
    seen = []
    orig = O.Bits.put

    def spy(self, v, n):
        if v == 1 and n in (15, 16):                   # level_prefix 14 / 15: 14 / 15 zeros, then a one
            seen.append(n)
        return orig(self, v, n)

    O.Bits.put = spy
    try:
        _, _, types = O.encode(_blocks(32, 64), 0)
    finally:
        O.Bits.put = orig
    assert (types != O.PCM).any() and 16 in seen


def test_colour_rule_is_within_one_of_float_bt601():
    rng = np.random.default_rng(2)
    f = rng.integers(0, 256, (64, 64, 3), dtype=np.uint8)
    f[:2, :2] = [[[0, 0, 0], [255, 255, 255]], [[255, 0, 0], [0, 0, 255]]]
    y, cb, cr = O.colour(f)
    x = f.astype(np.float64)
    yf = 16 + (65.481 * x[..., 0] + 128.553 * x[..., 1] + 24.966 * x[..., 2]) / 255
    m = x.reshape(32, 2, 32, 2, 3).mean((1, 3))
    cbf = 128 + (-37.797 * m[..., 0] - 74.203 * m[..., 1] + 112.0 * m[..., 2]) / 255
    crf = 128 + (112.0 * m[..., 0] - 93.786 * m[..., 1] - 18.214 * m[..., 2]) / 255
    for got, want in ((y, yf), (cb, cbf), (cr, crf)):
        assert np.abs(got - want).max() <= 1
        assert got.min() >= 16 and got.max() <= 240


def test_bound_is_the_products_and_holds_on_noise():
    rng = np.random.default_rng(3)
    for h, w in ((16, 16), (32, 96), (720, 960), (720, 480)):
        assert O.max_bytes(h, w) == video.max_bytes(h, w)
        assert video.slot_bytes(h, w) % 4 == 0 and video.slot_bytes(h, w) - video.max_bytes(h, w) < 4
    for qp in (0, 51):
        b, _, _ = O.encode(rng.integers(0, 256, (48, 64, 3), dtype=np.uint8), qp)
        assert len(b) <= video.max_bytes(48, 64)


def test_sizes_are_checked():
    for h, w in ((15, 16), (16, 8), (0, 16), (16 * 544, 16), (16 * 200, 16 * 200)):
        with pytest.raises(ValueError):
            video.check_size(h, w)
        with pytest.raises(ValueError):
            O.check_shape(h, w)
    video.check_size(16 * 543, 16 * 16)


def test_parameter_sets_match_the_oracle():
    for h, w in ((16, 16), (720, 960), (720, 480), (16 * 543, 16 * 64)):
        assert video.sps(h, w) == O.sps(h, w)
    assert video.pps() == O.pps()


def test_samples_are_length_prefixed_slices_one_per_row():
    f = np.random.default_rng(4).integers(0, 256, (48, 32, 3), dtype=np.uint8)
    for idx in (0, 1, 2):
        b, _, _ = O.encode(f, 20, idx)
        at, rows = 0, 0
        while at < len(b):
            n = int.from_bytes(b[at:at + 4], "big")
            nal = b[at + 4:at + 4 + n]
            assert nal[0] == 0x65 and b"\x00\x00\x00" not in nal and b"\x00\x00\x01" not in nal
            at += 4 + n
            rows += 1
        assert at == len(b) and rows == 3
    assert O.encode(f, 20, 0)[0] == O.encode(f, 20, 2)[0] != O.encode(f, 20, 1)[0]


def test_emulation_prevention():
    assert O.emulation_prevent(b"\x00\x00\x00\x00\x00\x01\x00\x00\x04") == b"\x00\x00\x03\x00\x00\x03\x00\x01\x00\x00\x04"


def _boxes(b, at=0, end=None, depth=0):
    """The box tree of an ISO BMFF byte string as (type, payload offset, end, children)."""
    end = len(b) if end is None else end
    out = []
    containers = {b"moov", b"trak", b"mdia", b"minf", b"dinf", b"stbl"}
    while at < end:
        size, kind = struct.unpack(">I4s", b[at:at + 8])
        assert size >= 8 and at + size <= end
        kids = _boxes(b, at + 8, at + size, depth + 1) if kind in containers else []
        out.append((kind, at + 8, at + size, kids))
        at += size
    assert at == end
    return out


def test_mp4_box_tree_parses():
    samples = [b"\x00\x00\x00\x02\x65\x88", b"\x00\x00\x00\x03\x65\x88\x80", b"\x00\x00\x00\x01\x65"]
    blob = video.mp4_bytes(samples, 32, 48, 30)
    top = _boxes(blob)
    assert [t[0] for t in top] == [b"ftyp", b"moov", b"mdat"]
    find = lambda boxes, *path: find([c for c in boxes if c[0] == path[0]][0][3], *path[1:]) if len(path) > 1 \
        else [c for c in boxes if c[0] == path[0]][0]
    stbl = find(top, b"moov", b"trak", b"mdia", b"minf", b"stbl")
    assert [c[0] for c in stbl[3]] == [b"stsd", b"stts", b"stsc", b"stsz", b"stco"]
    body = {c[0]: blob[c[1]:c[2]] for c in stbl[3]}
    assert struct.unpack(">IIII", body[b"stts"]) == (0, 1, 3, 1)
    assert struct.unpack(">IIIII", body[b"stsz"][:20]) == (0, 0, 3, 6, 7)
    off = struct.unpack(">III", body[b"stco"])[2]
    mdat = top[2]
    assert off == mdat[1] and blob[off:mdat[2]] == b"".join(samples)
    assert b"avcC" in body[b"stsd"] and video.sps(32, 48) in body[b"stsd"] and video.pps() in body[b"stsd"]
    mdhd = find(top, b"moov", b"trak", b"mdia", b"mdhd")
    assert struct.unpack(">III", blob[mdhd[1] + 12:mdhd[1] + 24])[0:2] == (30, 3)
    with pytest.raises(ValueError):
        video.mp4_bytes(samples, 32, 48, 0)
    with pytest.raises(ValueError):
        video.mp4_bytes(samples, 32, 48, -1.5)
    with pytest.raises(ValueError):
        video.mp4_bytes([], 32, 48, 30)
    with pytest.raises(ValueError):
        video.mp4_bytes([memoryview(bytearray(1 << 20))] * 4096, 32, 48, 30)   # 4 GiB of samples


def test_encode_rejects_bad_inputs_on_the_host():
    with pytest.raises(ValueError):
        video.encode(torch.zeros(2, 16, 16, 3, dtype=torch.uint8))             # CPU tensor
    with pytest.raises(ValueError):
        video.encode(np.zeros((2, 16, 16, 3), np.uint8))                       # not a tensor
    for qp in (-1, 52, 2.0, True):
        with pytest.raises(ValueError):
            video._qp(qp)


def test_ops_h264_wrapper_marshals_valid_arguments(monkeypatch):
    """ops.h264_encode with the library call replaced by a recorder: every argument converts to its declared ctypes
    type, the slots are cleared first, and the two stages share the workspace."""
    from pantomatrix_b200 import _lib, ops
    calls = []

    def record(name, *args):
        sig = _lib.SIGNATURES[name]
        assert len(args) == len(sig), (name, len(args), len(sig))
        for i, (a, t) in enumerate(zip(args, sig)):
            if t is ctypes.c_void_p:
                assert a is None or isinstance(a, int), (name, i, type(a))
            else:
                assert isinstance(a, int) and not isinstance(a, bool), (name, i, type(a))
                t(a)
        calls.append((name, args))

    monkeypatch.setattr(_lib, "call", record)
    monkeypatch.setattr(ops, "_chk", lambda t, dtype=torch.float32: t)
    monkeypatch.setattr(ops, "_stream", lambda: 0)
    frames = torch.zeros(3, 32, 48, 3, dtype=torch.uint8)
    cap, sc = video.slot_bytes(32, 48), video.slice_bytes(48)
    data, nbytes = torch.zeros(3, cap, dtype=torch.uint8), torch.zeros(3, dtype=torch.int64)
    scratch, sizes = torch.zeros(3, 2, sc, dtype=torch.uint8), torch.zeros(3, 2, dtype=torch.int32)
    ops.h264_encode(frames, 3, 20, data, nbytes, scratch, sizes)
    assert [c[0] for c in calls] == ["pm_memset_async", "pm_h264_encode", "pm_h264_gather"]
    by = dict(calls)
    assert by["pm_memset_async"][1:3] == (0, 3 * cap)
    assert by["pm_h264_encode"][1:7] == (32 * 48 * 3, 3, 3, 32, 48, 20)
    assert by["pm_h264_encode"][7:10] == (scratch.data_ptr(), sc, sizes.data_ptr())
    assert by["pm_h264_gather"][3:6] == (scratch.data_ptr(), sc, sizes.data_ptr())
    assert by["pm_h264_gather"][6:9] == (data.data_ptr(), cap, nbytes.data_ptr())

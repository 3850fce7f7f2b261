"""The H.264 GOP rule on the CPU (tests/h264_ref.py, DESIGN.md section 12): clips of IDR and P frames decode with
OpenCV's FFmpeg to the restatement's reconstruction; gop 1 is the intra rule; the gop > 1 bound, SPS and stss box; and
the ops wrapper's ctypes arguments for pm_h264_encode_gop.  The GPU's bytes are compared with these in
tests/test_video_gop_gpu.py."""
import ctypes
import functools
import struct

import numpy as np
import pytest
import torch

import h264_ref as R
from oracle import h264_oracle as O
from pantomatrix_b200 import video
from test_video import _boxes, _grad, decode


def _same_luma_colour(base):
    """An RGB colour with the colour rule's Y of base and a different Cb."""
    y = lambda c: ((66 * c[0] + 129 * c[1] + 25 * c[2] + 128) >> 8) + 16
    for r in range(256):
        for b in range(0, 256, 5):
            g = base[1] + (66 * (base[0] - r) + 25 * (base[2] - b)) // 129
            if 0 <= g < 256 and y((r, g, b)) == y(base) and abs(r - base[0]) > 40:
                return (r, g, b)
    raise AssertionError


def gop_cases():
    """(name, frames, qp) clips, shared with the GPU test."""
    rng = np.random.default_rng(17)
    noise = lambda h, w: rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
    smooth = np.repeat(np.repeat(noise(4, 6), 8, 0), 8, 1)
    square = []
    for t in range(6):
        f = np.zeros((48, 64, 3), np.uint8)
        f[6 + 3 * t:22 + 3 * t, 4 + 5 * t:24 + 5 * t] = (200, 60, 120)
        square.append(f)
    grad = [np.roll(_grad(48, 64), 2 * t, 1) for t in range(5)]
    base = (90, 140, 60)
    other = _same_luma_colour(base)
    chroma = [np.full((32, 48, 3), base, np.uint8) for _ in range(4)]
    for t in range(1, 4):
        chroma[t][8 * t:8 * t + 12, 8:40] = other
    n0 = noise(32, 48)
    # small drift: inter macroblocks with level escapes; new noise: I_PCM in a P slice
    drift = [n0, np.clip(n0.astype(int) + rng.integers(-24, 25, n0.shape), 0, 255).astype(np.uint8), noise(32, 48)]
    drift.append(np.clip(drift[2].astype(int) + rng.integers(-4, 5, n0.shape), 0, 255).astype(np.uint8))
    return [("static", [smooth] * 5, 20),
            ("square", square, 20),
            ("gradient_shift", grad, 20),
            ("chroma_only", chroma, 20),
            ("noise_qp0", drift, 0),
            ("noise_qp36", [noise(32, 48)] + [noise(32, 48)] * 3, 36),
            ("one_row", [noise(16, 80), noise(16, 80) // 2 + 60, noise(16, 80)], 20),
            ("one_column", [noise(64, 16)] * 2 + [noise(64, 16)], 26)]


GOPS = (2, 3, 7, "T", "T+5")


def gop_of(g, t):
    return t if g == "T" else (t + 5 if g == "T+5" else g)


@functools.lru_cache(maxsize=None)
def encoded(name, g):
    frames, qp = {c[0]: (c[1], c[2]) for c in gop_cases()}[name]
    return R.encode_clip(frames, qp, gop_of(g, len(frames)))


@functools.lru_cache(maxsize=None)
def every_qp(qp):
    """The two-frame clip of test_every_qp_decodes_to_the_reconstruction at qp, gop 2."""
    rng = np.random.default_rng(5)
    a = rng.integers(0, 256, (32, 32, 3), dtype=np.uint8)
    a[:16] = _grad(16, 32)
    b = a.copy()
    b[4:20, 6:30] = np.clip(b[4:20, 6:30].astype(int) + rng.integers(-12, 13, (16, 24, 3)), 0, 255)
    return R.encode_clip([a, b], qp, 2)


@functools.lru_cache(maxsize=None)
def noise_bound(qp):
    """The noise clip of test_bound_holds_on_noise_for_gop_above_1 at qp 0 or 51, gop 3."""
    rng = np.random.default_rng(3)
    for q in (0, 51):
        a = rng.integers(0, 256, (48, 64, 3), dtype=np.uint8)
        frames = [a, np.clip(a.astype(int) + rng.integers(-6, 7, a.shape), 0, 255).astype(np.uint8),
                  rng.integers(0, 256, (48, 64, 3), dtype=np.uint8)]
        if q == qp:
            return R.encode_clip(frames, qp, 3)


def check_clip(enc, h, w, gop, tmp_path, fps=30):
    """The restatement's MP4 decodes to its reconstruction: frame count, size, fps, luma exact, BGR within 3 where
    nominal (as test_video.check_clip)."""
    cv2 = pytest.importorskip("cv2")
    path = str(tmp_path / "clip.mp4")
    with open(path, "wb") as f:
        f.write(video.mp4_bytes([e[0] for e in enc], h, w, fps, gop=gop))
    lumas, bgrs, got_fps = decode(path)
    assert len(lumas) == len(enc) == len(bgrs)
    assert abs(got_fps - fps) < 1e-6
    for e, y, bgr in zip(enc, lumas, bgrs):
        ry, rcb, rcr = e[1]
        assert y.reshape(-1)[:h * w].reshape(h, w).tolist() == ry.tolist()
        i420 = np.concatenate([ry.reshape(-1), rcb.reshape(-1), rcr.reshape(-1)]).astype(np.uint8)
        want = cv2.cvtColor(i420.reshape(h * 3 // 2, w), cv2.COLOR_YUV2BGR_I420)
        c = lambda p: np.repeat(np.repeat(p, 2, 0), 2, 1)
        nominal = (ry >= 16) & (ry <= 235) & (c(rcb) >= 16) & (c(rcb) <= 240) & (c(rcr) >= 16) & (c(rcr) <= 240)
        assert nominal.mean() > 0.9              # edges against black reconstruct to Y just under 16
        assert np.abs(bgr.astype(int) - want.astype(int))[nominal].max(initial=0) <= 3
        assert len(e[0]) <= video.max_bytes(h, w, gop)


@pytest.mark.parametrize("g", GOPS, ids=[str(g) for g in GOPS])
@pytest.mark.parametrize("name", [c[0] for c in gop_cases()])
def test_gop_clips_decode_to_the_reconstruction(name, g, tmp_path):
    enc = encoded(name, g)
    h, w = enc[0][1][0].shape
    check_clip(enc, h, w, gop_of(g, len(enc)), tmp_path)


def test_every_macroblock_type_occurs():
    seen = set()
    for name, _, _ in gop_cases():
        for e in encoded(name, 3):
            seen |= set(e[2].reshape(-1))
    assert seen == {R.SKIP, R.INTER, "DC", "H", O.PCM}
    # P frames of the noise clip at qp 0 hold I_PCM macroblocks
    assert any((e[2] == O.PCM).any() for e in encoded("noise_qp0", 3)[1:3])


def test_static_p_slices_are_a_header_and_one_skip_run():
    frames, qp = gop_cases()[0][1:]
    h, w, _ = frames[0].shape
    for e in encoded("static", 7)[1:]:
        assert (e[2] == R.SKIP).all()
        ry = encoded("static", 7)[0][1]
        assert all(np.array_equal(a, b) for a, b in zip(e[1], ry))
    for t, e in enumerate(encoded("static", 7)[1:], 1):
        want = bytearray()
        for my in range(h // 16):
            b = R.p_slice_header(my * (w // 16), t, qp)
            b.ue(w // 16)
            b.trailing()
            nal = O.emulation_prevent(b.tobytes())
            want += len(nal).to_bytes(4, "big") + nal
        assert e[0] == bytes(want)


def test_p_slices_use_level_escapes_at_qp0():
    """Inter macroblocks of the drifting noise clip at qp 0 code levels with level_prefix 14 or 15."""
    frames = gop_cases()[4][1]
    ref = O.encode(frames[0], 0, 0)[1]
    seen = []
    orig = O.Bits.put

    def spy(self, v, n):
        if v == 1 and n in (15, 16):
            seen.append(n)
        return orig(self, v, n)

    O.Bits.put = spy
    try:
        types = R.encode_frame(frames[1], ref, 0, 1, 2).types
    finally:
        O.Bits.put = orig
    assert (types == R.INTER).any() and seen


def test_every_qp_decodes_to_the_reconstruction(tmp_path):
    for qp in range(52):
        check_clip(every_qp(qp), 32, 32, 2, tmp_path)


def test_gop_1_is_the_intra_rule():
    for name, frames, qp in gop_cases()[:4]:
        for t, e in enumerate(R.encode_clip(frames, qp, 1)):
            want = O.encode(frames[t], qp, t)
            assert e[0] == want[0] and (e[2] == want[2]).all()
    # idr_pic_id = (t div gop) mod 2
    sq = gop_cases()[1][1]
    enc = R.encode_clip(sq, 20, 2)
    for t in (0, 2, 4):
        assert enc[t][0] == O.encode(sq[t], 20, t // 2)[0]


def test_bound_holds_on_noise_for_gop_above_1():
    for h, w in ((16, 16), (32, 96), (720, 960), (720, 480), (16 * 543, 16 * 64)):
        assert video.max_bytes(h, w) == O.max_bytes(h, w)
        for gop in (2, 30):
            assert video.max_bytes(h, w, gop) == R.max_bytes(h, w, gop) > video.max_bytes(h, w)
            assert video.slot_bytes(h, w, gop) % 4 == 0 and video.slot_bytes(h, w, gop) - video.max_bytes(h, w, gop) < 4
    for qp in (0, 51):
        for e in noise_bound(qp):
            assert len(e[0]) <= video.max_bytes(48, 64, 3)


def _rbsp_bits(nal):
    """The RBSP bits of an SPS without emulation prevention bytes (none occur here), up to the stop bit."""
    bits = "".join(f"{x:08b}" for x in nal)
    return bits[:bits.rindex("1")]


def test_sps_differs_only_in_max_num_ref_frames():
    for h, w in ((16, 16), (720, 960), (720, 480), (16 * 543, 16 * 64)):
        one, many = _rbsp_bits(video.sps(h, w)), _rbsp_bits(video.sps(h, w, 30))
        assert video.sps(h, w, 1) == video.sps(h, w) == O.sps(h, w)
        assert video.sps(h, w, 2) == video.sps(h, w, 30) == R.sps(h, w, 7)
        # bits 32..36: seq_parameter_set_id, log2_max_frame_num_minus4, pic_order_cnt_type 2; then ue(0) -> ue(1)
        assert one[32:38] == "110111" and many[:37] + many[40:] == one[:37] + one[38:] and many[37:40] == "010"


def _stbl(blob):
    top = _boxes(blob)
    find = lambda boxes, *path: find([c for c in boxes if c[0] == path[0]][0][3], *path[1:]) if len(path) > 1 \
        else [c for c in boxes if c[0] == path[0]][0]
    stbl = find(top, b"moov", b"trak", b"mdia", b"minf", b"stbl")
    return [c[0] for c in stbl[3]], {c[0]: blob[c[1]:c[2]] for c in stbl[3]}


def test_mp4_has_stss_exactly_when_gop_above_1():
    samples = [b"\x00\x00\x00\x02\x65\x88"] + [b"\x00\x00\x00\x02\x41\x9a"] * 6
    assert video.mp4_bytes(samples, 32, 48, 30, gop=1) == video.mp4_bytes(samples, 32, 48, 30)
    kinds, _ = _stbl(video.mp4_bytes(samples, 32, 48, 30))
    assert b"stss" not in kinds
    for gop, want in ((3, [1, 4, 7]), (2, [1, 3, 5, 7]), (7, [1]), (30, [1])):
        blob = video.mp4_bytes(samples, 32, 48, 30, gop=gop)
        kinds, body = _stbl(blob)
        assert kinds == [b"stsd", b"stts", b"stss", b"stsc", b"stsz", b"stco"]
        n = struct.unpack(">I", body[b"stss"][4:8])[0]
        assert list(struct.unpack(f">{n}I", body[b"stss"][8:])) == want
        assert video.sps(32, 48, gop) in body[b"stsd"] and video.sps(32, 48) not in body[b"stsd"]


def test_bad_gop_raises_value_error():
    f = np.zeros((2, 16, 16, 3), np.uint8)
    for gop in (0, -1, 2.0, True, "3", None):
        with pytest.raises(ValueError):
            video._gop(gop)
        with pytest.raises(ValueError):
            video.mp4_bytes([b"\x00"], 16, 16, 30, gop=gop)
        with pytest.raises(ValueError):
            video.sps(16, 16, gop)
        with pytest.raises(ValueError):
            video.max_bytes(16, 16, gop)
    # the gop check comes before the input checks, so even a CPU tensor fails on the gop
    for gop in (0, 2.0, True):
        with pytest.raises(ValueError, match="gop must be"):
            video.encode(torch.zeros(2, 16, 16, 3, dtype=torch.uint8), gop=gop)
        with pytest.raises(ValueError, match="gop must be"):
            video.write_mp4(torch.as_tensor(f), "unused.mp4", gop=gop)


@pytest.mark.parametrize("gop", [5, 6, 2 ** 31 - 1, 2 ** 32 + 2, 2 ** 64])
def test_encode_passes_at_most_the_clip_length_as_gop(gop, monkeypatch):
    """Any gop >= T codes a clip as one GOP (the bytes of gop = T): video.encode hands the library min(gop, T), a
    32-bit int, and sizes the reconstruction workspace for it; the slots still follow the Python gop's bound."""
    from pantomatrix_b200 import ops, slots
    seen = {}

    def record(frames, clip_len, qp, data, nbytes, scratch, sizes, gop=1, recon=None):
        seen.update(clip_len=clip_len, gop=gop, recon=None if recon is None else tuple(recon.shape),
                    cap=data.shape[1], slice_cap=scratch.shape[2])

    monkeypatch.setattr(slots, "frames", lambda f: (f.reshape(-1, *f.shape[-3:]), f.shape[1]))
    monkeypatch.setattr(ops, "h264_encode", record)
    video.encode(torch.zeros(3, 5, 32, 48, 3, dtype=torch.uint8), gop=gop)
    assert seen["clip_len"] == 5 and seen["gop"] == 5 and seen["recon"] == (3, 2, 24 * 48)
    assert seen["cap"] == video.slot_bytes(32, 48, 2) and seen["slice_cap"] == video.slice_bytes(48, 2)


def test_ops_h264_gop_wrapper_marshals_valid_arguments(monkeypatch):
    """ops.h264_encode(..., gop=7) with the library call replaced by a recorder: every argument converts to its
    declared ctypes type, pm_h264_encode_gop gets gop, the workspace and its row stride, and gather follows."""
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
    frames = torch.zeros(20, 32, 48, 3, dtype=torch.uint8)
    cap, sc = video.slot_bytes(32, 48, 7), video.slice_bytes(48, 7)
    data, nbytes = torch.zeros(20, cap, dtype=torch.uint8), torch.zeros(20, dtype=torch.int64)
    scratch, sizes = torch.zeros(20, 2, sc, dtype=torch.uint8), torch.zeros(20, 2, dtype=torch.int32)
    recon = torch.zeros(2 * 2, 2, 24 * 48, dtype=torch.uint8)          # 2 clips of 10 frames: 2 GOPs each
    ops.h264_encode(frames, 10, 20, data, nbytes, scratch, sizes, gop=7, recon=recon)
    assert [c[0] for c in calls] == ["pm_memset_async", "pm_h264_encode_gop", "pm_h264_gather"]
    by = dict(calls)
    assert by["pm_memset_async"][1:3] == (0, 20 * cap)
    assert by["pm_h264_encode_gop"][1:7] == (32 * 48 * 3, 20, 10, 32, 48, 20)
    assert by["pm_h264_encode_gop"][7:13] == (scratch.data_ptr(), sc, sizes.data_ptr(), 7, recon.data_ptr(), 24 * 48)
    assert by["pm_h264_gather"][3:6] == (scratch.data_ptr(), sc, sizes.data_ptr())
    assert by["pm_h264_gather"][6:9] == (data.data_ptr(), cap, nbytes.data_ptr())

"""The FLAC encoding rule on the CPU (oracle/flac_oracle.py, DESIGN.md section 13): its MP4 files decode with FFmpeg's
own flac decoder (driven through ctypes, CRC-16 checked) to the input samples exactly, with the rate, channels,
STREAMINFO MD5 and frame sizes right and every frame within the bound; OpenCV still decodes the video track of the
same file; the box tree and the chunk interleave; and the ops wrapper's ctypes arguments.  The GPU's bytes are
compared with these in tests/test_flac_gpu.py."""
import ctypes
import glob
import os
import struct

import numpy as np
import pytest
import torch

from oracle import flac_oracle as O
from oracle import h264_oracle as H
from pantomatrix_b200 import audio_io, flac, video

# ---- FFmpeg's libraries, as bundled with opencv-python-headless ----

_AV = {}


def _av():
    """(libavformat, libavcodec, libavutil) loaded with ctypes from the OpenCV wheel, or skip."""
    if not _AV:
        cv2 = pytest.importorskip("cv2")
        libs = os.path.join(os.path.dirname(os.path.dirname(cv2.__file__)), "opencv_python_headless.libs")
        found = {k: glob.glob(os.path.join(libs, f"lib{k}-*.so*")) for k in ("avformat", "avcodec", "avutil")}
        if not all(found.values()):
            pytest.skip("FFmpeg's shared libraries are not bundled with this OpenCV")
        _AV.update({k: ctypes.CDLL(v[0]) for k, v in found.items()})
        fmt, codec, util = _AV["avformat"], _AV["avcodec"], _AV["avutil"]
        P, I = ctypes.c_void_p, ctypes.c_int
        for lib, name, res, args in (
                (fmt, "avformat_open_input", I, [ctypes.POINTER(P), ctypes.c_char_p, P, P]),
                (fmt, "avformat_find_stream_info", I, [P, P]),
                (fmt, "av_find_best_stream", I, [P, I, I, I, P, I]),
                (fmt, "av_read_frame", I, [P, P]),
                (fmt, "avformat_close_input", None, [ctypes.POINTER(P)]),
                (codec, "avcodec_find_decoder_by_name", P, [ctypes.c_char_p]),
                (codec, "avcodec_alloc_context3", P, [P]),
                (codec, "avcodec_parameters_to_context", I, [P, P]),
                (codec, "avcodec_open2", I, [P, P, P]),
                (codec, "avcodec_send_packet", I, [P, P]),
                (codec, "avcodec_receive_frame", I, [P, P]),
                (codec, "avcodec_free_context", None, [ctypes.POINTER(P)]),
                (codec, "av_packet_alloc", P, []),
                (codec, "av_packet_unref", None, [P]),
                (codec, "av_packet_free", None, [ctypes.POINTER(P)]),
                (util, "av_frame_alloc", P, []),
                (util, "av_frame_free", None, [ctypes.POINTER(P)]),
                (util, "av_opt_set", I, [P, ctypes.c_char_p, ctypes.c_char_p, I]),
                (util, "av_opt_get_int", I, [P, ctypes.c_char_p, I, ctypes.POINTER(ctypes.c_int64)]),
                (util, "av_opt_get_chlayout", I, [P, ctypes.c_char_p, I, P])):
            fn = getattr(lib, name)
            fn.restype, fn.argtypes = res, args
    return _AV["avformat"], _AV["avcodec"], _AV["avutil"]


AVERROR_EOF = -0x20464F45                    # FFERRTAG('E','O','F',' ')
AVERROR_EAGAIN = -11
S16, S32, S16P, S32P = 1, 2, 6, 7            # AVSampleFormat


def decode_audio(path):
    """(samples (n, C) int64, rate) of the audio track of path, by FFmpeg's flac decoder with CRC checks on.  Any
    decoding error fails the test."""
    fmt, codec, util = _av()
    ctx = ctypes.c_void_p()
    assert fmt.avformat_open_input(ctypes.byref(ctx), path.encode(), None, None) == 0
    try:
        assert fmt.avformat_find_stream_info(ctx, None) >= 0
        idx = fmt.av_find_best_stream(ctx, 1, -1, -1, None, 0)          # AVMEDIA_TYPE_AUDIO
        assert idx >= 0
        streams = ctypes.c_void_p.from_address(ctx.value + 48).value        # AVFormatContext.streams
        st = ctypes.c_void_p.from_address(streams + 8 * idx).value
        par = ctypes.c_void_p.from_address(st + 16).value                   # AVStream.codecpar
        dec = codec.avcodec_find_decoder_by_name(b"flac")
        assert dec
        cc = ctypes.c_void_p(codec.avcodec_alloc_context3(dec))
        assert codec.avcodec_parameters_to_context(cc, par) >= 0
        assert util.av_opt_set(cc, b"err_detect", b"crccheck+explode", 0) >= 0
        assert codec.avcodec_open2(cc, dec, None) == 0
        pkt, frm = ctypes.c_void_p(codec.av_packet_alloc()), ctypes.c_void_p(util.av_frame_alloc())
        out = []

        def drain():
            while True:
                r = codec.avcodec_receive_frame(cc, frm)
                if r in (AVERROR_EAGAIN, AVERROR_EOF):
                    return
                assert r == 0, r
                ns = ctypes.c_int.from_address(frm.value + 112).value           # AVFrame.nb_samples
                sf = ctypes.c_int.from_address(frm.value + 116).value           # AVFrame.format
                ext = ctypes.c_void_p.from_address(frm.value + 96).value        # AVFrame.extended_data
                nch = out_ch[0]
                dt = np.int16 if sf in (S16, S16P) else np.int32
                if sf in (S16P, S32P):
                    planes = [np.ctypeslib.as_array(ctypes.cast(ctypes.c_void_p.from_address(ext + 8 * c).value,
                                                                ctypes.POINTER(ctypes.c_int16 if dt == np.int16
                                                                               else ctypes.c_int32)), (ns,))
                              for c in range(nch)]
                    a = np.stack(planes, 1).astype(np.int64)
                else:
                    assert sf in (S16, S32), sf
                    p = ctypes.cast(ctypes.c_void_p.from_address(ext).value,
                                    ctypes.POINTER(ctypes.c_int16 if dt == np.int16 else ctypes.c_int32))
                    a = np.ctypeslib.as_array(p, (ns * nch,)).reshape(ns, nch).astype(np.int64)
                if dt == np.int32:
                    assert not (a & 0xFF).any()                     # 24-bit samples left-aligned in s32
                    a >>= 8
                out.append(a)

        out_ch = [0]
        while fmt.av_read_frame(ctx, pkt) >= 0:
            if ctypes.c_int.from_address(pkt.value + 36).value == idx:          # AVPacket.stream_index
                if not out_ch[0]:
                    lay = (ctypes.c_int * 8)()
                    assert util.av_opt_get_chlayout(cc, b"ch_layout", 0, lay) >= 0
                    out_ch[0] = lay[1]                                          # AVChannelLayout.nb_channels
                assert codec.avcodec_send_packet(cc, pkt) == 0
                drain()
            codec.av_packet_unref(pkt)
        assert codec.avcodec_send_packet(cc, None) == 0
        drain()
        rate = ctypes.c_int64()
        assert util.av_opt_get_int(cc, b"ar", 0, ctypes.byref(rate)) >= 0
        codec.av_packet_free(ctypes.byref(pkt))
        util.av_frame_free(ctypes.byref(frm))
        codec.avcodec_free_context(ctypes.byref(cc))
    finally:
        fmt.avformat_close_input(ctypes.byref(ctx))
    return np.concatenate(out), rate.value


# ---- the files ----

def _boxes(b, at=0, end=None):
    """The box tree of an ISO BMFF byte string as {type: [(payload start, end, children)]}, containers opened."""
    end = len(b) if end is None else end
    out = []
    containers = {b"moov", b"trak", b"mdia", b"minf", b"dinf", b"stbl"}
    while at < end:
        size, kind = struct.unpack(">I4s", b[at:at + 8])
        assert size >= 8 and at + size <= end
        out.append((kind, at + 8, at + size, _boxes(b, at + 8, at + size) if kind in containers else []))
        at += size
    assert at == end
    return out


def _find(boxes, *path):
    hits = [c for c in boxes if c[0] == path[0]]
    return hits if len(path) == 1 else [x for h in hits for x in _find(h[3], *path[1:])]


VIDEO = [np.random.default_rng(1).integers(0, 256, (16, 32, 3), dtype=np.uint8) for _ in range(3)]


def clip_file(pcm, rate, tmp_path, frames=None, fps=30):
    """(path, frames, assignments) of an MP4 of the oracle's FLAC of pcm beside a few oracle H.264 frames."""
    frames_, chans = O.encode(pcm, rate)
    info = O.streaminfo(pcm, rate, frames_)
    video_frames = VIDEO if frames is None else frames
    samples = [H.encode(f, 20, i)[0] for i, f in enumerate(video_frames)]
    h, w = video_frames[0].shape[:2]
    path = str(tmp_path / "clip.mp4")
    with open(path, "wb") as f:
        f.write(video.mp4_bytes(samples, h, w, fps, audio=(frames_, info)))
    return path, frames_, chans


def native_file(frames, info, path):
    """A native FLAC file: the stream marker, STREAMINFO as the last metadata block, the frames."""
    with open(path, "wb") as f:
        f.write(b"fLaC" + bytes([0x80, 0, 0, 34]) + info + b"".join(frames))
    return str(path)


def check_clip(pcm, rate, tmp_path):
    """Decode the oracle's MP4 and native FLAC files; check samples, rate, channels, STREAMINFO and the bound; return
    the assignments.  FFmpeg's MP4 demuxer reads a track whose samples all last one tick as raw PCM chunks, so a
    one-sample clip is decoded from the native file only."""
    path, frames, chans = clip_file(pcm, rate, tmp_path)
    paths = [native_file(frames, O.streaminfo(pcm, rate, frames), tmp_path / "clip.flac")]
    for p in paths + ([path] if len(pcm) > 1 else []):
        got, got_rate = decode_audio(p)
        assert got_rate == rate and got.shape == pcm.shape
        assert np.array_equal(got, pcm.astype(np.int64))
    blob = open(path, "rb").read()
    top = _boxes(blob)
    dfla = _find(top, b"moov", b"trak", b"mdia", b"minf", b"stbl", b"stsd")[1]
    at = blob.index(b"dfLa", dfla[1]) + 8
    assert blob[at:at + 4] == bytes([0x80, 0, 0, 34])
    info = blob[at + 4:at + 38]
    bps = O.check(pcm, rate)
    assert info[16 + 2:] == O.md5(pcm, bps) == flac.md5(pcm, bps)
    sizes = [len(f) for f in frames]
    assert int.from_bytes(info[4:7], "big") == min(sizes) and int.from_bytes(info[7:10], "big") == max(sizes)
    assert flac.parse_streaminfo(info) == (rate, pcm.shape[1], bps, len(pcm))
    assert info == flac.streaminfo(pcm, rate, sizes)
    for k, f in enumerate(frames):
        bs = min(O.BLOCK, len(pcm) - k * O.BLOCK)
        assert len(f) <= flac.max_frame_bytes(pcm.shape[1], bps, bs) == O.max_frame_bytes(pcm.shape[1], bps, bs)
    cv2 = pytest.importorskip("cv2")
    cap = cv2.VideoCapture(path, cv2.CAP_FFMPEG)
    cap.set(cv2.CAP_PROP_CONVERT_RGB, 0)
    lumas = []
    while True:
        ok, fr = cap.read()
        if not ok:
            break
        lumas.append(np.asarray(fr).reshape(-1)[:16 * 32].reshape(16, 32))
    cap.release()
    assert len(lumas) == len(VIDEO)
    for i, (f, y) in enumerate(zip(VIDEO, lumas)):
        assert np.array_equal(y, H.encode(f, 20, i)[1][0]), i
    return chans


# ---- cases, shared with the GPU test ----

def speech(n, rate, seed=0):
    """Tones with a slow envelope plus noise, int16."""
    rng = np.random.default_rng(seed)
    t = np.arange(n) / rate
    x = sum(a * np.sin(2 * np.pi * f * t + ph) for a, f, ph in ((6000, 180, 0.3), (3000, 450, 1.1), (1500, 1230, 2)))
    x = x * (0.6 + 0.4 * np.sin(2 * np.pi * 3 * t)) + rng.normal(0, 200, n)
    return np.clip(np.round(x), -32768, 32767).astype(np.int16)[:, None]


def stereo(kind, n=5000, seed=3):
    """Stereo clips built to win one channel assignment each: a is smooth, d small noise."""
    rng = np.random.default_rng(seed)
    a = np.round(12000 * np.sin(2 * np.pi * 200 * np.arange(n) / 48000)).astype(np.int64)
    d = rng.integers(-200, 201, n)
    l, r = {O.INDEPENDENT: (a, rng.integers(-32768, 32768, n)),     # R noise: S and M cost more than R
            O.LEFT_SIDE: (a, a + d),                                 # S = -d is cheaper than R, L than M
            O.SIDE_RIGHT: (a + d, a),
            O.MID_SIDE: (a + d, a - d)}[kind]                        # M = a, S = 2 d
    return np.stack([l, r], 1).clip(-32768, 32767).astype(np.int16)


def cases():
    """(name, pcm, rate) cases."""
    rng = np.random.default_rng(7)
    noise16 = lambda n, c: rng.integers(-32768, 32768, (n, c)).astype(np.int16)
    out = [("speech_16k", speech(3 * 4096 + 1, 16000), 16000),
           ("silence", np.zeros((5000, 1), np.int16), 16000),
           ("noise", noise16(4096, 1), 16000),
           ("alternating", np.tile(np.array([-32768, 32767], np.int16), 2500)[:, None], 16000),
           ("pcm24", np.round(speech(6000, 48000, 2).astype(np.float64) * 200.3).astype(np.int32), 48000),
           ("pcm24_noise", rng.integers(-(1 << 23), 1 << 23, (4100, 2)).astype(np.int32), 48000),
           ("eight_channels", np.concatenate([speech(5000, 44100, s) for s in range(7)]
                                             + [noise16(5000, 1)], 1), 44100)]
    for n in (1, 15, 4095, 4096, 4097, 3 * 4096 + 1):
        out.append((f"n{n}", speech(n, 22050, n), 22050))
    for rate in (8000, 11025, 12000, 16000, 22050, 24000, 32000, 44100, 48000, 65535):
        out.append((f"rate{rate}", speech(4500, rate, rate), rate))
    for kind, name in ((O.INDEPENDENT, "independent"), (O.LEFT_SIDE, "left_side"), (O.SIDE_RIGHT, "side_right"),
                       (O.MID_SIDE, "mid_side")):
        out.append((f"stereo_{name}", stereo(kind), 48000))
    return out


@pytest.mark.parametrize("name,pcm,rate", cases(), ids=[c[0] for c in cases()])
def test_oracle_clips_decode_to_the_input(name, pcm, rate, tmp_path):
    chans = check_clip(pcm, rate, tmp_path)
    if name in ("silence", "noise"):                     # first subframe type: CONSTANT / VERBATIM
        frames, _ = O.encode(pcm, rate)
        for k, f in enumerate(frames):
            at = len(O.header(k, min(O.BLOCK, len(pcm) - k * O.BLOCK), rate, 0, 16))
            assert f[at] >> 1 == (0 if name == "silence" else 1)
    want = {"stereo_independent": O.INDEPENDENT, "stereo_left_side": O.LEFT_SIDE, "stereo_side_right": O.SIDE_RIGHT,
            "stereo_mid_side": O.MID_SIDE}.get(name)
    if want is not None:
        assert chans[0] == want, chans


def test_rate_codes_take_every_branch():
    for rate, code, tail in ((8000, 4, b""), (16000, 5, b""), (22050, 6, b""), (24000, 7, b""), (32000, 8, b""),
                             (44100, 9, b""), (48000, 10, b""), (12000, 12, b"\x0c"), (49000, 12, b"\x31"),
                             (11025, 13, struct.pack(">H", 11025)), (65535, 13, b"\xff\xff")):
        h = O.header(0, 4096, rate, 0, 16)
        assert h[2] == 0xC0 | code and h[5:-1] == tail, rate
    h = O.header(40000, 100, 11025, 9, 24)             # frame number in 3 bytes, block size and rate in the header
    assert h[2] == 0x7D and h[3] == 0x9C and h[4:7] == O.utf8(40000) and len(O.utf8(40000)) == 3
    assert h[7:9] == struct.pack(">H", 99) and h[9:11] == struct.pack(">H", 11025) and len(h) == 12
    assert O.crc8(h[:-1]) == h[-1]
    # the longest header the rule writes: 4 + 4 (frame numbers below 2^21 cover 2^31 samples) + 2 + 2 + 1 bytes
    assert len(O.header((1 << 31) // 4096, 7, 11025, 7, 24)) == 13 <= 16


def test_utf8_frame_numbers():
    for v, want in ((0, b"\x00"), (0x7F, b"\x7f"), (0x80, b"\xc2\x80"), (0x7FF, b"\xdf\xbf"),
                    (0x800, b"\xe0\xa0\x80"), (0xFFFF, b"\xef\xbf\xbf"), (0x10000, b"\xf0\x90\x80\x80")):
        assert O.utf8(v) == want


def test_crcs_match_the_formats_check_values():
    assert O.crc8(b"123456789") == 0xF4 and O.crc16(b"123456789") == 0xFEE8


def test_inputs_are_checked():
    ok = np.zeros((10, 2), np.int16)
    for bad, rate in ((np.zeros((10, 9), np.int16), 8000), (np.zeros((0, 1), np.int16), 8000), (ok, 0),
                      (ok, 65536), (np.zeros((4, 1), np.float32), 8000),
                      (np.full((4, 1), 1 << 23, np.int32), 8000)):
        with pytest.raises(ValueError):
            O.check(bad, rate)
    for rate in (0, 65536, 8000.0, True):
        with pytest.raises(ValueError):
            flac._rate(rate)
    with pytest.raises(ValueError):
        flac.encode(torch.zeros(10, 2, dtype=torch.int16), 8000)                   # CPU tensor
    with pytest.raises(ValueError):
        flac.encode(np.zeros((10, 2), np.int16), 8000)                               # not a tensor


def test_track_samples_from_read_pcm(tmp_path):
    """16-bit stays int16; 8- and 24-bit become their exact 24-bit values, float is clamped and rounded."""
    def wav(path, tag, bits, raw, ch=1):
        fmt = struct.pack("<HHIIHH", tag, ch, 8000, 8000 * ch * bits // 8, ch * bits // 8, bits)
        with open(path, "wb") as f:
            f.write(b"RIFF" + struct.pack("<I", 36 + len(raw)) + b"WAVE" + b"fmt " + struct.pack("<I", 16) + fmt
                    + b"data" + struct.pack("<I", len(raw)) + raw)
        return str(path)

    v16 = np.array([-32768, -1, 0, 1, 32767], "<i2")
    x, _ = audio_io.read_pcm(wav(tmp_path / "a.wav", 1, 16, v16.tobytes()))
    assert audio_io.track_samples(x).dtype == np.int16 and np.array_equal(audio_io.track_samples(x)[:, 0], v16)
    v24 = np.array([-(1 << 23), -1, 0, 1, (1 << 23) - 1, 123456], np.int64)
    raw = b"".join(int(v & 0xFFFFFF).to_bytes(3, "little") for v in v24)
    x, _ = audio_io.read_pcm(wav(tmp_path / "b.wav", 1, 24, raw))
    t = audio_io.track_samples(x)
    assert t.dtype == np.int32 and np.array_equal(t[:, 0], v24)
    v8 = np.array([0, 1, 127, 128, 255], np.uint8)
    x, _ = audio_io.read_pcm(wav(tmp_path / "c.wav", 1, 8, v8.tobytes()))
    assert np.array_equal(audio_io.track_samples(x)[:, 0], (v8.astype(np.int64) - 128) << 16)
    f = np.array([-2.0, -1.0, 0.5 / (1 << 23), 1.5 / (1 << 23), 1.0, 3.0], "<f4")
    x, _ = audio_io.read_pcm(wav(tmp_path / "d.wav", 3, 32, f.tobytes()))
    assert audio_io.track_samples(x)[:, 0].tolist() == [-(1 << 23), -(1 << 23), 0, 2, (1 << 23) - 1, (1 << 23) - 1]


def test_mp4_box_tree_and_chunk_interleave():
    rng = np.random.default_rng(4)
    pcm = rng.integers(-30, 30, (3 * 4096 + 100, 2)).astype(np.int16)
    rate, fps = 8000, 2                                # 4096-sample frames start at 0, 0.512, 1.024 and 1.536 s
    frames, _ = O.encode(pcm, rate)
    info = O.streaminfo(pcm, rate, frames)
    samples = [bytes([0, 0, 0, 1, 0x65]) * (i + 1) for i in range(5)]     # 2.5 s of video at 2 fps
    blob = video.mp4_bytes(samples, 16, 32, fps, audio=(frames, info))
    top = _boxes(blob)
    assert [t[0] for t in top] == [b"ftyp", b"moov", b"mdat"]
    traks = _find(top, b"moov", b"trak")
    assert len(traks) == 2
    stbl = [{c[0]: blob[c[1]:c[2]] for c in _find(t[3], b"mdia", b"minf", b"stbl")[0][3]} for t in traks]
    assert list(stbl[1]) == [b"stsd", b"stts", b"stsc", b"stsz", b"stco"]
    assert struct.unpack(">IIIIII", stbl[1][b"stts"][:24]) == (0, 2, 3, 4096, 1, 100)
    # seconds: video 0, 1 | audio 0, 1 | video 2, 3 | audio 2, 3 | video 4
    vstsc = struct.unpack(">II" + "III" * 2, stbl[0][b"stsc"])
    assert vstsc == (0, 2, 1, 2, 1, 3, 1, 1)
    assert struct.unpack(">IIIII", stbl[1][b"stsc"]) == (0, 1, 1, 2, 1)
    vco = struct.unpack(">II" + "I" * 3, stbl[0][b"stco"])[2:]
    aco = struct.unpack(">II" + "I" * 2, stbl[1][b"stco"])[2:]
    mdat = top[2]
    order = [(vco[0], samples[0] + samples[1]), (aco[0], frames[0] + frames[1]), (vco[1], samples[2] + samples[3]),
             (aco[1], frames[2] + frames[3]), (vco[2], samples[4])]
    assert vco[0] == mdat[1]
    for (at, want), nxt in zip(order, [o[0] for o in order[1:]] + [mdat[2]]):
        assert blob[at:nxt] == want
    mvhd = _find(top, b"moov", b"mvhd")[0]
    assert struct.unpack(">I", blob[mvhd[1] + 16:mvhd[1] + 20])[0] == 2500 == max(2500, len(pcm) * 1000 // rate)
    assert blob[mvhd[2] - 4:mvhd[2]] == struct.pack(">I", 3)
    mdhd = _find(traks[1][3], b"mdia", b"mdhd")[0]
    assert struct.unpack(">II", blob[mdhd[1] + 12:mdhd[1] + 20]) == (rate, len(pcm))
    entry = stbl[1][b"stsd"][8:]
    assert entry[4:8] == b"fLaC" and struct.unpack(">HHHHI", entry[24:36]) == (2, 16, 0, 0, rate << 16)
    assert _find(traks[1][3], b"mdia", b"hdlr") and b"soun" in blob[traks[1][1]:traks[1][2]]
    assert b"smhd" in blob[traks[1][1]:traks[1][2]]
    # audio=None is the silent file, byte for byte
    assert video.mp4_bytes(samples, 16, 32, fps) == video.mp4_bytes(samples, 16, 32, fps, audio=None)
    assert len(_find(_boxes(video.mp4_bytes(samples, 16, 32, fps)), b"moov", b"trak")) == 1
    with pytest.raises(ValueError):
        video.mp4_bytes(samples, 16, 32, fps, audio=(frames[:-1], info))


def test_ops_flac_wrapper_marshals_valid_arguments(monkeypatch):
    """ops.flac_encode with the library call replaced by a recorder: every argument converts to its declared ctypes
    type, the slots are cleared first, and the two stages share the records."""
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
    pcm = torch.zeros(3, 5000, 2, dtype=torch.int16)
    cap = flac.slot_bytes(2, 16)
    data, nbytes = torch.zeros(6, cap, dtype=torch.uint8), torch.zeros(6, dtype=torch.int64)
    rec = torch.zeros(24, flac.REC_WORDS, dtype=torch.int32)
    ops.flac_encode(pcm, 16, 48000, data, nbytes, rec)
    assert [c[0] for c in calls] == ["pm_memset_async", "pm_flac_analyse", "pm_flac_emit"]
    by = dict(calls)
    assert by["pm_memset_async"][1:3] == (0, 6 * cap)
    assert by["pm_flac_analyse"][1:6] == (10000, 3, 5000, 2, 16) and by["pm_flac_analyse"][6] == rec.data_ptr()
    assert by["pm_flac_emit"][1:7] == (10000, 3, 5000, 2, 16, 48000)
    assert by["pm_flac_emit"][7:11] == (rec.data_ptr(), data.data_ptr(), cap, nbytes.data_ptr())

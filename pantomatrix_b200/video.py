"""H.264 video of rendered frames, encoded on the GPU, muxed into MP4 on the host.

Each (H, W, 3) uint8 RGB frame (H, W multiples of 16) becomes one IDR access unit of a Constrained Baseline stream by
one fixed rule (DESIGN.md section 12, include/pm_emage.h pm_h264_*): BT.601 limited-range colour in integers, one I
slice per macroblock row with deblocking off, every macroblock Intra16x16 (DC or Horizontal luma, DC chroma) or I_PCM
when it would pass 3200 bits or need a level escape Baseline lacks, CAVLC, and each slice as one length-prefixed NAL
unit.  A frame's bytes depend only on the frame, qp and the parity of its index in its clip: the same frame gives the
same sample alone or in any batch at the same index parity.

    data, nbytes = video.encode(renderer.render_sequence(poses, expression, trans))   # (B*T, cap) uint8, (B*T,) int64
    video.write_mp4(frames[0], "out/clip.mp4", fps=30)                                 # one silent clip
    video.write_mp4(frames[0], "out/clip.mp4", fps=30, audio=(pcm, 48000))            # with a FLAC sound track

Deblocking is off, so a decoder's output is the encoder's reconstruction exactly.
"""
from __future__ import annotations

import struct
from fractions import Fraction

import torch

from . import flac, ops

MB_BITS_LIMIT = 3200                      # 128 + RawMbBits: the most bits one macroblock_layer() may take (A.3.1)
MAX_FS, MAX_DIM_MBS = 36864, 543          # level 5.1: MaxFS, and the most macroblocks in a row or column
SLICE_HEADER_BITS = 62                    # NAL header byte and the longest slice header this encoder writes


def _rbsp_bytes(w: int) -> int:
    """The most RBSP bytes of one slice: header, w / 16 macroblocks of at most 3200 bits, stop bit and alignment."""
    return (SLICE_HEADER_BITS + MB_BITS_LIMIT * (w // 16) + 8 + 7) // 8


def slice_bytes(w: int) -> int:
    """The most bytes of one length-prefixed slice: 4-byte length, the RBSP, at most one emulation prevention byte per
    two RBSP bytes (each needs two zero bytes before it)."""
    p = _rbsp_bytes(w)
    return 4 + p + p // 2


def max_bytes(h: int, w: int) -> int:
    """The size bound of one (h, w) frame's sample: h / 16 slices of at most slice_bytes(w)."""
    return (h // 16) * slice_bytes(w)


def slot_bytes(h: int, w: int) -> int:
    """Bytes of one output slot: max_bytes rounded up to a multiple of 4."""
    return (max_bytes(h, w) + 3) & ~3


def check_size(h: int, w: int) -> None:
    if h < 16 or w < 16 or h % 16 or w % 16:
        raise ValueError(f"frames: H and W must be positive multiples of 16, got {h} x {w}")
    if (h // 16) * (w // 16) > MAX_FS or h // 16 > MAX_DIM_MBS or w // 16 > MAX_DIM_MBS:
        raise ValueError(f"a {h} x {w} frame passes level 5.1's limits ({MAX_FS} macroblocks, {MAX_DIM_MBS} per side)")


def _qp(qp) -> int:
    if isinstance(qp, bool) or not isinstance(qp, int) or not 0 <= qp <= 51:
        raise ValueError(f"qp must be an int in 0..51, got {qp!r}")
    return qp


# ---- parameter sets, built on the host (the CPU restatement of the rule builds its own) ----

class _Bits:
    def __init__(self):
        self.bits = []

    def u(self, v, n):
        self.bits += [(v >> (n - 1 - i)) & 1 for i in range(n)]

    def ue(self, v):
        n = (v + 1).bit_length()
        self.u(v + 1, 2 * n - 1)

    def se(self, v):
        self.ue(2 * v - 1 if v > 0 else -2 * v)

    def nal(self):
        self.bits += [1] + [0] * (-(len(self.bits) + 1) % 8)
        raw = bytes(int("".join(map(str, self.bits[i:i + 8])), 2) for i in range(0, len(self.bits), 8))
        out, zeros = bytearray(), 0
        for b in raw:                                     # emulation prevention
            if zeros >= 2 and b <= 3:
                out.append(3)
                zeros = 0
            out.append(b)
            zeros = zeros + 1 if b == 0 else 0
        return bytes(out)


def sps(h: int, w: int) -> bytes:
    """Sequence parameter set NAL unit: Constrained Baseline, level 5.1, pic_order_cnt_type 2, no reference frames,
    and a VUI holding only the video signal type (limited range, SMPTE 170M primaries, transfer and matrix)."""
    check_size(h, w)
    b = _Bits()
    b.u(0x67, 8)                          # nal_ref_idc 3, nal_unit_type 7
    b.u(66, 8), b.u(0b11000000, 8), b.u(51, 8)   # profile_idc, constraint_set0/1, level_idc
    b.ue(0), b.ue(0), b.ue(2), b.ue(0)    # sps id, log2_max_frame_num_minus4, poc type, max_num_ref_frames
    b.u(0, 1)                             # gaps_in_frame_num_value_allowed_flag
    b.ue(w // 16 - 1), b.ue(h // 16 - 1)
    b.u(1, 1), b.u(1, 1), b.u(0, 1)       # frame_mbs_only, direct_8x8_inference, frame_cropping
    b.u(1, 1)                             # vui_parameters_present_flag
    b.u(0, 1), b.u(0, 1)                  # aspect ratio, overscan
    b.u(1, 1), b.u(5, 3), b.u(0, 1), b.u(1, 1)   # video signal type: unspecified format, limited range, colour
    b.u(6, 8), b.u(6, 8), b.u(6, 8)       # primaries, transfer, matrix: SMPTE 170M
    b.u(0, 1), b.u(0, 1), b.u(0, 1), b.u(0, 1), b.u(0, 1), b.u(0, 1)   # chroma loc, timing, hrd x2, pic_struct, restr.
    return b.nal()


def pps() -> bytes:
    """Picture parameter set NAL unit: CAVLC, pic_init_qp 26, deblocking_filter_control_present_flag 1."""
    b = _Bits()
    b.u(0x68, 8)
    b.ue(0), b.ue(0), b.u(0, 1), b.u(0, 1), b.ue(0), b.ue(0), b.ue(0), b.u(0, 1), b.u(0, 2)
    b.se(0), b.se(0), b.se(0)
    b.u(1, 1), b.u(0, 1), b.u(0, 1)
    return b.nal()


# ---- encoding on the GPU ----

def _frames(frames):
    if not torch.is_tensor(frames):
        raise ValueError(f"frames must be a tensor, got {type(frames).__name__}")
    if not frames.is_cuda:
        raise ValueError("frames must be a CUDA tensor")
    if frames.dtype != torch.uint8:
        raise ValueError(f"frames must be uint8, got {frames.dtype}")
    if frames.dim() not in (4, 5) or frames.shape[-1] != 3:
        raise ValueError(f"frames must be (N, H, W, 3) or (B, T, H, W, 3), got {tuple(frames.shape)}")
    h, w = frames.shape[-3:-1]
    check_size(h, w)
    if frames.stride(-1) != 1 or frames.stride(-2) != 3 or frames.stride(-3) != 3 * w:
        raise ValueError("frames: each frame must be dense")
    if frames.dim() == 5:
        b, t = frames.shape[:2]
        if b > 1 and t > 1 and frames.stride(0) != t * frames.stride(1):
            raise ValueError("frames (B, T, H, W, 3): the clips' frames must be evenly spaced")
        fs = frames.stride(1) if t > 1 else frames.stride(0)
        clip_len = t
        frames = frames.as_strided((b * t, h, w, 3), (fs, 3 * w, 3, 1))
    else:
        clip_len = frames.shape[0]
    if frames.shape[0] > 1 and frames.stride(0) < 3 * h * w:
        raise ValueError("frames: frames must not overlap")
    return frames, max(clip_len, 1)


@torch.no_grad()
def encode(frames, qp=20, out=None):
    """H.264 samples of frames (N, H, W, 3) or (B, T, H, W, 3) uint8 CUDA, each frame dense (a MeshRenderer result is
    read in place), H and W multiples of 16.  A frame's index in its clip (t, or n for (N, ...) input) sets its
    idr_pic_id (index mod 2).  Returns (data, nbytes): data (N, cap) uint8 holds sample i (its slices, each prefixed
    by its 4-byte big-endian length) in data[i, :nbytes[i]] (zeros after it), nbytes (N,) int64, both on the frames'
    device.  out: an optional (data, nbytes) pair to fill, data (N, cap) uint8 contiguous with cap >= slot_bytes(H, W)
    and a multiple of 4, nbytes (N,) int64 contiguous.  No host synchronisation; with out given the call can be
    captured in a CUDA graph.  Raises ValueError on a CPU tensor, a wrong dtype or shape, H or W not a multiple of 16,
    a frame past level 5.1, frames that are not dense, qp outside 0..51 or an out too small."""
    qp = _qp(qp)
    frames, clip_len = _frames(frames)
    n, h, w, _ = frames.shape
    dev = frames.device
    if out is None:
        data = torch.empty(n, slot_bytes(h, w), dtype=torch.uint8, device=dev)
        nbytes = torch.empty(n, dtype=torch.int64, device=dev)
    else:
        data, nbytes = out
        if not (torch.is_tensor(data) and data.device == dev and data.dtype == torch.uint8 and data.dim() == 2
                and data.shape[0] == n and data.shape[1] >= max_bytes(h, w) and data.shape[1] % 4 == 0
                and data.is_contiguous()):
            raise ValueError(f"out data must be a contiguous ({n}, cap) uint8 tensor on {dev} with cap >= "
                             f"{max_bytes(h, w)} a multiple of 4")
        if not (torch.is_tensor(nbytes) and nbytes.device == dev and nbytes.dtype == torch.int64
                and tuple(nbytes.shape) == (n,) and nbytes.is_contiguous()):
            raise ValueError(f"out nbytes must be a contiguous ({n},) int64 tensor on {dev}")
    if n == 0:
        return data, nbytes
    scratch = torch.empty(n, h // 16, slice_bytes(w), dtype=torch.uint8, device=dev)
    sizes = torch.empty(n, h // 16, dtype=torch.int32, device=dev)
    ops.h264_encode(frames, clip_len, qp, data, nbytes, scratch, sizes)
    return data, nbytes


# ---- MP4 (ISO BMFF) on the host ----

def _box(kind: bytes, *parts: bytes) -> bytes:
    body = b"".join(parts)
    return struct.pack(">I", 8 + len(body)) + kind + body


def _full(kind: bytes, version: int, flags: int, *parts: bytes) -> bytes:
    return _box(kind, struct.pack(">I", version << 24 | flags), *parts)


_MATRIX = struct.pack(">9i", 0x10000, 0, 0, 0, 0x10000, 0, 0, 0, 0x40000000)


def _chunks(sizes, starts):
    """stsc and stco payloads of one track from its chunks' sample counts and file offsets."""
    runs = []
    for i, k in enumerate(sizes):
        if not runs or runs[-1][1] != k:
            runs.append((i + 1, k))
    stsc = struct.pack(">I", len(runs)) + b"".join(struct.pack(">III", first, k, 1) for first, k in runs)
    return stsc, struct.pack(">I", len(starts)) + struct.pack(f">{len(starts)}I", *starts)


def _audio_trak(frames, info, movie_dur, stsc, stco):
    """The sound track: fLaC sample entry with its dfLa (STREAMINFO, last-block flag set), one sample per frame."""
    rate, channels, bps, total = flac.parse_streaminfo(info)
    n = len(frames)
    last = total - flac.BLOCK * (n - 1)
    runs = [(n, flac.BLOCK)] if last == flac.BLOCK else [(n - 1, flac.BLOCK), (1, last)] if n > 1 else [(1, last)]
    dfla = _full(b"dfLa", 0, 0, bytes([0x80, 0, 0, len(info)]), info)
    entry = _box(b"fLaC", bytes(6), struct.pack(">H", 1), bytes(8), struct.pack(">HHHHI", channels, bps, 0, 0,
                                                                                 rate << 16), dfla)
    stbl = _box(b"stbl",
                _full(b"stsd", 0, 0, struct.pack(">I", 1), entry),
                _full(b"stts", 0, 0, struct.pack(">I", len(runs)), *(struct.pack(">II", *r) for r in runs)),
                _full(b"stsc", 0, 0, stsc),
                _full(b"stsz", 0, 0, struct.pack(">II", 0, n), struct.pack(f">{n}I", *map(len, frames))),
                _full(b"stco", 0, 0, stco))
    minf = _box(b"minf", _full(b"smhd", 0, 0, bytes(4)),
                _box(b"dinf", _full(b"dref", 0, 0, struct.pack(">I", 1), _full(b"url ", 0, 1))), stbl)
    mdia = _box(b"mdia",
                _full(b"mdhd", 0, 0, struct.pack(">IIIIHH", 0, 0, rate, total, 0x55C4, 0)),
                _full(b"hdlr", 0, 0, bytes(4), b"soun", bytes(12), b"SoundHandler\0"), minf)
    tkhd = _full(b"tkhd", 0, 3, struct.pack(">IIIII", 0, 0, 2, 0, movie_dur), bytes(8),
                 struct.pack(">hhhH", 0, 0, 0x100, 0), _MATRIX, struct.pack(">II", 0, 0))
    return _box(b"trak", tkhd, mdia)


def mp4_bytes(samples, h: int, w: int, fps=30, audio=None) -> bytes:
    """An MP4 file of one H.264 video track: samples (a list of bytes-like, each a sample as encode() writes it), h x w
    frames at a constant fps.  ftyp, then moov (avc1 with its avcC holding the SPS and PPS, stts, stsc, stsz, stco, no
    stss: every sample is a sync sample), then mdat, so the file plays while it downloads.
    audio: None (a silent file), or (frames, info), a FLAC track: its frames (bytes-like, as flac.encode writes them)
    and their 34-byte STREAMINFO (flac.streaminfo).  The file then has a second track, and mdat holds one-second
    chunks: each second's video samples, then the audio frames that start in that second.
    Raises ValueError on no samples, fps <= 0 or a file that would pass 2^32 bytes."""
    check_size(h, w)
    if isinstance(fps, bool) or not isinstance(fps, (int, float, Fraction)) or not fps > 0:
        raise ValueError(f"fps must be a positive number, got {fps!r}")
    samples = [bytes(s) for s in samples]
    if not samples:
        raise ValueError("mp4_bytes needs at least one sample")
    rate = Fraction(fps).limit_denominator(1001)
    timescale, delta = rate.numerator, rate.denominator
    n = len(samples)
    media_dur = n * delta
    movie_dur = media_dur * 1000 // timescale
    if timescale >= 1 << 32 or media_dur >= 1 << 32 or movie_dur >= 1 << 32:
        raise ValueError(f"{n} frames at {fps} fps do not fit 32-bit MP4 durations")
    if audio is None:
        plan = [(0, list(range(n)))]                   # one chunk: every video sample
        sound, audio_dur = [], 0
    else:
        sound, info = [bytes(f) for f in audio[0]], bytes(audio[1])
        srate, _, _, total = flac.parse_streaminfo(info)
        if len(info) != 34 or not sound or len(sound) != flac.frames_of(total) or total >= 1 << 32:
            raise ValueError("audio must be (frames, STREAMINFO) of one FLAC clip of fewer than 2^32 samples")
        audio_dur = total * 1000 // srate
        second = {}
        for i in range(n):
            second.setdefault(i * delta // timescale, ([], []))[0].append(i)
        for k in range(len(sound)):
            second.setdefault(k * flac.BLOCK // srate, ([], []))[1].append(k)
        plan = [(t, idx) for s in sorted(second) for t, idx in enumerate(second[s]) if idx]
    movie = max(movie_dur, audio_dur)
    data = (samples, sound)
    s, p = sps(h, w), pps()
    avcc = _box(b"avcC", bytes([1, 66, 0xC0, 51, 0xFF, 0xE1]), struct.pack(">H", len(s)), s,
                bytes([1]), struct.pack(">H", len(p)), p)
    avc1 = _box(b"avc1", bytes(6), struct.pack(">H", 1), bytes(16), struct.pack(">HH", w, h),
                struct.pack(">II", 0x480000, 0x480000), bytes(4), struct.pack(">H", 1), bytes(32),
                struct.pack(">Hh", 0x18, -1), avcc)

    def moov(offset):
        starts, at = ([], []), offset
        for t, idx in plan:
            starts[t].append(at)
            at += sum(len(data[t][i]) for i in idx)
        tables = [_chunks([len(idx) for t, idx in plan if t == tr], starts[tr]) for tr in (0, 1)]
        stbl = _box(b"stbl",
                    _full(b"stsd", 0, 0, struct.pack(">I", 1), avc1),
                    _full(b"stts", 0, 0, struct.pack(">III", 1, n, delta)),
                    _full(b"stsc", 0, 0, tables[0][0]),
                    _full(b"stsz", 0, 0, struct.pack(">II", 0, n), struct.pack(f">{n}I", *map(len, samples))),
                    _full(b"stco", 0, 0, tables[0][1]))
        minf = _box(b"minf", _full(b"vmhd", 0, 1, bytes(8)),
                    _box(b"dinf", _full(b"dref", 0, 0, struct.pack(">I", 1), _full(b"url ", 0, 1))), stbl)
        mdia = _box(b"mdia",
                    _full(b"mdhd", 0, 0, struct.pack(">IIIIHH", 0, 0, timescale, media_dur, 0x55C4, 0)),
                    _full(b"hdlr", 0, 0, bytes(4), b"vide", bytes(12), b"VideoHandler\0"), minf)
        tkhd = _full(b"tkhd", 0, 3, struct.pack(">IIIII", 0, 0, 1, 0, movie_dur), bytes(8),
                     struct.pack(">hhhH", 0, 0, 0, 0), _MATRIX, struct.pack(">II", w << 16, h << 16))
        mvhd = _full(b"mvhd", 0, 0, struct.pack(">IIII", 0, 0, 1000, movie), struct.pack(">IH", 0x10000, 0x100),
                     bytes(10), _MATRIX, bytes(24), struct.pack(">I", 2 if audio is None else 3))
        traks = [_box(b"trak", tkhd, mdia)]
        if audio is not None:
            traks.append(_audio_trak(sound, info, audio_dur, *tables[1]))
        return _box(b"moov", mvhd, *traks)

    ftyp = _box(b"ftyp", b"isom", struct.pack(">I", 0x200), b"isomiso2avc1mp41")
    head = len(ftyp) + len(moov(0)) + 8
    total = head + sum(len(x) for x in samples) + sum(len(x) for x in sound)
    if total >= 1 << 32:
        raise ValueError(f"the file would take {total} bytes, past 2^32")
    body = b"".join(data[t][i] for t, idx in plan for i in idx)
    return ftyp + moov(head) + struct.pack(">I", 8 + total - head) + b"mdat" + body


def write_mp4(frames, path, fps=30, qp=20, audio=None):
    """Encode one clip (T, H, W, 3) uint8 CUDA frames and write it to path as an MP4 file.  audio: None (one silent
    video track), or (pcm, rate): pcm (n, C) CUDA int16 or int32 (24-bit) samples at rate Hz, coded as a FLAC track
    (flac.encode) and trimmed to the video's duration: the first min(n, floor(T rate / fps)) samples.  That matches
    ffmpeg's -shortest when the audio is the longer stream; shorter audio is kept whole, and the video plays on past
    its end in silence.  Both streams are encoded on the current stream; the sizes are read once (one
    synchronisation), only the encoded bytes (and the samples, for the MD5) are copied to pinned host memory, and
    the copies are waited for once.  Returns path."""
    if torch.is_tensor(frames) and frames.dim() != 4:
        raise ValueError(f"write_mp4 takes one clip (T, H, W, 3), got {tuple(frames.shape)}")
    if isinstance(fps, bool) or not isinstance(fps, (int, float, Fraction)) or not fps > 0:
        raise ValueError(f"fps must be a positive number, got {fps!r}")
    if audio is not None:
        pcm, rate = audio
        flac._rate(rate)
        if not torch.is_tensor(pcm) or pcm.dim() != 2:
            raise ValueError("write_mp4: audio must be (pcm (n, C) CUDA tensor, rate)")
        keep = min(pcm.shape[0], int(frames.shape[0] * rate / Fraction(fps).limit_denominator(1001)))
        if keep < 1:
            raise ValueError(f"write_mp4: {frames.shape[0]} frames at {fps} fps hold no sample at {rate} Hz")
        pcm = pcm[:keep]
    data, nbytes = encode(frames, qp=qp)
    h, w = frames.shape[1:3]
    if audio is None:
        sizes, sound_sizes = nbytes.tolist(), []
    else:
        adata, anbytes = flac.encode(pcm, rate)
        both = torch.cat([nbytes, anbytes]).tolist()
        sizes, sound_sizes = both[:len(nbytes)], both[len(nbytes):]
        if min(sound_sizes) < 0:
            raise ValueError("write_mp4: int32 audio samples must lie in -2^23 .. 2^23 - 1")
        host_pcm = torch.empty(pcm.shape, dtype=pcm.dtype, pin_memory=True)
        host_pcm.copy_(pcm, non_blocking=True)
    host = torch.empty(sum(sizes) + sum(sound_sizes), dtype=torch.uint8, pin_memory=True)
    at = 0
    for src, ks in ((data, sizes), (adata if audio is not None else None, sound_sizes)):
        for i, k in enumerate(ks):
            host[at:at + k].copy_(src[i, :k], non_blocking=True)
            at += k
    torch.cuda.current_stream(data.device).synchronize()
    flat = memoryview(host.numpy())
    pieces, at = [], 0
    for k in sizes + sound_sizes:
        pieces.append(flat[at:at + k])
        at += k
    track = None
    if audio is not None:
        track = (pieces[len(sizes):], flac.streaminfo(host_pcm, rate, sound_sizes))
    blob = mp4_bytes(pieces[:len(sizes)], h, w, fps, audio=track)
    with open(path, "wb") as f:
        f.write(blob)
    return path

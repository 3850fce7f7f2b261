"""H.264 video of rendered frames, encoded on the GPU, muxed into MP4 on the host.

Each (H, W, 3) uint8 RGB frame (H, W multiples of 16) becomes one IDR access unit of a Constrained Baseline stream by
one fixed rule (DESIGN.md section 12, include/pm_emage.h pm_h264_*): BT.601 limited-range colour in integers, one I
slice per macroblock row with deblocking off, every macroblock Intra16x16 (DC or Horizontal luma, DC chroma) or I_PCM
when it would pass 3200 bits or need a level escape Baseline lacks, CAVLC, and each slice as one length-prefixed NAL
unit.  A frame's bytes depend only on the frame, qp and the parity of its index in its clip: the same frame gives the
same sample alone or in any batch at the same index parity.  With a keyframe interval gop > 1 (encode(..., gop=30)),
every gop-th frame is an IDR frame and the frames between are P frames of P_Skip, zero-motion inter, Intra16x16 or
I_PCM macroblocks, each coded against the frame before it; a GOP's bytes depend only on its frames, qp, gop and the
parity of its index in the clip.  With a motion search range search > 0 (encode(..., gop=30, search=16)) the inter
macroblocks carry quarter-pel motion vectors searched against the whole previous frame.  With intra4x4=True
(encode(..., intra4x4=True)) any intra macroblock of an I or P slice may also be Intra 4x4 (I_NxN): its 16 4x4 blocks
each predicted by one of the nine modes from the reconstructed samples next to it, chosen by SAD and mode bits; off,
the default, every byte is as before.

    data, nbytes = video.encode(renderer.render_sequence(poses, expression, trans))   # (B*T, cap) uint8, (B*T,) int64
    video.write_mp4(frames[0], "out/clip.mp4", fps=30)                                 # one silent clip
    video.write_mp4(frames[0], "out/clip.mp4", fps=30, audio=(pcm, 48000))            # with a FLAC sound track

Deblocking is off, so a decoder's output is the encoder's reconstruction exactly.
"""
from __future__ import annotations

import struct
from fractions import Fraction

import torch

from . import flac, ops, slots

MB_BITS_LIMIT = 3200                      # 128 + RawMbBits: the most bits one macroblock_layer() may take (A.3.1)
MAX_FS, MAX_DIM_MBS = 36864, 543          # level 5.1: MaxFS, and the most macroblocks in a row or column
SLICE_HEADER_BITS = 62                    # NAL header byte and the slice header, as the gop = 1 bound counts it
SLICE_HEADER_BITS_GOP = 70                # the longest slice header of either kind: IDR, last row, qp 0
RECON_ROW_BYTES = 24                      # reconstruction bytes per pixel column of a row: 16 Y + 4 Cb + 4 Cr
MAX_SEARCH = 32                           # the widest motion search range, in whole pixels


def _rbsp_bytes(w: int, gop: int = 1) -> int:
    """The most RBSP bytes of one slice: header, w / 16 macroblocks, stop bit and alignment.  gop 1: at most 3200
    bits per macroblock.  gop > 1: at most 3201, a macroblock_layer() of at most 3200 bits after its 1-bit ue(0)
    mb_skip_run; a run of r >= 1 skipped macroblocks takes at most 2 log2(r + 1) + 1 <= 3 r bits, and I_PCM 9 + 7 +
    3072."""
    if gop == 1:
        return (SLICE_HEADER_BITS + MB_BITS_LIMIT * (w // 16) + 8 + 7) // 8
    return (SLICE_HEADER_BITS_GOP + (MB_BITS_LIMIT + 1) * (w // 16) + 8 + 7) // 8


def slice_bytes(w: int, gop: int = 1) -> int:
    """The most bytes of one length-prefixed slice: 4-byte length, the RBSP, at most one emulation prevention byte per
    two RBSP bytes (each needs two zero bytes before it)."""
    p = _rbsp_bytes(w, _gop(gop))
    return 4 + p + p // 2


def max_bytes(h: int, w: int, gop=1) -> int:
    """The size bound of one (h, w) frame's sample: h / 16 slices of at most slice_bytes(w, gop)."""
    return (h // 16) * slice_bytes(w, gop)


def slot_bytes(h: int, w: int, gop=1) -> int:
    """Bytes of one output slot: max_bytes rounded up to a multiple of 4."""
    return (max_bytes(h, w, gop) + 3) & ~3


def check_size(h: int, w: int) -> None:
    if h < 16 or w < 16 or h % 16 or w % 16:
        raise ValueError(f"frames: H and W must be positive multiples of 16, got {h} x {w}")
    if (h // 16) * (w // 16) > MAX_FS or h // 16 > MAX_DIM_MBS or w // 16 > MAX_DIM_MBS:
        raise ValueError(f"a {h} x {w} frame passes level 5.1's limits ({MAX_FS} macroblocks, {MAX_DIM_MBS} per side)")


def _qp(qp) -> int:
    if isinstance(qp, bool) or not isinstance(qp, int) or not 0 <= qp <= 51:
        raise ValueError(f"qp must be an int in 0..51, got {qp!r}")
    return qp


def _gop(gop) -> int:
    if isinstance(gop, bool) or not isinstance(gop, int) or gop < 1:
        raise ValueError(f"gop must be an int >= 1, got {gop!r}")
    return gop


def _search(search) -> int:
    if isinstance(search, bool) or not isinstance(search, int) or not 0 <= search <= MAX_SEARCH:
        raise ValueError(f"search must be an int in 0..{MAX_SEARCH}, got {search!r}")
    return search


def _intra4x4(intra4x4) -> bool:
    if not isinstance(intra4x4, bool):
        raise ValueError(f"intra4x4 must be a bool, got {intra4x4!r}")
    return intra4x4


def _fps(fps) -> Fraction:
    """The frame rate as the MP4 file states it: timescale / sample duration, a denominator of at most 1001."""
    if isinstance(fps, bool) or not isinstance(fps, (int, float, Fraction)) or not fps > 0:
        raise ValueError(f"fps must be a positive number, got {fps!r}")
    return Fraction(fps).limit_denominator(1001)


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


def sps(h: int, w: int, gop=1) -> bytes:
    """Sequence parameter set NAL unit: Constrained Baseline, level 5.1, pic_order_cnt_type 2, no reference frames
    (one when gop > 1: each P frame references the frame before it), and a VUI holding only the video signal type
    (limited range, SMPTE 170M primaries, transfer and matrix)."""
    check_size(h, w)
    gop = _gop(gop)
    b = _Bits()
    b.u(0x67, 8)                          # nal_ref_idc 3, nal_unit_type 7
    b.u(66, 8), b.u(0b11000000, 8), b.u(51, 8)   # profile_idc, constraint_set0/1, level_idc
    b.ue(0), b.ue(0), b.ue(2), b.ue(int(gop > 1))   # sps id, log2_max_frame_num_minus4, poc type, max_num_ref_frames
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

@torch.no_grad()
def encode(frames, qp=20, out=None, gop=1, search=0, intra4x4=False):
    """H.264 samples of frames (N, H, W, 3) or (B, T, H, W, 3) uint8 CUDA, each frame dense (a MeshRenderer result is
    read in place), H and W multiples of 16.  gop: frames per group of pictures.  Frame t of a clip (t, or n for
    (N, ...) input) is an IDR frame with idr_pic_id (t div gop) mod 2 when t mod gop == 0, else a P frame coded
    against frame t - 1 (P_Skip, zero-motion inter, Intra16x16 or I_PCM macroblocks); gop 1 makes every frame IDR,
    and any gop >= T codes each clip as one GOP (the bytes of gop = T).  A GOP's bytes depend only on its frames, qp,
    gop and the parity of t div gop.  search: the motion search range in whole pixels, 0..32.  0 codes P frames with
    zero motion; search > 0 gives their inter macroblocks the quarter-pel vector of the lowest SAD + lambda(qp) x
    vector bits within +-search pixels of zero, against the whole previous frame (DESIGN.md section 12).  It trades
    encode time for size and changes no SPS, PPS or MP4 box; with gop 1 (or T = 1) there are no P frames and the
    output is the gop 1 output.  intra4x4: also code intra macroblocks as Intra 4x4 (I_NxN) where its cost
    J4 + 6 lambda(qp) is below the Intra16x16 SAD (DESIGN.md section 12); the SPS, PPS, MP4 boxes and size bounds are
    unchanged, and False gives the bytes of the rule without it.  Returns (data, nbytes): data (N, cap) uint8 holds sample i (its slices, each
    prefixed by its 4-byte big-endian length) in data[i, :nbytes[i]] (zeros after it), nbytes (N,) int64, both on the
    frames' device.  out: an optional (data, nbytes) pair to fill, data (N, cap) uint8 contiguous with
    cap >= slot_bytes(H, W, gop) and a multiple of 4, nbytes (N,) int64 contiguous.  No host synchronisation; with
    out given the call can be captured in a CUDA graph.  Raises ValueError on a CPU tensor, a wrong dtype or shape,
    H or W not a multiple of 16, a frame past level 5.1, frames that are not dense, qp outside 0..51, gop not an int
    >= 1, search not an int in 0..32, intra4x4 not a bool or an out too small (cap >= slot_bytes(H, W, gop))."""
    qp, gop, search, intra4x4 = _qp(qp), _gop(gop), _search(search), _intra4x4(intra4x4)
    frames, clip_len = slots.frames(frames)
    n, h, w, _ = frames.shape
    check_size(h, w)
    dev = frames.device
    data, nbytes = slots.output(n, max_bytes(h, w, gop), slot_bytes(h, w, gop), dev, out)
    if n == 0:
        return data, nbytes
    scratch = torch.empty(n, h // 16, slice_bytes(w, gop), dtype=torch.uint8, device=dev)
    sizes = torch.empty(n, h // 16, dtype=torch.int32, device=dev)
    # a gop past the clip length gives the gop = T bytes (the same idr_pic_id and frame_num); the kernel takes at most T
    kgop = min(gop, clip_len)
    recon = None
    i4 = {"intra4x4": True} if intra4x4 else {}         # without the switch the call is exactly as before
    chains = n // clip_len * -(-clip_len // kgop)
    if kgop > 1 and search > 0:           # two whole-frame reconstructions per GOP, and frame k's vectors
        recon = torch.empty(chains, 3 * h * w, dtype=torch.uint8, device=dev)
        mv = torch.empty(chains, h // 16, w // 16, 2, dtype=torch.int16, device=dev)
        ops.h264_encode(frames, clip_len, qp, data, nbytes, scratch, sizes, gop=kgop, recon=recon, search=search,
                        mv=mv, **i4)
        return data, nbytes
    if kgop > 1:                          # one macroblock row's reconstruction per (GOP, row), updated frame by frame
        recon = torch.empty(chains, h // 16, RECON_ROW_BYTES * w, dtype=torch.uint8, device=dev)
    ops.h264_encode(frames, clip_len, qp, data, nbytes, scratch, sizes, gop=kgop, recon=recon, **i4)
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


def _trak(track_id, duration, volume, size, timescale, media_dur, handler, media_header, entry, stts, sample_sizes,
          chunks, sync=None):
    """One track: tkhd (its duration in movie ticks, volume, size (w, h)), then mdia: mdhd (timescale and duration),
    hdlr (handler: type and name), and minf holding the media header box, dinf with its dref, and stbl: stsd with the
    sample entry, the stts payload, stss of the sync sample numbers (sync; none when sync is None), the stsc and stco
    payloads of _chunks (chunks), stsz of the samples' sizes."""
    n = len(sample_sizes)
    stsc, stco = chunks
    stbl = _box(b"stbl",
                _full(b"stsd", 0, 0, struct.pack(">I", 1), entry),
                _full(b"stts", 0, 0, stts),
                *([] if sync is None else [_full(b"stss", 0, 0, struct.pack(f">I{len(sync)}I", len(sync), *sync))]),
                _full(b"stsc", 0, 0, stsc),
                _full(b"stsz", 0, 0, struct.pack(">II", 0, n), struct.pack(f">{n}I", *sample_sizes)),
                _full(b"stco", 0, 0, stco))
    minf = _box(b"minf", media_header,
                _box(b"dinf", _full(b"dref", 0, 0, struct.pack(">I", 1), _full(b"url ", 0, 1))), stbl)
    kind, name = handler
    mdia = _box(b"mdia",
                _full(b"mdhd", 0, 0, struct.pack(">IIIIHH", 0, 0, timescale, media_dur, 0x55C4, 0)),
                _full(b"hdlr", 0, 0, bytes(4), kind, bytes(12), name), minf)
    w, h = size
    tkhd = _full(b"tkhd", 0, 3, struct.pack(">IIIII", 0, 0, track_id, 0, duration), bytes(8),
                 struct.pack(">hhhH", 0, 0, volume, 0), _MATRIX, struct.pack(">II", w << 16, h << 16))
    return _box(b"trak", tkhd, mdia)


def mp4_bytes(samples, h: int, w: int, fps=30, audio=None, gop=1) -> bytes:
    """An MP4 file of one H.264 video track: samples (a list of bytes-like, each a sample as encode() writes it), h x w
    frames at a constant fps, encoded with keyframe interval gop.  ftyp, then moov (avc1 with its avcC holding the SPS
    (sps(h, w, gop)) and PPS, stts, stsc, stsz, stco; with gop 1 no stss, as every sample is a sync sample, else an
    stss listing the IDR samples 1, 1 + gop, ...), then mdat, so the file plays while it downloads.
    audio: None (a silent file), or (frames, info), a FLAC track: its frames (bytes-like, as flac.encode writes them)
    and their 34-byte STREAMINFO (flac.streaminfo).  The file then has a second track, and mdat holds one-second
    chunks: each second's video samples, then the audio frames that start in that second.
    Raises ValueError on no samples, fps <= 0 or a file that would pass 2^32 bytes."""
    check_size(h, w)
    rate = _fps(fps)
    gop = _gop(gop)
    samples = [bytes(s) for s in samples]
    if not samples:
        raise ValueError("mp4_bytes needs at least one sample")
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
        srate, channels, bps, pcm_n = flac.parse_streaminfo(info)
        if len(info) != 34 or not sound or len(sound) != flac.frames_of(pcm_n) or pcm_n >= 1 << 32:
            raise ValueError("audio must be (frames, STREAMINFO) of one FLAC clip of fewer than 2^32 samples")
        audio_dur = pcm_n * 1000 // srate
        # one sample per FLAC frame: fLaC sample entry with its dfLa (STREAMINFO, last-block flag set)
        nf, last = len(sound), pcm_n - flac.BLOCK * (len(sound) - 1)
        runs = ([(nf, flac.BLOCK)] if last == flac.BLOCK
                else [(nf - 1, flac.BLOCK), (1, last)] if nf > 1 else [(1, last)])
        dfla = _full(b"dfLa", 0, 0, bytes([0x80, 0, 0, len(info)]), info)
        fla = _box(b"fLaC", bytes(6), struct.pack(">H", 1), bytes(8),
                   struct.pack(">HHHHI", channels, bps, 0, 0, srate << 16), dfla)
        sound_stts = struct.pack(">I", len(runs)) + b"".join(struct.pack(">II", *r) for r in runs)
        second = {}
        for i in range(n):
            second.setdefault(i * delta // timescale, ([], []))[0].append(i)
        for k in range(len(sound)):
            second.setdefault(k * flac.BLOCK // srate, ([], []))[1].append(k)
        plan = [(t, idx) for s in sorted(second) for t, idx in enumerate(second[s]) if idx]
    movie = max(movie_dur, audio_dur)
    data = (samples, sound)
    s, p = sps(h, w, gop), pps()
    avcc = _box(b"avcC", bytes([1, 66, 0xC0, 51, 0xFF, 0xE1]), struct.pack(">H", len(s)), s,
                bytes([1]), struct.pack(">H", len(p)), p)
    avc1 = _box(b"avc1", bytes(6), struct.pack(">H", 1), bytes(16), struct.pack(">HH", w, h),
                struct.pack(">II", 0x480000, 0x480000), bytes(4), struct.pack(">H", 1), bytes(32),
                struct.pack(">Hh", 0x18, -1), avcc)

    sync = None if gop == 1 else list(range(1, n + 1, gop))

    def moov(offset):
        starts, at = ([], []), offset
        for t, idx in plan:
            starts[t].append(at)
            at += sum(len(data[t][i]) for i in idx)
        tables = [_chunks([len(idx) for t, idx in plan if t == tr], starts[tr]) for tr in (0, 1)]
        mvhd = _full(b"mvhd", 0, 0, struct.pack(">IIII", 0, 0, 1000, movie), struct.pack(">IH", 0x10000, 0x100),
                     bytes(10), _MATRIX, bytes(24), struct.pack(">I", 2 if audio is None else 3))
        traks = [_trak(1, movie_dur, 0, (w, h), timescale, media_dur, (b"vide", b"VideoHandler\0"),
                       _full(b"vmhd", 0, 1, bytes(8)), avc1, struct.pack(">III", 1, n, delta),
                       [len(x) for x in samples], tables[0], sync)]
        if audio is not None:
            traks.append(_trak(2, audio_dur, 0x100, (0, 0), srate, pcm_n, (b"soun", b"SoundHandler\0"),
                               _full(b"smhd", 0, 0, bytes(4)), fla, sound_stts, [len(x) for x in sound], tables[1]))
        return _box(b"moov", mvhd, *traks)

    ftyp = _box(b"ftyp", b"isom", struct.pack(">I", 0x200), b"isomiso2avc1mp41")
    head = len(ftyp) + len(moov(0)) + 8
    total = head + sum(len(x) for x in samples) + sum(len(x) for x in sound)
    if total >= 1 << 32:
        raise ValueError(f"the file would take {total} bytes, past 2^32")
    body = b"".join(data[t][i] for t, idx in plan for i in idx)
    return ftyp + moov(head) + struct.pack(">I", 8 + total - head) + b"mdat" + body


def write_mp4(frames, path, fps=30, qp=20, audio=None, gop=1, search=0, intra4x4=False):
    """Encode one clip (T, H, W, 3) uint8 CUDA frames with keyframe interval gop, motion search range search and the
    Intra 4x4 switch intra4x4 (encode) and write it to path as an MP4 file.  audio: None (one silent video track), or (pcm, rate): pcm (n, C) CUDA int16 or int32 (24-bit) samples
    at rate Hz, coded as a FLAC track (flac.encode) and trimmed to the video's duration: the first
    min(n, floor(T rate / fps)) samples.  That matches ffmpeg's -shortest when the audio is the longer stream; shorter
    audio is kept whole, and the video plays on past its end in silence.  Both streams are encoded on the current
    stream; the sizes are read once (one synchronisation), only the encoded bytes (and the samples, for the MD5) are
    copied to pinned host memory, and the copies are waited for once.  Returns path."""
    if torch.is_tensor(frames) and frames.dim() != 4:
        raise ValueError(f"write_mp4 takes one clip (T, H, W, 3), got {tuple(frames.shape)}")
    frame_rate = _fps(fps)
    gop, search, intra4x4 = _gop(gop), _search(search), _intra4x4(intra4x4)
    if audio is not None:
        pcm, rate = audio
        flac._rate(rate)
        if not torch.is_tensor(pcm) or pcm.dim() != 2:
            raise ValueError("write_mp4: audio must be (pcm (n, C) CUDA tensor, rate)")
        keep = min(pcm.shape[0], int(frames.shape[0] * rate / frame_rate))
        if keep < 1:
            raise ValueError(f"write_mp4: {frames.shape[0]} frames at {fps} fps hold no sample at {rate} Hz")
        pcm = pcm[:keep]
    data, nbytes = encode(frames, qp=qp, gop=gop, search=search, intra4x4=intra4x4)
    h, w = frames.shape[1:3]
    if audio is None:
        (pieces,) = slots.to_host((data, nbytes.tolist()))
        track = None
    else:
        adata, anbytes = flac.encode(pcm, rate)
        both = torch.cat([nbytes, anbytes]).tolist()
        sizes, sound_sizes = both[:len(nbytes)], both[len(nbytes):]
        if min(sound_sizes) < 0:
            raise ValueError("write_mp4: int32 audio samples must lie in -2^23 .. 2^23 - 1")
        host_pcm = torch.empty(pcm.shape, dtype=pcm.dtype, pin_memory=True)
        host_pcm.copy_(pcm, non_blocking=True)          # done by the time to_host's one synchronisation returns
        pieces, sound = slots.to_host((data, sizes), (adata, sound_sizes))
        track = (sound, flac.streaminfo(host_pcm, rate, sound_sizes))
    blob = mp4_bytes(pieces, h, w, fps, audio=track, gop=gop)
    with open(path, "wb") as f:
        f.write(blob)
    return path

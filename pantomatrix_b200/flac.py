"""FLAC audio of recorded samples, encoded on the GPU, for the MP4 files of pantomatrix_b200/video.py.

A clip (n, C) of int16 (coded at 16 bits) or int32 within -2^23 .. 2^23 - 1 (coded at 24 bits) becomes frames of 4096
samples (the last may be shorter) by one fixed rule (DESIGN.md section 13, include/pm_emage.h pm_flac_*): per channel
the exact smallest of CONSTANT, FIXED orders 0..4 with partitioned Rice residuals, and VERBATIM; for stereo the
smallest of independent, left/side, side/right and mid/side.  A clip's frames depend only on its samples, channel
count, bits per sample and rate: the same clip gives the same bytes alone or in any batch.

    data, nbytes = flac.encode(pcm, 48000)              # (B*F, cap) uint8, (B*F,) int64
    info = flac.streaminfo(host_pcm, 48000, sizes)      # 34-byte STREAMINFO for the dfLa box

The format is lossless: a decoder returns the samples exactly.
"""
from __future__ import annotations

import hashlib
import struct

import numpy as np
import torch

from . import ops

BLOCK = 4096                 # samples per frame (fixed blocking)
MAX_CHANNELS = 8
MAX_RATE = 65535             # the 16.16 samplerate field of the MP4 audio sample entry
REC_WORDS = 66               # int32 words of one analysis record (include/pm_emage.h)


def frames_of(n: int) -> int:
    """Frames of an n-sample clip."""
    return (n + BLOCK - 1) // BLOCK


def max_frame_bytes(channels: int, bps: int, n: int = BLOCK) -> int:
    """The size bound of one frame of n samples: a header of at most 16 bytes, C independent VERBATIM subframes of
    8 + bps n bits (the rule's exact minimum never passes them), padding and CRC-16: 18 + ceil(C (8 + bps n) / 8)."""
    return 18 + (channels * (8 + bps * n) + 7) // 8


def slot_bytes(channels: int, bps: int, n: int = BLOCK) -> int:
    """Bytes of one output slot: max_frame_bytes rounded up to a multiple of 4."""
    return (max_frame_bytes(channels, bps, n) + 3) & ~3


def _rate(rate) -> int:
    if isinstance(rate, bool) or not isinstance(rate, int) or not 1 <= rate <= MAX_RATE:
        raise ValueError(f"rate must be an int in 1..{MAX_RATE} Hz (the MP4 sample entry's 16.16 field), "
                         f"got {rate!r}")
    return rate


def bps_of(dtype) -> int:
    """16 for int16 samples, 24 for int32 ones."""
    if dtype in (torch.int16, np.int16):
        return 16
    if dtype in (torch.int32, np.int32):
        return 24
    raise ValueError(f"samples must be int16 (16-bit) or int32 (24-bit), got {dtype}")


def _pcm(pcm):
    if not torch.is_tensor(pcm):
        raise ValueError(f"pcm must be a tensor, got {type(pcm).__name__}")
    if not pcm.is_cuda:
        raise ValueError("pcm must be a CUDA tensor")
    bps = bps_of(pcm.dtype)
    if pcm.dim() not in (2, 3):
        raise ValueError(f"pcm must be (n, C) or (B, n, C), got {tuple(pcm.shape)}")
    if pcm.dim() == 2:
        pcm = pcm[None]
    b, n, c = pcm.shape
    if n < 1 or not 1 <= c <= MAX_CHANNELS:
        raise ValueError(f"pcm needs n >= 1 samples and 1..{MAX_CHANNELS} channels, got {tuple(pcm.shape)}")
    if n >= 1 << 31:
        raise ValueError(f"a clip of {n} samples is past 2^31 - 1")
    if (c > 1 and pcm.stride(2) != 1) or (n > 1 and pcm.stride(1) != c):
        raise ValueError("pcm: each clip's samples must be dense (n, C)")
    if b > 1 and pcm.stride(0) < n * c:
        raise ValueError("pcm: clips must not overlap")
    return pcm, bps


@torch.no_grad()
def encode(pcm, rate, out=None):
    """FLAC frames of pcm (n, C) or (B, n, C) CUDA int16 (16-bit) or int32 (24-bit, values in -2^23 .. 2^23 - 1), each
    clip dense, clips any stride apart, 1..8 channels, at rate Hz.  Returns (data, nbytes): data (B F, cap) uint8 holds
    frame k of clip b in data[b F + k, :nbytes[b F + k]] (zeros after it), F = ceil(n / 4096), nbytes (B F,) int64,
    both on pcm's device.  An int32 frame holding a value outside the 24-bit range is not coded: its nbytes is -1.
    out: an optional (data, nbytes) pair to fill, data (B F, cap) uint8 contiguous with cap >= max_frame_bytes(C, bps,
    min(n, 4096)) a multiple of 4, nbytes (B F,) int64 contiguous.  No host synchronisation; with out given the call
    can be captured in a CUDA graph.  Raises ValueError on a CPU tensor, a wrong dtype or shape, a rate outside
    1..65535, clips that are not dense or an out too small."""
    rate = _rate(rate)
    pcm, bps = _pcm(pcm)
    b, n, c = pcm.shape
    f = frames_of(n)
    dev = pcm.device
    need = max_frame_bytes(c, bps, min(n, BLOCK))
    if out is None:
        data = torch.empty(b * f, slot_bytes(c, bps, min(n, BLOCK)), dtype=torch.uint8, device=dev)
        nbytes = torch.empty(b * f, dtype=torch.int64, device=dev)
    else:
        data, nbytes = out
        if not (torch.is_tensor(data) and data.device == dev and data.dtype == torch.uint8 and data.dim() == 2
                and data.shape[0] == b * f and data.shape[1] >= need and data.shape[1] % 4 == 0
                and data.is_contiguous()):
            raise ValueError(f"out data must be a contiguous ({b * f}, cap) uint8 tensor on {dev} with cap >= "
                             f"{need} a multiple of 4")
        if not (torch.is_tensor(nbytes) and nbytes.device == dev and nbytes.dtype == torch.int64
                and tuple(nbytes.shape) == (b * f,) and nbytes.is_contiguous()):
            raise ValueError(f"out nbytes must be a contiguous ({b * f},) int64 tensor on {dev}")
    if b > 65535 or f * (4 if c == 2 else c) >= 1 << 31:
        raise ValueError(f"{b} clips of {f} frames are past the launch grid")
    rec = torch.empty(b * f * (4 if c == 2 else c), REC_WORDS, dtype=torch.int32, device=dev)
    ops.flac_encode(pcm, bps, rate, data, nbytes, rec)
    return data, nbytes


def md5(pcm, bps: int) -> bytes:
    """MD5 of host samples (n, C) as FLAC defines it: interleaved, little-endian, bps / 8 bytes each."""
    a = np.ascontiguousarray(np.asarray(pcm))
    if bps == 16:
        return hashlib.md5(a.astype("<i2", copy=False).tobytes()).digest()
    b = a.astype("<i4", copy=False).view(np.uint8).reshape(-1, 4)[:, :3]
    return hashlib.md5(np.ascontiguousarray(b).tobytes()).digest()


def streaminfo(pcm, rate: int, sizes) -> bytes:
    """The 34-byte STREAMINFO block body of one clip: pcm (n, C) host samples (NumPy or CPU tensor, int16 or int32),
    sizes its frames' byte counts.  Block size 4096 (min = max), the exact min and max frame sizes, rate, channels,
    bits per sample, total samples and the samples' MD5."""
    rate = _rate(rate)
    if torch.is_tensor(pcm):
        pcm = pcm.numpy()
    bps = bps_of(pcm.dtype)
    n, c = pcm.shape
    sizes = [int(s) for s in sizes]
    if len(sizes) != frames_of(n) or min(sizes) < 1:
        raise ValueError(f"streaminfo: {n} samples need {frames_of(n)} coded frames, got sizes {sizes[:4]}...")
    v = rate << 44 | (c - 1) << 41 | (bps - 1) << 36 | n
    return (struct.pack(">HH", BLOCK, BLOCK) + min(sizes).to_bytes(3, "big") + max(sizes).to_bytes(3, "big")
            + v.to_bytes(8, "big") + md5(pcm, bps))


def parse_streaminfo(info: bytes):
    """(rate, channels, bits per sample, total samples) of a STREAMINFO block body."""
    v = int.from_bytes(info[10:18], "big")
    return v >> 44, (v >> 41 & 7) + 1, (v >> 36 & 31) + 1, v & ((1 << 36) - 1)

"""CPU restatement of the FLAC encoding rule of pantomatrix_b200/flac.py (DESIGN.md section 13, include/pm_emage.h
pm_flac_*), in NumPy.  Written from the FLAC format description, not from the GPU code: the tests require the GPU's
frames to equal these byte for byte, and FFmpeg's flac decoder to return the input from these exactly.

A clip's frames depend only on its samples (n, C), the bits per sample (16 or 24) and the rate.
"""
from __future__ import annotations

import hashlib
import struct

import numpy as np

BLOCK = 4096
MAX_P = 8
KMAX = (14, 30)                  # largest Rice parameter of method 00 (4-bit) and 01 (5-bit): 15 / 31 are escapes
RATE_CODES = {8000: 4, 16000: 5, 22050: 6, 24000: 7, 32000: 8, 44100: 9, 48000: 10}
CONSTANT, FIXED, VERBATIM = 0, 1, 2
INDEPENDENT, LEFT_SIDE, SIDE_RIGHT, MID_SIDE = 1, 8, 9, 10      # stereo channel assignment codes


def max_frame_bytes(channels: int, bps: int, n: int = BLOCK) -> int:
    """18 + ceil(C (8 + bps n) / 8): a header of at most 16 bytes, independent VERBATIM subframes, CRC-16."""
    return 18 + (channels * (8 + bps * n) + 7) // 8


# ---- bits ----

def pack(fields) -> bytes:
    """MSB-first bit string of fields [(values, widths)] (arrays or scalars, widths may be 0 or > 32 for zero runs)."""
    vals = np.concatenate([np.atleast_1d(np.asarray(v, np.int64)) for v, _ in fields])
    wid = np.concatenate([np.atleast_1d(np.asarray(w, np.int64)) * np.ones_like(np.atleast_1d(np.asarray(v)),
                                                                              np.int64) for v, w in fields])
    total = int(wid.sum())
    owner = np.repeat(np.arange(len(wid)), wid)
    pos = np.arange(total) - np.repeat(np.cumsum(wid) - wid, wid)
    shift = wid[owner] - 1 - pos
    bits = np.where(shift < 63, (vals[owner] >> np.minimum(shift, 62)) & 1, 0).astype(np.uint8)
    bits = np.concatenate([bits, np.zeros(-total % 8, np.uint8)])
    return np.packbits(bits).tobytes()


def _crc(data: bytes, poly: int, width: int) -> int:
    top, mask, c = 1 << (width - 1), (1 << width) - 1, 0
    table = []
    for b in range(256):
        r = b << (width - 8)
        for _ in range(8):
            r = ((r << 1) ^ poly) & mask if r & top else (r << 1) & mask
        table.append(r)
    for b in data:
        c = ((c << 8) & mask) ^ table[((c >> (width - 8)) ^ b) & 0xFF]
    return c


def crc8(data: bytes) -> int:
    return _crc(data, 0x07, 8)


def crc16(data: bytes) -> int:
    return _crc(data, 0x8005, 16)


def utf8(v: int) -> bytes:
    """The frame number in FLAC's UTF-8-like coding."""
    if v < 0x80:
        return bytes([v])
    n = 2
    while v >= 1 << (5 * n + 1):
        n += 1
    out = [0x80 | (v >> (6 * i) & 0x3F) for i in range(n - 1)][::-1]
    return bytes([(0xFF00 >> n) & 0xFF | v >> (6 * (n - 1))] + out)


def header(k: int, bs: int, rate: int, chan: int, bps: int) -> bytes:
    """Frame header of frame k (block size bs) with its CRC-8."""
    bcode = 12 if bs == BLOCK else 7
    if rate in RATE_CODES:
        rcode, tail = RATE_CODES[rate], b""
    elif rate % 1000 == 0 and rate // 1000 < 256:
        rcode, tail = 12, bytes([rate // 1000])
    else:
        rcode, tail = 13, struct.pack(">H", rate)
    h = bytes([0xFF, 0xF8, bcode << 4 | rcode, chan << 4 | (4 if bps == 16 else 6) << 1]) + utf8(k)
    h += (struct.pack(">H", bs - 1) if bcode == 7 else b"") + tail
    return h + bytes([crc8(h)])


# ---- subframes ----

def residuals(x: np.ndarray, order: int) -> np.ndarray:
    """FIXED predictor residual e[i], i = order .. n - 1."""
    e = x.astype(np.int64)
    for _ in range(order):
        e = e[1:] - e[:-1]
    return e


def best_subframe(x: np.ndarray, bps: int):
    """(bits, kind, order, p, method, params) of the exact smallest subframe of x at bps bits, ties to the earlier
    candidate (CONSTANT, FIXED 0..4, VERBATIM), then the lower order, p and k."""
    n = len(x)
    if (x == x[0]).all():
        return 8 + bps, CONSTANT, 0, 0, 0, []
    best = (8 + bps * n, VERBATIM, 0, 0, 0, [])
    ks = np.arange(31, dtype=np.int64)
    pmax = 0
    while pmax < MAX_P and n % (2 << pmax) == 0:
        pmax += 1
    fixed = None
    for order in range(min(4, n) + 1):
        e = residuals(x, order)
        u = np.concatenate([np.zeros(order, np.int64), (e << 1) ^ (e >> 63)])   # zigzag; warm-up slots count 0
        sums = (u[:, None] >> ks[None]).reshape(1 << pmax, -1, 31).sum(1)          # (partitions, k) at pmax
        choice = None
        for p in range(pmax, -1, -1):
            s = n >> p
            if s >= order:
                count = np.full(1 << p, s, np.int64)
                count[0] -= order
                cost = count[:, None] * (ks[None] + 1) + sums
                per = []
                for m in (0, 1):
                    c = cost[:, :KMAX[m] + 1]
                    per.append((int((c.min(1) + 4 + m).sum()), c.argmin(1)))
                m = 1 if per[1][0] < per[0][0] else 0
                cand = (6 + per[m][0], p, m, per[m][1].tolist())
                if choice is None or cand[0] <= choice[0]:       # walking p downwards: ties go to the lower p
                    choice = cand
            if p:
                sums = sums.reshape(-1, 2, 31).sum(1)
        bits = 8 + order * bps + choice[0]
        if fixed is None or bits < fixed[0]:
            fixed = (bits, FIXED, order) + choice[1:]
    return fixed if fixed[0] <= best[0] else best


def subframe_fields(x: np.ndarray, bps: int, sub):
    _, kind, order, p, method, params = sub
    mask = (1 << bps) - 1
    if kind == CONSTANT:
        return [(0, 8), (int(x[0]) & mask, bps)]
    if kind == VERBATIM:
        return [(1 << 1, 8), (x.astype(np.int64) & mask, bps)]
    f = [((8 | order) << 1, 8), (x[:order].astype(np.int64) & mask, bps), (method, 2), (p, 4)]
    e = residuals(x, order)
    u = (e << 1) ^ (e >> 63)
    s = len(x) >> p
    at = 0
    for j, k in enumerate(params):
        cnt = s - (order if j == 0 else 0)
        uj = u[at:at + cnt]
        at += cnt
        q = uj >> k
        f.append((k, 4 + method))
        # each code: q zeros, then a one and the k low bits
        v = np.stack([np.zeros_like(q), (1 << k) | (uj & ((1 << k) - 1))], 1).reshape(-1)
        w = np.stack([q, np.full_like(q, k + 1)], 1).reshape(-1)
        f.append((v, w))
    return f


def frame(pcm: np.ndarray, k: int, rate: int, bps: int):
    """(bytes, channel assignment) of frame k of pcm (n, C)."""
    blk = pcm[k * BLOCK:(k + 1) * BLOCK].astype(np.int64)
    bs, c = blk.shape
    if c == 2:
        l, r = blk[:, 0], blk[:, 1]
        chans = {"L": (l, bps), "R": (r, bps), "S": (l - r, bps + 1), "M": ((l + r) >> 1, bps)}
        subs = {name: best_subframe(x, b) for name, (x, b) in chans.items()}
        pairs = [(INDEPENDENT, "LR"), (LEFT_SIDE, "LS"), (SIDE_RIGHT, "SR"), (MID_SIDE, "MS")]
        chan, names = min(pairs, key=lambda a: subs[a[1][0]][0] + subs[a[1][1]][0])   # min keeps the first of ties
        parts = [(chans[nm][0], chans[nm][1], subs[nm]) for nm in names]
    else:
        chan = c - 1
        parts = [(blk[:, i], bps, best_subframe(blk[:, i], bps)) for i in range(c)]
    fields = []
    for x, b, sub in parts:
        fields += subframe_fields(x, b, sub)
    body = header(k, bs, rate, chan, bps) + pack(fields)
    body += struct.pack(">H", crc16(body))
    return body, chan


def check(pcm: np.ndarray, rate: int) -> int:
    """The bits per sample of pcm (n, C) int16 (16) or int32 (24); ValueError on anything the rule does not take."""
    if pcm.ndim != 2 or not 1 <= pcm.shape[1] <= 8 or pcm.shape[0] < 1:
        raise ValueError(f"pcm must be (n >= 1, C in 1..8), got {pcm.shape}")
    if not 1 <= rate <= 65535:
        raise ValueError(f"rate must be in 1..65535 Hz, got {rate}")
    if pcm.dtype == np.int16:
        return 16
    if pcm.dtype == np.int32 and pcm.min() >= -(1 << 23) and pcm.max() < 1 << 23:
        return 24
    raise ValueError("pcm must be int16, or int32 within -2^23 .. 2^23 - 1")


def encode(pcm: np.ndarray, rate: int):
    """(frames: list of bytes, channel assignments) of a clip pcm (n, C)."""
    bps = check(pcm, rate)
    out = [frame(pcm, k, rate, bps) for k in range((len(pcm) + BLOCK - 1) // BLOCK)]
    return [f for f, _ in out], [c for _, c in out]


def md5(pcm: np.ndarray, bps: int) -> bytes:
    """MD5 of the samples interleaved, little-endian, bps / 8 bytes each."""
    b = np.ascontiguousarray(pcm.astype("<i4")).view(np.uint8).reshape(-1, 4)[:, :bps // 8]
    return hashlib.md5(np.ascontiguousarray(b).tobytes()).digest()


def streaminfo(pcm: np.ndarray, rate: int, frames) -> bytes:
    """The 34-byte STREAMINFO block body."""
    bps = check(pcm, rate)
    n, c = pcm.shape
    sizes = [len(f) for f in frames]
    v = rate << 44 | (c - 1) << 41 | (bps - 1) << 36 | n
    return (struct.pack(">HH", BLOCK, BLOCK) + min(sizes).to_bytes(3, "big") + max(sizes).to_bytes(3, "big")
            + v.to_bytes(8, "big") + md5(pcm, bps))

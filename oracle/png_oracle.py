"""CPU restatement of the PNG encoding rule of pantomatrix_b200.png (DESIGN.md section 11) (TEST / MEASUREMENT
INFRASTRUCTURE; never imported by the product).

Each (H, W, 3) uint8 frame becomes one PNG file:
  - scanlines: filter type 1 (Sub) on every row, S = the H * s filtered bytes, s = 3 W + 1;
  - parse: per row, greedily at each position p, the longest match over the candidate distances DISTANCES(s) (valid when
    1 <= d <= min(p, 32768), length <= min(258, row end - p), overlap allowed), the first distance in the list that
    reaches it; a match of length >= 3 is emitted, otherwise the literal S[p];
  - deflate: one fixed-Huffman block (BFINAL = 1, BTYPE = 01) with every row's tokens in order, then end-of-block;
  - zlib: 0x78 0x01, the deflate data, Adler-32 of S big-endian;
  - PNG: signature, IHDR (W, H, 8, 2, 0, 0, 0), one IDAT with the whole zlib stream, IEND, each chunk's CRC-32 over its
    type and data.
Checksums are restated here (Adler-32 in numpy, CRC-32 from its table), not taken from zlib, so the tests can hold
both against zlib.
"""
from __future__ import annotations

import numpy as np

MAX_MATCH, MIN_MATCH, WINDOW = 258, 3, 32768
FIXED_OVERHEAD = 63                 # signature 8, IHDR 25, IDAT length + type 8, zlib header 2, Adler 4, CRC 4, IEND 12
SIGNATURE = b"\x89PNG\r\n\x1a\n"

LEN_BASE = [3, 4, 5, 6, 7, 8, 9, 10, 11, 13, 15, 17, 19, 23, 27, 31, 35, 43, 51, 59, 67, 83, 99, 115, 131, 163, 195,
            227, 258]
LEN_EXTRA = [0] * 8 + [1] * 4 + [2] * 4 + [3] * 4 + [4] * 4 + [5] * 4 + [0]
DIST_BASE = [1, 2, 3, 4, 5, 7, 9, 13, 17, 25, 33, 49, 65, 97, 129, 193, 257, 385, 513, 769, 1025, 1537, 2049, 3073,
             4097, 6145, 8193, 12289, 16385, 24577]
DIST_EXTRA = [0, 0, 0, 0] + [e for e in range(1, 14) for _ in (0, 1)]


def distances(s):
    """The candidate distances in the order the tie rule reads them."""
    return (1, 2, 3, 4, 5, 6, 7, 8, 9, 12, s, s - 3, s + 3, s - 6, s + 6)


def max_bytes(h, w):
    """Size bound of one frame's file: 9 bits per filtered byte, the 3-bit block header, end-of-block, the fixed
    overhead."""
    return (3 + 9 * h * (3 * w + 1) + 7 + 7) // 8 + FIXED_OVERHEAD


def filtered(frame):
    """The Sub-filtered scanlines S of an (H, W, 3) uint8 frame, (H, s) uint8."""
    h, w, _ = frame.shape
    raw = np.asarray(frame, np.uint8).reshape(h, 3 * w).astype(np.int16)
    out = np.empty((h, 3 * w + 1), np.uint8)
    out[:, 0] = 1
    out[:, 1:4] = raw[:, :3]
    out[:, 4:] = (raw[:, 3:] - raw[:, :-3]) & 0xFF
    return out


def tokens(S):
    """The greedy parse of S (H, s): a list of (literal byte) ints and (length, distance) tuples in row order."""
    h, s = S.shape
    flat = S.reshape(-1)
    n = flat.size
    pos = np.arange(n)
    room = np.minimum(MAX_MATCH, s - pos % s)
    ds = [d for d in distances(s)]
    lengths = np.zeros((len(ds), n), np.int16)
    for k, d in enumerate(ds):
        if d < 1 or d > WINDOW or d >= n:
            continue                                   # never valid (d <= p < n): length 0 everywhere
        eq = np.zeros(n, bool)
        eq[d:] = flat[d:] == flat[:-d]
        nxt = np.minimum.accumulate(np.where(eq, n, pos)[::-1])[::-1]   # first mismatch at or after p
        lengths[k] = np.minimum(nxt - pos, room)
    best = lengths.max(0)
    first = np.argmax(lengths == best[None], axis=0)
    out, p = [], 0
    while p < n:
        if best[p] >= MIN_MATCH:
            out.append((int(best[p]), ds[first[p]]))
            p += int(best[p])
        else:
            out.append(int(flat[p]))
            p += 1
    return out


def _rev(code, n):
    return int(format(code, f"0{n}b")[::-1], 2)


def _code(tok):
    """(value, bit count) of one token in the LSB-first stream."""
    if isinstance(tok, int):
        code, n = (0x30 + tok, 8) if tok < 144 else (0x190 + tok - 144, 9)
        return _rev(code, n), n
    length, dist = tok
    i = max(k for k in range(29) if LEN_BASE[k] <= length) if length < 258 else 28
    sym = 257 + i
    code, n = (sym - 256, 7) if sym < 280 else (0xC0 + sym - 280, 8)
    v, nb = _rev(code, n), n
    v |= (length - LEN_BASE[i]) << nb
    nb += LEN_EXTRA[i]
    j = max(k for k in range(30) if DIST_BASE[k] <= dist)
    v |= _rev(j, 5) << nb
    nb += 5
    v |= (dist - DIST_BASE[j]) << nb
    return v, nb + DIST_EXTRA[j]


def deflate(toks):
    """One fixed-Huffman block holding toks, then end-of-block (7 zero bits), padded to a byte."""
    codes = [(3, 3)] + [_code(t) for t in toks] + [(0, 7)]          # BFINAL = 1, BTYPE = 01 (LSB first)
    vals = np.array([c[0] for c in codes], np.int64)
    nbits = np.array([c[1] for c in codes], np.int64)
    offs = np.concatenate([[0], np.cumsum(nbits)])
    bits = np.zeros((offs[-1] + 7) // 8 * 8, np.uint8)
    for j in range(int(nbits.max())):
        m = nbits > j
        bits[offs[:-1][m] + j] = (vals[m] >> j) & 1
    return np.packbits(bits, bitorder="little").tobytes()


def adler32(data):
    x = np.frombuffer(bytes(data), np.uint8).astype(np.int64)
    n, mod = x.size, 65521
    a = (1 + int(x.sum())) % mod
    b = (n + int((((n - np.arange(n)) % mod) * x).sum())) % mod
    return (b << 16) | a


def _crc_table():
    t = []
    for i in range(256):
        c = i
        for _ in range(8):
            c = (c >> 1) ^ 0xEDB88320 if c & 1 else c >> 1
        t.append(c)
    return t


_CRC_TABLE = _crc_table()


def crc32(data):
    c = 0xFFFFFFFF
    for b in bytes(data):
        c = _CRC_TABLE[(c ^ b) & 0xFF] ^ (c >> 8)
    return c ^ 0xFFFFFFFF


def _chunk(kind, data):
    return len(data).to_bytes(4, "big") + kind + data + crc32(kind + data).to_bytes(4, "big")


def encode(frame):
    """The PNG file of one (H, W, 3) uint8 frame, as bytes."""
    frame = np.asarray(frame)
    assert frame.dtype == np.uint8 and frame.ndim == 3 and frame.shape[2] == 3 and frame.shape[0] * frame.shape[1] > 0
    h, w, _ = frame.shape
    S = filtered(frame)
    z = b"\x78\x01" + deflate(tokens(S)) + adler32(S.tobytes()).to_bytes(4, "big")
    ihdr = w.to_bytes(4, "big") + h.to_bytes(4, "big") + bytes([8, 2, 0, 0, 0])
    out = SIGNATURE + _chunk(b"IHDR", ihdr) + _chunk(b"IDAT", z) + _chunk(b"IEND", b"")
    assert len(out) <= max_bytes(h, w)
    return out

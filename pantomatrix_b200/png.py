"""PNG files of rendered frames, encoded on the GPU.

Each (H, W, 3) uint8 frame becomes one PNG file by one fixed rule (DESIGN.md section 11, include/pm_emage.h pm_png_*):
every scanline is Sub-filtered; each row of the filtered bytes S is parsed greedily, taking at every position the longest
match (3 to 258 bytes, within the row) over the distances (1, 2, 3, 4, 5, 6, 7, 8, 9, 12, s, s-3, s+3, s-6, s+6), s =
3 W + 1, the first distance in that order on ties, and otherwise a literal; the tokens of all rows go into one deflate
block with fixed Huffman codes, wrapped as zlib (Adler-32 of S) in one IDAT chunk between IHDR and IEND.  The bytes
depend only on the frame: the same frame gives the same file alone or in any batch.

    data, nbytes = png.encode(renderer.render_sequence(poses, expression, trans))   # (B*T, cap) uint8, (B*T,) int64
    png.write_frames(frames[0], "out/clip_frames")                                   # frame_00000.png, ...

The encoder is lossless: a decoder gives back the frame bit for bit.
"""
from __future__ import annotations

import os

import torch

from . import ops, slots

FIXED_OVERHEAD = 63        # signature 8, IHDR 25, IDAT length and type 8, zlib header 2, Adler 4, IDAT CRC 4, IEND 12
MAX_FILE_BYTES = 1 << 31


def max_bytes(h: int, w: int) -> int:
    """The size bound of one (h, w) frame's file: a literal costs at most 9 bits, a match at most 9 bits per byte it
    covers, so at most ceil((3 + 9 h s + 7) / 8) bytes of deflate data (header, tokens, end-of-block) plus the fixed
    overhead."""
    return (3 + 9 * h * (3 * w + 1) + 7 + 7) // 8 + FIXED_OVERHEAD


def slot_bytes(h: int, w: int) -> int:
    """Bytes of one output slot: max_bytes rounded up to a multiple of 4 (the kernels write 32-bit words)."""
    return (max_bytes(h, w) + 3) & ~3


@torch.no_grad()
def encode(frames, out=None):
    """PNG files of frames (N, H, W, 3) or (B, T, H, W, 3) uint8 CUDA, each frame dense (a MeshRenderer result is read
    in place).  Returns (data, nbytes): data (N, cap) uint8 holds file i in data[i, :nbytes[i]] (zeros after it),
    nbytes (N,) int64, both on the frames' device.  out: an optional (data, nbytes) pair to fill, data (N, cap) uint8
    contiguous with cap >= slot_bytes(H, W) and a multiple of 4, nbytes (N,) int64 contiguous.  No host
    synchronisation; with out given the call can be captured in a CUDA graph.  Raises ValueError on a CPU tensor, a wrong
    dtype or shape, frames that are not dense, an out too small, or a frame whose bound passes 2^31 bytes."""
    frames, _ = slots.frames(frames)
    n, h, w, _ = frames.shape
    if max_bytes(h, w) > MAX_FILE_BYTES:
        raise ValueError(f"a {h} x {w} frame may take {max_bytes(h, w)} bytes, more than 2^31")
    dev = frames.device
    data, nbytes = slots.output(n, max_bytes(h, w), slot_bytes(h, w), dev, out)
    if n == 0:
        return data, nbytes
    row_bits = torch.empty(n, h, dtype=torch.int64, device=dev)
    row_adler = torch.empty(n, h, dtype=torch.int64, device=dev)
    ops.png_encode(frames, data, nbytes, row_bits, row_adler)
    return data, nbytes


def write_frames(frames, folder, pattern="frame_%05d.png"):
    """Encode frames (as encode() takes them) and write file i to folder/(pattern % i).  Reads the sizes once (one
    synchronisation), copies only the encoded bytes to the host and waits for those copies.  Returns the paths."""
    data, nbytes = encode(frames)
    sizes = nbytes.tolist()
    os.makedirs(folder, exist_ok=True)
    paths = []
    if not sizes:
        return paths
    (files,) = slots.to_host((data, sizes))
    for i, blob in enumerate(files):
        path = os.path.join(folder, pattern % i)
        with open(path, "wb") as f:
            f.write(blob)
        paths.append(path)
    return paths

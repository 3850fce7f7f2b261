"""The PNG encoding rule on the CPU (oracle/png_oracle.py, DESIGN.md section 11): its files decode to the exact frame
with zlib and numpy, with Pillow, and carry the checksums zlib computes; random noise stays within the size bound; and
the ops wrapper marshals valid ctypes arguments.  The GPU's bytes are compared with these in tests/test_png_gpu.py."""
import ctypes
import io
import struct
import zlib

import numpy as np
import pytest
import torch
from PIL import Image

from oracle import png_oracle as P
from pantomatrix_b200 import png


def _chunks(b):
    assert b[:8] == P.SIGNATURE
    out, at = [], 8
    while at < len(b):
        n = struct.unpack(">I", b[at:at + 4])[0]
        kind, data, crc = b[at + 4:at + 8], b[at + 8:at + 8 + n], struct.unpack(">I", b[at + 8 + n:at + 12 + n])[0]
        out.append((kind, data, crc))
        at += 12 + n
    assert at == len(b)
    return out


def _unfilter(raw, h, w):
    rows = np.frombuffer(raw, np.uint8).reshape(h, 3 * w + 1)
    assert (rows[:, 0] == 1).all()
    out = rows[:, 1:].astype(np.int64)
    for i in range(3, 3 * w):
        out[:, i] = (out[:, i] + out[:, i - 3]) & 0xFF
    return out.astype(np.uint8).reshape(h, w, 3)


def check_file(b, frame):
    """b decodes to frame three ways: zlib + un-filtering, Pillow, and checksums against zlib's."""
    h, w, _ = frame.shape
    chunks = _chunks(b)
    assert [c[0] for c in chunks] == [b"IHDR", b"IDAT", b"IEND"]
    assert chunks[0][1] == struct.pack(">IIBBBBB", w, h, 8, 2, 0, 0, 0)
    for kind, data, crc in chunks:
        assert crc == zlib.crc32(kind + data)
    z = chunks[1][1]
    assert z[:2] == b"\x78\x01" and z[2] & 7 == 3                  # BFINAL = 1, BTYPE = 01
    raw = zlib.decompress(z)
    assert struct.unpack(">I", z[-4:])[0] == zlib.adler32(raw)
    assert np.array_equal(_unfilter(raw, h, w), frame)
    im = Image.open(io.BytesIO(b))
    assert im.mode == "RGB" and np.array_equal(np.asarray(im), frame)
    assert len(b) <= P.max_bytes(h, w)


def cases():
    """(name, frame) edge cases, shared with the GPU test."""
    rng = np.random.default_rng(7)
    noise = lambda h, w: rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
    grad = np.zeros((37, 53, 3), np.uint8)
    grad[..., 0] = np.arange(53)[None] * 4
    grad[..., 1] = np.arange(37)[:, None] * 6
    grad[..., 2] = (np.arange(37)[:, None] + np.arange(53)[None]) * 2
    runs = np.zeros((5, 400, 3), np.uint8)                         # rows of 1201 bytes: zero runs past 258
    runs[2, 390:] = 200
    return [("1x1", noise(1, 1)), ("1xW", noise(1, 97)), ("Hx1", noise(83, 1)),
            ("zeros", np.zeros((24, 40, 3), np.uint8)), ("gray", np.full((19, 33, 3), 128, np.uint8)),
            ("zero_runs", runs), ("gradient", grad), ("noise", noise(31, 45)),
            ("wide", np.tile(noise(3, 7), (1, 1572, 1))[:, :11000])]   # s = 33001: no row candidate is valid


@pytest.mark.parametrize("name,frame", cases(), ids=[c[0] for c in cases()])
def test_oracle_files_decode_to_the_frame(name, frame):
    check_file(P.encode(frame), frame)


def test_noise_stays_within_the_bound_and_the_bound_is_the_products():
    rng = np.random.default_rng(3)
    for h, w in ((1, 1), (2, 3), (16, 16), (40, 77)):
        f = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
        b = P.encode(f)
        assert len(b) <= P.max_bytes(h, w) == png.max_bytes(h, w)
        check_file(b, f)
        assert png.slot_bytes(h, w) % 4 == 0 and png.slot_bytes(h, w) - png.max_bytes(h, w) < 4


def test_row_candidates_beyond_the_window_are_skipped():
    """s = 33001: the row distances s +- k all exceed 32768, so a row equal to the previous one is still coded from
    its own bytes; with s = 3001 it becomes matches at distance s."""
    row = np.random.default_rng(5).integers(0, 256, (1, 11000, 3), dtype=np.uint8)
    toks = P.tokens(P.filtered(np.repeat(row, 2, 0)))
    assert all(isinstance(t, int) or t[1] <= 32768 for t in toks)
    assert sum(1 for t in toks if isinstance(t, int)) >= 2 * 11000 * 3 * 0.9
    small = np.repeat(row[:, :1000], 2, 0)
    toks = P.tokens(P.filtered(small))
    assert sum(t[0] for t in toks if not isinstance(t, int) and t[1] == 3001) >= 3000


def test_greedy_parse_takes_the_first_distance_on_ties():
    # a constant row: distance 1 and 3 both reach 258, the rule takes 1
    toks = P.tokens(P.filtered(np.full((1, 200, 3), 9, np.uint8)))
    assert toks[:2] == [1, 9] and all(t[1] == 1 for t in toks if not isinstance(t, int))


def test_encode_rejects_bad_inputs_on_the_host():
    with pytest.raises(ValueError):
        png.encode(torch.zeros(2, 4, 4, 3, dtype=torch.uint8))                 # CPU tensor
    with pytest.raises(ValueError):
        png.encode(np.zeros((2, 4, 4, 3), np.uint8))                           # not a tensor


def test_ops_png_wrapper_marshals_valid_arguments(monkeypatch):
    """ops.png_encode with the library call replaced by a recorder: every argument converts to its declared ctypes type,
    the slots are cleared first, and the four stages run in order on the same workspace."""
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
    frames = torch.zeros(3, 5, 7, 3, dtype=torch.uint8)
    cap = png.slot_bytes(5, 7)
    data, nbytes = torch.zeros(3, cap, dtype=torch.uint8), torch.zeros(3, dtype=torch.int64)
    rb, ra = torch.zeros(3, 5, dtype=torch.int64), torch.zeros(3, 5, dtype=torch.int64)
    ops.png_encode(frames, data, nbytes, rb, ra)
    assert [c[0] for c in calls] == ["pm_memset_async", "pm_png_count", "pm_png_scan", "pm_png_emit", "pm_png_crc"]
    by = dict(calls)
    assert by["pm_memset_async"][1:3] == (0, 3 * cap)
    assert by["pm_png_count"][1:5] == (105, 3, 5, 7)
    assert by["pm_png_scan"][3] == by["pm_png_emit"][5] == rb.data_ptr() and by["pm_png_scan"][6] == cap
    assert by["pm_png_crc"][5] == by["pm_png_scan"][7] == nbytes.data_ptr()

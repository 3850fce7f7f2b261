"""The H.264 Intra 4x4 rule on the CPU (tests/h264_ref.py, DESIGN.md section 12): clips coded with intra4x4 decode
with OpenCV's FFmpeg to the restatement's reconstruction, which anchors the nine prediction modes, the sample
availability, the mode prediction, the Intra cbp mapping and nC beside every neighbour type; every mode, both
prev_intra4x4_pred_mode_flag values, both intra macroblock types and I_NxN in P slices occur; bad intra4x4 values; and
the ops wrapper's ctypes arguments.  The GPU's bytes are compared with these in tests/test_video_i4_gpu.py."""
import ctypes
import functools
import hashlib
import json
import os

import numpy as np
import pytest
import torch

import h264_ref as R
from oracle import h264_oracle as O
from pantomatrix_b200 import video
from test_video_gop import check_clip


def stripes(h, w, angle, period, phase=0.0):
    """RGB stripes at angle (radians) with the given period in pixels: an edge direction every mode can follow."""
    y, x = np.mgrid[0:h, 0:w].astype(np.float64)
    v = np.sin(2 * np.pi * (x * np.cos(angle) + y * np.sin(angle) + phase) / period)
    g = 128 + 100 * v
    return np.clip(np.rint(np.stack([g, 0.7 * g + 30, 255 - g], -1)), 0, 255).astype(np.uint8)


def edges(h, w, t=0):
    """Sharp edges of each orientation in 16x16 tiles, shifted by t pixels: steps, wedges and corners."""
    y, x = np.mgrid[0:h, 0:w]
    k = (y // 16 * 7 + x // 16) % 6
    xx, yy = (x + t) % 16, y % 16
    m = np.select([k == 0, k == 1, k == 2, k == 3, k == 4, k == 5],
                  [xx + yy < 16, xx - yy > 2, 2 * xx + yy < 20, xx + 2 * yy < 22, xx > 9, (yy > 6) & (xx < 11)])
    f = np.where(m[..., None], np.array([220, 200, 40]), np.array([30, 60, 150]))
    return f.astype(np.uint8)


def scene(h, w, t, rng):
    """A flat background that stays (P_Skip), stripes that move (inter), a block of new noise each frame (I_PCM at qp
    0) and edges beside each."""
    f = np.full((h, w, 3), 90, np.uint8)
    f[:, 16:48] = stripes(h, 32, 0.6, 7, 1.5 * t)
    f[:, 48:64] = rng.integers(0, 256, (h, 16, 3), dtype=np.uint8)
    f[:, 64:96] = edges(h, 32, t)
    f[:16, 96:112] = np.roll(f[:16, 16:32], 3 * t, 1)
    return f


@functools.lru_cache(maxsize=None)
def i4_cases():
    """(name, frames, qp, search) clips, shared with the GPU test."""
    rng = np.random.default_rng(31)
    angles = [stripes(48, 64, a, p, t) for t, (a, p) in enumerate([(0.0, 6), (np.pi / 2, 5), (np.pi / 4, 6),
                                                                  (3 * np.pi / 4, 7), (0.35, 5), (1.2, 6)])]
    sc = [scene(48, 128, t, rng) for t in range(4)]
    return [("stripes_qp20", angles, 20, 0),
            ("stripes_qp26_search16", angles, 26, 16),
            ("edges_qp20", [edges(48, 96, t) for t in range(4)], 20, 16),
            ("scene_qp0", sc, 0, 0),
            ("scene_qp20", sc, 20, 16),
            ("stripes_qp0", angles[:3], 0, 0),
            ("stripes_qp51", angles[:3], 51, 16),
            ("one_row", [stripes(16, 80, 0.3 * t + 0.2, 5) for t in range(3)], 20, 16),
            ("one_column", [stripes(64, 16, 0.4 * t + 1.0, 6) for t in range(3)], 26, 0)]


GOPS = (1, 2, 7, "T", "T+5")


def gop_of(g, t):
    return t if g == "T" else (t + 5 if g == "T+5" else g)


def case(name):
    return {c[0]: c[1:] for c in i4_cases()}[name]


@functools.lru_cache(maxsize=None)
def encoded(name, g):
    frames, qp, rng = case(name)
    return R.encode_clip(frames, qp, gop_of(g, len(frames)), rng, True)


@functools.lru_cache(maxsize=None)
def noise_bound(gop):
    """The clip of test_bound_holds_on_noise_at_qp_0 at gop 1 or 3."""
    rng = np.random.default_rng(8)
    frames = [rng.integers(0, 256, (32, 64, 3), dtype=np.uint8) for _ in range(3)]
    frames[1][:, :32] = stripes(32, 32, 0.5, 4)
    return R.encode_clip(frames, 0, gop, 0, True)


@pytest.mark.parametrize("g", GOPS, ids=[str(g) for g in GOPS])
@pytest.mark.parametrize("name", [c[0] for c in i4_cases()])
def test_i4_clips_decode_to_the_reconstruction(name, g, tmp_path):
    enc = encoded(name, g)
    h, w = enc[0][1][0].shape
    check_clip(enc, h, w, gop_of(g, len(enc)), tmp_path)


def _all():
    return [e for name, *_ in i4_cases() for g in GOPS for e in encoded(name, g)]


def test_every_mode_flag_and_macroblock_type_occurs():
    modes, flags, types, p_i4 = set(), set(), set(), False
    for e in _all():
        types |= set(e[2].reshape(-1))
        m = e.modes[e[2] == R.I4]
        modes |= set(m.reshape(-1).tolist())
        p_i4 |= e.mv is not None and bool((e[2] == R.I4).any())
        for my, mx in zip(*np.nonzero(e[2] == R.I4)):
            lm = e.modes[my, mx - 1] if mx and e[2][my, mx - 1] == R.I4 else np.full((4, 4), 2)
            for by, bx in R.LUMA_BLK:
                if by == 0 or (bx == 0 and mx == 0):
                    pm = 2
                else:
                    pm = min(e.modes[my, mx, by, bx - 1] if bx else lm[by, 3], e.modes[my, mx, by - 1, bx])
                flags.add(bool(e.modes[my, mx, by, bx] == pm))
    assert modes == set(range(9)), sorted(modes)
    assert flags == {True, False}
    assert {"DC", "H", R.I4, O.PCM, R.SKIP, R.INTER} <= types, types
    assert p_i4


def test_i_nxn_sits_right_of_every_macroblock_type():
    left = set()
    for e in _all():
        t = e[2]
        left |= {t[my, mx - 1] for my, mx in zip(*np.nonzero(t == R.I4)) if mx}
    assert {R.SKIP, R.INTER, R.I4, O.PCM} <= left and left & {"DC", "H"}, left     # DC, H: Intra16x16


@pytest.mark.parametrize("name", [c[0] for c in i4_cases() if R.LAMBDA[c[2]] > 0])   # lambda 0: c lambda is 0
def test_a_constant_past_every_cost_is_the_rule_without_intra4x4(name):
    """At gop > 1 the rule without intra4x4 is the candidate never computed, and the bytes the motion search rule's own
    restatement coded, pinned by their digests."""
    frames, qp, rng = case(name)
    with open(os.path.join(os.path.dirname(__file__), "golden", "h264_ref_digests.json")) as f:
        pinned = json.load(f)["without_i4"]
    for gop in (1, 2, len(frames)):
        off = [e[0] for e in R.encode_clip(frames, qp, gop, rng, True, c=1 << 40)]
        if gop == 1:
            assert off == [O.encode(f, qp, t)[0] for t, f in enumerate(frames)]
        else:
            assert off == [e[0] for e in R.encode_clip(frames, qp, gop, rng, False)]
            assert [hashlib.sha256(b).hexdigest() for b in off] == pinned[f"{name}/{gop}"]


def test_intra_cbp_table_is_a_permutation():
    assert sorted(R.INTRA_CBP) == list(range(48))
    assert R.INTRA_CBP[:4] == [47, 31, 15, 0] and R.INTRA_CBP[-1] == 41


def test_bound_holds_on_noise_at_qp_0():
    for gop in (1, 3):
        for e in noise_bound(gop):
            assert len(e[0]) <= video.max_bytes(32, 64, gop)


def test_bad_intra4x4_raises_value_error():
    f = torch.zeros(2, 16, 16, 3, dtype=torch.uint8)
    for v in (1, 0, None, "yes", 1.0, np.bool_(True)):
        with pytest.raises(ValueError, match="intra4x4 must be"):
            video._intra4x4(v)
        with pytest.raises(ValueError, match="intra4x4 must be"):
            video.encode(f, intra4x4=v)
        with pytest.raises(ValueError, match="intra4x4 must be"):
            video.write_mp4(f, "unused.mp4", intra4x4=v)


@pytest.mark.parametrize("gop,search,entry", [(1, 0, "pm_h264_encode"), (7, 0, "pm_h264_encode_gop"),
                                              (7, 16, "pm_h264_encode_me")])
@pytest.mark.parametrize("intra4x4", [False, True])
def test_ops_h264_wrapper_passes_the_flag_in_qp(gop, search, entry, intra4x4, monkeypatch):
    """ops.h264_encode(..., intra4x4) with the library call replaced by a recorder: every argument converts to its
    declared ctypes type and the entry point gets qp | PM_H264_I4X4 exactly when intra4x4 is set."""
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
    cap, sc = video.slot_bytes(32, 48, gop), video.slice_bytes(48, gop)
    data, nbytes = torch.zeros(20, cap, dtype=torch.uint8), torch.zeros(20, dtype=torch.int64)
    scratch, sizes = torch.zeros(20, 2, sc, dtype=torch.uint8), torch.zeros(20, 2, dtype=torch.int32)
    kw = {}
    if gop > 1:
        kw["recon"] = (torch.zeros(4, 3 * 32 * 48, dtype=torch.uint8) if search
                       else torch.zeros(4, 2, 24 * 48, dtype=torch.uint8))
    if search:
        kw.update(search=search, mv=torch.zeros(4, 2, 3, 2, dtype=torch.int16))
    ops.h264_encode(frames, 10, 26, data, nbytes, scratch, sizes, gop=gop, intra4x4=intra4x4, **kw)
    assert [c[0] for c in calls] == ["pm_memset_async", entry, "pm_h264_gather"]
    args = dict(calls)[entry]
    assert args[1:6] == (32 * 48 * 3, 20, 10, 32, 48)
    assert args[6] == (26 | 0x100 if intra4x4 else 26)
    assert ops.H264_I4X4 == 0x100


def test_encode_passes_intra4x4_only_when_set(monkeypatch):
    from pantomatrix_b200 import ops, slots
    seen = []
    monkeypatch.setattr(slots, "frames", lambda f: (f.reshape(-1, *f.shape[-3:]), f.shape[1]))
    monkeypatch.setattr(ops, "h264_encode", lambda *a, **kw: seen.append(kw.get("intra4x4")))
    for gop, search in ((1, 0), (3, 0), (3, 8)):
        for v in (False, True):
            video.encode(torch.zeros(1, 5, 32, 48, 3, dtype=torch.uint8), gop=gop, search=search, intra4x4=v)
    assert seen == [None, True] * 3

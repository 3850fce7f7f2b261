"""The H.264 motion search rule on the CPU (tests/h264_ref.py, DESIGN.md section 12): clips coded with quarter-pel
motion decode with OpenCV's FFmpeg to the restatement's reconstruction, which anchors the interpolation and the vector
predictor; translating clips get their true displacement; search 0 is the zero-motion rule (the bytes pinned in
tests/golden/h264_ref_digests.json); lambda(qp); the bound;
bad search values; and the ops wrapper's ctypes arguments for pm_h264_encode_me.  The GPU's bytes are compared with
these in tests/test_video_me_gpu.py."""
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


def texture(h, w, dx=0.0, dy=0.0):
    """A smooth RGB texture sampled at (x - dx, y - dy): sub-pixel motion the 6-tap filter follows closely."""
    y, x = np.mgrid[0:h, 0:w].astype(np.float64)
    x, y = x - dx, y - dy
    out = [128 + 55 * np.sin(2 * np.pi * x / 23 + k) + 45 * np.cos(2 * np.pi * y / 19 - k)
           + 20 * np.sin(2 * np.pi * (x + y) / 13 + 2 * k) for k in range(3)]
    return np.clip(np.rint(np.stack(out, -1)), 0, 255).astype(np.uint8)


def square(h, w, steps, at=(8, 12), size=48):
    """A textured square on black moving by steps[t] (pixels, x and y) before frame t + 1; also the true quarter-pel
    vector of each frame after the first."""
    frames, truth, ox, oy = [], [], 0.0, 0.0
    for t in range(len(steps) + 1):
        if t:
            ox, oy = ox + steps[t - 1][0], oy + steps[t - 1][1]
            truth.append((round(-4 * steps[t - 1][0]), round(-4 * steps[t - 1][1])))
        f = np.zeros((h, w, 3), np.uint8)
        tex = texture(h, w, ox, oy)
        y0, x0 = at[0] + int(np.floor(oy)), at[1] + int(np.floor(ox))
        f[y0:y0 + size, x0:x0 + size] = tex[y0:y0 + size, x0:x0 + size]
        frames.append(f)
    return frames, truth


PHASES = [(fx / 4 + (1 if fx == 0 and fy == 0 else 0), fy / 4) for fy in range(4) for fx in range(4)]


@functools.lru_cache(maxsize=None)
def me_cases():
    """(name, frames, qp, search, true vectors or None) clips, shared with the GPU test."""
    rng = np.random.default_rng(23)
    noise = lambda h, w: rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
    sq_int, t_int = square(64, 96, [(3, -2), (-2, 1), (4, 3)])
    sq_sub, t_sub = square(64, 96, [(0.25, 0.75), (0.5, -0.25), (0.75, 0.5), (-0.5, -0.75)])
    field = noise(96, 128)
    pan = [field[8 + t:56 + t, 16 - 2 * t:80 - 2 * t] for t in range(4)]
    # every quarter-pel phase: a whole-frame texture panning by each (fx / 4, fy / 4), reading clipped samples at all
    # four frame edges
    edges, ox, oy = [texture(32, 48)], 0.0, 0.0
    for sx, sy in PHASES:
        ox, oy = ox + sx, oy + sy
        edges.append(texture(32, 48, ox, oy))
    drift = [noise(32, 48)]
    drift.append(np.clip(drift[0].astype(int) + rng.integers(-24, 25, drift[0].shape), 0, 255).astype(np.uint8))
    drift.append(noise(32, 48))
    return [("square_int", sq_int, 20, 16, t_int),
            ("square_subpel", sq_sub, 20, 16, t_sub),
            ("pan_noise", pan, 20, 32, [(-8, 4)] * 3),
            ("edges_all_phases", edges, 20, 1, None),
            ("noise_qp0", drift, 0, 16, None),
            ("square_qp51", sq_sub, 51, 32, None),
            ("one_row", [texture(16, 80, 1.5 * t, 0) for t in range(3)], 20, 16, None),
            ("one_column", [texture(64, 16, 0, -1.25 * t) for t in range(3)], 26, 16, None)]


GOPS = (2, 7, "T", "T+5")


def gop_of(g, t):
    return t if g == "T" else (t + 5 if g == "T+5" else g)


def case(name):
    return {c[0]: c[1:] for c in me_cases()}[name]


@functools.lru_cache(maxsize=None)
def encoded(name, g):
    frames, qp, rng, _ = case(name)
    return R.encode_clip(frames, qp, gop_of(g, len(frames)), rng)


@functools.lru_cache(maxsize=None)
def noise_bound():
    """The clip of test_bound_holds_on_noise_at_search_32_and_qp_0: gop 4, search 32, qp 0."""
    rng = np.random.default_rng(4)
    a = rng.integers(0, 256, (48, 64, 3), dtype=np.uint8)
    frames = [a, np.roll(a, (3, -5), (0, 1)), np.clip(a.astype(int) + rng.integers(-30, 31, a.shape), 0, 255)
              .astype(np.uint8), rng.integers(0, 256, (48, 64, 3), dtype=np.uint8)]
    return R.encode_clip(frames, 0, 4, 32)


@pytest.mark.parametrize("g", GOPS, ids=[str(g) for g in GOPS])
@pytest.mark.parametrize("name", [c[0] for c in me_cases()])
def test_me_clips_decode_to_the_reconstruction(name, g, tmp_path):
    enc = encoded(name, g)
    h, w = enc[0][1][0].shape
    check_clip(enc, h, w, gop_of(g, len(enc)), tmp_path)


def _interior(frames, t):
    """Macroblocks inside the textured square in frames t - 1 and t."""
    inside = lambda f: f.reshape(f.shape[0] // 16, 16, f.shape[1] // 16, 16, 3).min((1, 3, 4)) > 0
    return inside(frames[t - 1]) & inside(frames[t])


@pytest.mark.parametrize("name", ["square_int", "square_subpel", "pan_noise"])
def test_translating_clips_get_the_true_displacement(name):
    frames, _, _, truth = case(name)
    enc = encoded(name, "T")
    for t in range(1, len(frames)):
        if name.startswith("square"):
            where = _interior(frames, t)
        else:                                            # where the true block lies inside the frame
            where = np.ones(enc[t][2].shape, bool)
            where[-1], where[:, 0] = False, False
        coded = where & (enc[t][2] == R.INTER)
        assert coded.sum() >= 2, (name, t)
        assert (enc[t].mv[coded] == truth[t - 1]).all(), (name, t, enc[t].mv[coded].tolist(), truth[t - 1])


def test_every_macroblock_type_phase_and_predictor_occurs():
    types, phases, mvd_nonzero, left_pred = set(), set(), False, False
    for name, *_ in me_cases():
        for e in encoded(name, "T"):
            types |= set(e[2].reshape(-1))
            if e.mv is None:
                continue
            p = e[2] == R.INTER
            phases |= {(int(x) & 3, int(y) & 3) for x, y in e.mv[p]}
            for my in range(p.shape[0]):
                for mx in range(p.shape[1]):
                    if not p[my, mx]:
                        continue
                    mvp = e.mv[my, mx - 1] if mx and p[my, mx - 1] else np.zeros(2)
                    mvd_nonzero |= bool((e.mv[my, mx] != mvp).any())
                    left_pred |= bool(mvp.any())
    assert types == {R.SKIP, R.INTER, "DC", "H", O.PCM}
    assert len(phases) == 16 and mvd_nonzero and left_pred


@pytest.mark.parametrize("name", [c[0] for c in me_cases()])
def test_search_0_is_the_zero_motion_rule(name):
    """The bytes of search 0 are those the zero-motion rule's own restatement coded, pinned by their digests."""
    frames, qp, _, _ = case(name)
    with open(os.path.join(os.path.dirname(__file__), "golden", "h264_ref_digests.json")) as f:
        want = json.load(f)["zero_motion"]
    for gop in (2, len(frames)):
        enc = R.encode_clip(frames, qp, gop, 0)
        assert [hashlib.sha256(e.data).hexdigest() for e in enc] == want[f"{name}/{gop}"]
        assert all(e.mv is None or not e.mv.any() for e in enc)


def test_lambda_table_is_the_formula():
    assert R.LAMBDA == [R.lam(qp) for qp in range(52)]
    assert R.LAMBDA[0] == 0 and R.LAMBDA[51] == 83


def test_bound_holds_on_noise_at_search_32_and_qp_0():
    enc = noise_bound()
    for e in enc:
        assert len(e[0]) <= video.max_bytes(48, 64, 4)
    assert any((e[2] == O.PCM).any() for e in enc[1:])


def test_bad_search_raises_value_error():
    f = np.zeros((2, 16, 16, 3), np.uint8)
    for search in (-1, 33, 2.0, True, "3", None):
        with pytest.raises(ValueError, match="search must be"):
            video._search(search)
        with pytest.raises(ValueError, match="search must be"):
            video.encode(torch.zeros(2, 16, 16, 3, dtype=torch.uint8), gop=2, search=search)
        with pytest.raises(ValueError, match="search must be"):
            video.write_mp4(torch.as_tensor(f), "unused.mp4", gop=2, search=search)


@pytest.mark.parametrize("gop,search,routed", [(5, 16, True), (2, 1, True), (9, 32, True), (5, 0, False),
                                                (1, 16, False)])
def test_encode_routes_search_and_sizes_its_workspaces(gop, search, routed, monkeypatch):
    """video.encode hands ops.h264_encode search and the two-frame and vector workspaces only when there are P frames
    and search > 0; otherwise the call is the zero-motion one, unchanged."""
    from pantomatrix_b200 import ops, slots
    seen = {}

    def record(frames, clip_len, qp, data, nbytes, scratch, sizes, gop=1, recon=None, **kw):
        seen.update(gop=gop, recon=None if recon is None else tuple(recon.shape), kw={k: (v if k == "search" else
                                                                                          tuple(v.shape))
                                                                                      for k, v in kw.items()})

    monkeypatch.setattr(slots, "frames", lambda f: (f.reshape(-1, *f.shape[-3:]), f.shape[1]))
    monkeypatch.setattr(ops, "h264_encode", record)
    video.encode(torch.zeros(3, 5, 32, 48, 3, dtype=torch.uint8), gop=gop, search=search)
    kgop = min(gop, 5)
    chains = 3 * -(-5 // kgop)
    assert seen["gop"] == kgop
    if routed:
        assert seen["recon"] == (chains, 3 * 32 * 48)
        assert seen["kw"] == {"search": search, "mv": (chains, 2, 3, 2)}
    else:
        assert seen["kw"] == {}


def test_ops_h264_me_wrapper_marshals_valid_arguments(monkeypatch):
    """ops.h264_encode(..., gop=7, search=16) with the library call replaced by a recorder: every argument converts to
    its declared ctypes type, pm_h264_encode_me gets gop, the workspaces, their sizes and search, and gather follows."""
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
    recon = torch.zeros(4, 3 * 32 * 48, dtype=torch.uint8)          # 2 clips of 10 frames: 2 GOPs each
    mv = torch.zeros(4, 2, 3, 2, dtype=torch.int16)
    ops.h264_encode(frames, 10, 20, data, nbytes, scratch, sizes, gop=7, recon=recon, search=16, mv=mv)
    assert [c[0] for c in calls] == ["pm_memset_async", "pm_h264_encode_me", "pm_h264_gather"]
    by = dict(calls)
    assert by["pm_h264_encode_me"][1:7] == (32 * 48 * 3, 20, 10, 32, 48, 20)
    assert by["pm_h264_encode_me"][7:16] == (scratch.data_ptr(), sc, sizes.data_ptr(), 7, recon.data_ptr(),
                                             3 * 32 * 48, 16, mv.data_ptr(), 4 * 2 * 3)
    assert by["pm_h264_gather"][3:6] == (scratch.data_ptr(), sc, sizes.data_ptr())

"""Every kernel that writes operand planes, held bit for bit to the one split rule (tests/plane_split.py) in both
plane formats and every split count: bf16 x1/2/3 and fp16 x1/2/3.

* pm_split_bf16 and the exact-copy producers (gather_rows, add2 with a zero addend, window_input) on an edge tensor:
  bf16 and fp16-head ties, mantissa carries, the fp16 subnormal thresholds after the x64 pre-scale, the fp16 overflow
  edge, fp32 subnormals, +-0, +-inf and NaN.  Each store path sees it: the 4-wide store, the scalar store, the scalar
  tails of unaligned rows.
* The arithmetic producers (add_layernorm, add_rows, attention, attention_tc, wav_stem, smplx_fk, the tap-GEMM
  epilogue): the planes of a call are the restated split of the fp32 output of the same call, and the planes-only call
  writes the same planes.  A NaN and an inf in one input row must leave non-finite plane sums wherever the fp32 output
  is not finite.

Finite elements are compared bit for bit (any NaN matches any NaN in a plane); at a non-finite value the plane sum
must be NaN for a NaN and not finite for an inf."""
import math

import numpy as np
import pytest
import torch

import plane_split as ps
from helpers import bf16_planes_by_default, slack_rows  # noqa: F401

pytestmark = [pytest.mark.gpu, pytest.mark.filterwarnings("ignore::RuntimeWarning")]

FORMATS = [ps.BF16, ps.FP16]
SPLITS = [1, 2, 3]
EDGE = ps.edge_values()


@pytest.fixture(scope="module")
def ops():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    from pantomatrix_b200 import _lib, ops as o
    _lib.load()
    assert _lib.load().pm_device_cc() == 90, "sm_90a kernels need a Hopper (H100) device"
    return o


@pytest.fixture(params=FORMATS)
def fmt(request, ops):
    ops.set_plane_format(request.param)
    return request.param


def _rand(*shape, seed=0, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(*shape, generator=g) * scale).cuda()


def _bits(t: torch.Tensor) -> np.ndarray:
    return t.contiguous().view(torch.int16).cpu().numpy().view(np.uint16)


def _same_bits(a: torch.Tensor, b: torch.Tensor) -> bool:
    """Bitwise equality (NaN payloads included)."""
    return a.shape == b.shape and torch.equal(a.contiguous().view(torch.int16 if a.element_size() == 2 else torch.int32),
                                              b.contiguous().view(torch.int16 if b.element_size() == 2 else torch.int32))


def check_rule(planes: torch.Tensor, x: torch.Tensor, fmt: str, tag: str, act: bool = True) -> None:
    """planes (nsplit, *x.shape) against the restated split of fp32 x, element by element."""
    xs = x.detach().float().cpu().numpy()
    got = _bits(planes)
    assert got.shape[1:] == xs.shape, (tag, got.shape, xs.shape)
    bad = ps.mismatches(got, xs, fmt, act)
    n = int(bad.sum())
    if n:
        i = np.unravel_index(int(np.flatnonzero(bad)[0]), xs.shape)
        want = ps.split(xs[i], got.shape[0], fmt, act)
        nf = int((bad & ~np.isfinite(xs)).sum())
        print(f"[{tag}] {n} of {bad.size} elements break the split rule, {nf} of them at non-finite values")
        raise AssertionError(f"{tag}: {n} of {bad.size} elements break the split rule ({nf} at non-finite values); "
                             f"first at {tuple(int(j) for j in i)}: "
                             f"x = {xs[i]!r} (0x{np.float32(xs[i]).view(np.uint32):08x}), planes "
                             f"{[hex(int(g)) for g in got[(slice(None),) + i]]}, rule {[hex(int(w)) for w in want]}")


def edge_tensor(shape, seed=0) -> torch.Tensor:
    """fp32 CUDA tensor of `shape` filled with the edge values (every one at least once when numel >= len(EDGE)), in a
    seeded order so each lands at various columns."""
    n = math.prod(shape)
    reps = -(-n // EDGE.size)
    rng = np.random.default_rng(seed)
    flat = np.concatenate([EDGE[rng.permutation(EDGE.size)] for _ in range(reps)])[:n]
    return torch.from_numpy(flat.reshape(shape).copy()).cuda()


def _with_nonfinite(x: torch.Tensor, row: int, cols=(5, 77)) -> torch.Tensor:
    """x with a NaN and an inf in one row (of its flattened leading dims)."""
    x = x.clone()
    v = x.view(-1, x.shape[-1])
    v[row, cols[0] % x.shape[-1]] = float("nan")
    v[row, cols[1] % x.shape[-1]] = float("inf")
    return x


def _nonfinite_reaches(f: torch.Tensor, tag: str) -> None:
    assert not bool(torch.isfinite(f).all()), f"{tag}: the NaN / inf input left the fp32 output finite"


# ------------------------------------------------------------------------------------------------------------------
# pm_split_bf16
# ------------------------------------------------------------------------------------------------------------------

SPLIT_SHAPES = [(1, 2221, 1), (3, 743, 3), (2, 227, 5), (1, 37, 61), (3, 35, 64), (2, 7, 337), (1, 3, 768)]


@pytest.mark.parametrize("nsplit", SPLITS)
def test_split_bf16_edge_values(ops, fmt, nsplit):
    """Dense inputs, column slices with 16-byte aligned rows (the 4-wide path when ch % 4 == 0) and unaligned ones (the
    scalar path); clip stride != rows * ldx; the zeroed slack rows after the last clip stay zero."""
    for k, (batch, rows, ch) in enumerate(SPLIT_SHAPES):
        x = edge_tensor((batch, rows, ch), seed=k)
        ld4 = (ch + 8 + 3) // 4 * 4
        wide = torch.zeros(batch, rows + 3, ld4, device="cuda")
        views = {"dense": x, "aligned slice": wide[:, 1:rows + 1, 4:4 + ch].copy_(x)}
        wide2 = torch.zeros(batch, rows + 2, ch + 5, device="cuda")
        views["unaligned slice"] = wide2[:, 2:, 1:1 + ch].copy_(x)
        if batch > 1:
            assert views["unaligned slice"].stride(0) != rows * views["unaligned slice"].stride(1)
        for name, v in views.items():
            tag = f"split {fmt} x{nsplit} {batch}x{rows}x{ch} {name}"
            pl = ops.split_bf16(v, nsplit, slack_rows=5)
            assert pl.t.dtype == (torch.bfloat16 if fmt == ps.BF16 else torch.float16)
            check_rule(pl.t[..., :ch], x, fmt, tag)
            assert not bool(slack_rows(pl).view(torch.int16).any()), f"{tag}: slack rows were written"


# ------------------------------------------------------------------------------------------------------------------
# exact-copy producers: the edge tensor through every store path
# ------------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("nsplit", SPLITS)
def test_gather_rows_edge_values(ops, fmt, nsplit):
    """Codebook rows = the edge values (4-wide store); the gathered fp32 rows are exact copies."""
    ch = 256
    n_codes = -(-EDGE.size // ch)
    cb = edge_tensor((n_codes, ch), seed=11)
    idx = torch.from_numpy(np.random.default_rng(12).permutation(np.arange(3 * 13) % n_codes).reshape(3, 13)).cuda()
    got = ops.gather_rows(cb, idx, nsplit=nsplit)
    assert _same_bits(got.f, cb[idx])
    check_rule(got.p.t[..., :ch], got.f, fmt, f"gather_rows {fmt} x{nsplit}")
    only = ops.gather_rows(cb, idx, nsplit=nsplit, f32=False)
    assert _same_bits(only.p.t[..., :ch], got.p.t[..., :ch])


@pytest.mark.parametrize("nsplit", SPLITS)
def test_add2_edge_values(ops, fmt, nsplit):
    """a + 0 with a = the edge values: 16-byte aligned rows take the 4-wide store, an operand 4 bytes off alignment the
    scalar store for every column.  (With planes, pm_add2_f32 needs ch % 4 == 0: the scalar path is reached through
    alignment, not through a ragged ch.)  x + 0 is exact except that -0 + 0 = +0, so the planes are compared with the
    split of the call's own fp32 output, and that output with a whose -0 became +0."""
    for rows, ch in ((37, 64), (5, 768), (61, 44)):
        a = edge_tensor((rows, ch), seed=rows)
        b = torch.zeros_like(a)
        buf = torch.empty(rows * ch + 4, device="cuda")
        a_off = buf[1:1 + rows * ch].view(rows, ch).copy_(a)
        assert a_off.data_ptr() % 16 != 0
        for name, aa in (("vector", a), ("scalar", a_off)):
            tag = f"add2 {fmt} x{nsplit} {rows}x{ch} {name}"
            got = ops.add2(aa, b, nsplit=nsplit)
            nan = torch.isnan(a)                          # NaN + 0 is a NaN, its payload is the hardware's
            assert torch.equal(torch.isnan(got.f), nan), tag
            assert _same_bits(got.f.masked_fill(nan, 0.0), torch.where(a == 0, 0.0, a).masked_fill(nan, 0.0)), tag
            check_rule(got.p.t[..., :ch].reshape(nsplit, rows, ch), got.f, fmt, tag)
            only = ops.add2(aa, b, nsplit=nsplit, f32=False)
            assert _same_bits(only.p.t[..., :ch], got.p.t[..., :ch]), tag


@pytest.mark.parametrize("nsplit", SPLITS)
def test_window_input_edge_values(ops, fmt, nsplit):
    """window_input at ch 337 (the scalar store): mask 0 copies the motion, mask 1 the mask embedding, and the defaults
    path (no motion / mask) copies the seed frames, then the embedding."""
    bs, total, ch, win, start = 2, 9, 337, 7, 1
    motion = edge_tensor((bs, total, ch), seed=21)
    zeros, ones = torch.zeros_like(motion), torch.ones_like(motion)
    emb0 = edge_tensor((ch,), seed=22)
    got = ops.window_input(motion, zeros, None, emb0, start, win, 0, nsplit=nsplit)
    assert _same_bits(got.f, motion[:, start:start + win])
    check_rule(got.p.t[..., :ch], got.f, fmt, f"window_input motion {fmt} x{nsplit}")
    only = ops.window_input(motion, zeros, None, emb0, start, win, 0, nsplit=nsplit, f32=False)
    assert _same_bits(only.p.t[..., :ch], got.p.t[..., :ch])
    for k in range(-(-EDGE.size // ch)):                 # every edge value once as an embedding column
        emb = torch.from_numpy(np.resize(np.roll(EDGE, -k * ch), ch).astype(np.float32)).cuda()
        got = ops.window_input(motion, ones, None, emb, start, win, 0, nsplit=nsplit)
        assert _same_bits(got.f, emb.expand(bs, win, ch))
        check_rule(got.p.t[..., :ch], got.f, fmt, f"window_input embedding {k} {fmt} x{nsplit}")
    pre = 3
    seed = edge_tensor((bs, 5, ch), seed=23)[:, 2:]
    got = ops.window_input(None, None, seed, emb0, 0, win, pre, nsplit=nsplit, shape=(bs, total, ch))
    assert _same_bits(got.f[:, :pre], seed) and _same_bits(got.f[:, pre:], emb0.expand(bs, win - pre, ch))
    check_rule(got.p.t[..., :ch], got.f, fmt, f"window_input defaults {fmt} x{nsplit}")


# ------------------------------------------------------------------------------------------------------------------
# arithmetic producers: planes = the rule applied to the same call's fp32 output
# ------------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("nsplit", SPLITS)
def test_add_layernorm_planes(ops, fmt, nsplit):
    for ch in (256, 768):
        for rows in (1, 301):
            x, r = _rand(rows, ch, seed=31, scale=3.0), _rand(rows, ch, seed=32)
            g, b = _rand(ch, seed=33, scale=300.0), _rand(ch, seed=34)       # outputs up to and past the fp16 edge
            for bad in (False, True):
                xx = _with_nonfinite(x, rows // 2) if bad else x
                tag = f"add_layernorm {fmt} x{nsplit} {rows}x{ch}{' nan/inf' if bad else ''}"
                got = ops.add_layernorm(xx, r, g, b, nsplit=nsplit)
                check_rule(got.p.t[..., :ch].reshape(nsplit, rows, ch), got.f, fmt, tag)
                only = ops.add_layernorm(xx, r, g, b, nsplit=nsplit, f32=False)
                assert _same_bits(only.p.t[..., :ch], got.p.t[..., :ch]), tag
                if bad:
                    _nonfinite_reaches(got.f[rows // 2], tag)


@pytest.mark.parametrize("nsplit", SPLITS)
def test_add_rows_planes(ops, fmt, nsplit):
    bs, t, ch = 3, 61, 768
    x, pe, spk = _rand(bs, t, ch, seed=35), _rand(128, ch, seed=36, scale=300.0), _rand(bs, ch, seed=37)
    for bad in (False, True):
        xx = _with_nonfinite(x, 70) if bad else x
        tag = f"add_rows {fmt} x{nsplit}{' nan/inf' if bad else ''}"
        got = ops.add_rows(xx, pe, spk, ops.ROW_SPK, ops.ROW_PE, bs, t, ch, nsplit=nsplit)
        check_rule(got.p.t[..., :ch], got.f, fmt, tag)
        only = ops.add_rows(xx, pe, spk, ops.ROW_SPK, ops.ROW_PE, bs, t, ch, nsplit=nsplit, f32=False)
        assert _same_bits(only.p.t[..., :ch], got.p.t[..., :ch]), tag
        if bad:
            _nonfinite_reaches(got.f, tag)


@pytest.mark.parametrize("bs,tq,tk", [(5, 64, 64), (3, 60, 60), (2, 11, 12), (2, 1, 1)])
@pytest.mark.parametrize("nsplit", SPLITS)
def test_attention_f32_planes(ops, fmt, nsplit, bs, tq, tk):
    """The fp32 attention kernel on column slices of the packed q|k|v and k|v projections (the shapes of
    test_kernels_gpu.py::test_attention)."""
    E, H, hd = 768, 4, 192
    qkv = _rand(bs * tq, 3 * E, seed=40, scale=2.0)
    kv = _rand(bs * tk, 2 * E, seed=41, scale=2.0)
    for bad in (False, True):
        q = _with_nonfinite(qkv, tq // 2, cols=(5, 400)) if bad else qkv
        tag = f"attention {fmt} x{nsplit} {bs}x{tq}x{tk}{' nan/inf' if bad else ''}"
        got = ops.attention(q[:, :E], kv[:, :E], kv[:, E:], bs, H, tq, tk, hd, nsplit=nsplit)
        check_rule(got.p.t[..., :E].reshape(nsplit, bs * tq, E), got.f, fmt, tag)
        only = ops.attention(q[:, :E], kv[:, :E], kv[:, E:], bs, H, tq, tk, hd, nsplit=nsplit, f32=False)
        assert _same_bits(only.p.t[..., :E], got.p.t[..., :E]), tag
        if bad:
            _nonfinite_reaches(got.f[tq // 2], tag)


def _stem(ops, audio, n, ws, bs, windows, n_samples, w, stride, pad, nsplit, fmt_bit):
    """pm_wav_stem_f32 writing fp32 y1 and its planes in the same call."""
    from pantomatrix_b200 import _lib
    w1, b1, wd, bd = w
    cout, ks = w1.shape
    rows_out = (n_samples + 2 * pad - ks) // stride + 1
    sc = torch.empty(bs * windows, rows_out, cout, device="cuda")
    y1 = torch.empty_like(sc)
    pl = ops._new_planes(nsplit, (bs * windows, rows_out), cout, audio.device)
    _lib.call("pm_wav_stem_f32", audio.data_ptr(), n, ws, bs, windows, n_samples, w1.data_ptr(), b1.data_ptr(),
              wd.data_ptr(), bd.data_ptr(), cout, ks, stride, pad, rows_out, 0.01, y1.data_ptr(), sc.data_ptr(),
              pl.t.data_ptr(), pl.t.stride(0), pl.t.stride(2), nsplit | fmt_bit, torch.cuda.current_stream().cuda_stream)
    return y1, sc, pl


@pytest.mark.parametrize("nsplit", SPLITS)
@pytest.mark.parametrize("cout", [32, 64])
def test_wav_stem_planes(ops, fmt, nsplit, cout):
    """Both stem widths, the stride-5 path and the generic one (stride 4), every format and split count (the pair
    store for two fp16 planes, the scalar store otherwise); the planes-only call through ops.wav_stem writes the same
    planes and the same downsample branch."""
    bs, n, windows, ws, ns_ = 2, 7000, 2, 2500, 4321
    w = (_rand(cout, 15, seed=42, scale=40.0), _rand(cout, seed=43, scale=0.1), _rand(cout, 15, seed=44, scale=0.5),
         _rand(cout, seed=45, scale=0.1))
    audio = _rand(bs, n, seed=46, scale=0.1)
    fmt_bit = ops.FMT_F16 if fmt == ps.FP16 else 0
    for stride, pad in ((5, 1600), (4, 3)):
        for bad in (False, True):
            au = _with_nonfinite(audio, 1, cols=(3000, 3040)) if bad else audio
            tag = f"wav_stem {fmt} x{nsplit} cout {cout} stride {stride}{' nan/inf' if bad else ''}"
            y1, sc, pl = _stem(ops, au, n, ws, bs, windows, ns_, w, stride, pad, nsplit, fmt_bit)
            check_rule(pl.t[..., :cout], y1, fmt, tag)
            only, sc2 = ops.wav_stem(au, n, ws, bs, windows, ns_, *w, stride=stride, pad=pad, slope=0.01, nsplit=nsplit)
            assert _same_bits(only.t[..., :cout], pl.t[..., :cout]) and _same_bits(sc2, sc), tag
            if bad:
                _nonfinite_reaches(y1, tag)


FK_COEF = 300 + 100 + 486          # body_model.N_COEF: importing body_model would pull in the whole EMAGE engine
FK_ALL_JOINTS = (1 << 55) - 1


def _fk_tables(rng):
    """Random FK tables of the SMPL-X joint tree (the kernel reads nothing else of a body model): joints ordered by
    depth and the start of each level, as body_model._levels builds them."""
    from synthetic_models import SMPLX_PARENTS
    parents = np.array(SMPLX_PARENTS, dtype=np.int64)
    depth = np.zeros(55, dtype=np.int64)
    for i in range(1, 55):
        depth[i] = depth[parents[i]] + 1
    order = np.argsort(depth, kind="stable")
    start = np.searchsorted(depth[order], np.arange(depth.max() + 2))
    f32 = lambda x: torch.from_numpy(np.asarray(x, np.float32)).cuda()
    i32 = lambda x: torch.from_numpy(np.asarray(x, np.int32)).cuda()
    return (f32(rng.normal(0, 0.3, 165)), f32(rng.normal(0, 0.01, (400, 165))), f32(rng.normal(0, 0.1, 165)),
            i32(parents), i32(order), i32(start))


@pytest.mark.parametrize("nsplit", SPLITS)
def test_smplx_fk_operand_row(ops, fmt, nsplit):
    """The vertex GEMM's operand row (betas | expression | pose features) written as fp32 `feat` and as planes in one
    call; the expression columns carry the finite edge values."""
    from body_cases import random_poses
    rng = np.random.default_rng(50)
    tables = _fk_tables(rng)
    dtype = torch.bfloat16 if fmt == ps.BF16 else torch.float16
    B, T = 2, 37
    poses = torch.from_numpy(random_poses(rng, B * T).astype(np.float32)).cuda().view(B, T, 165)
    betas = torch.from_numpy(rng.normal(0, 1, (B, 300)).astype(np.float32)).cuda()
    expr = edge_tensor((B, T, 100), seed=51)
    expr = torch.where(torch.isfinite(expr), expr, torch.zeros_like(expr))
    transl = _rand(B, T, 3, seed=52)
    rows = B * T
    for bad in (False, True):
        ex = _with_nonfinite(expr, 40, cols=(3, 60)) if bad else expr
        po = _with_nonfinite(poses, 41, cols=(10, 100)) if bad else poses
        tag = f"smplx_fk {fmt} x{nsplit}{' nan/inf' if bad else ''}"
        joints = torch.empty(rows, 55, 3, device="cuda")
        rel = torch.empty(rows, 55, 12, device="cuda")
        feat = torch.empty(rows, ops._round_up(FK_COEF, 8), device="cuda")
        planes = ops._new_planes(nsplit, (1, rows), FK_COEF, poses.device, dtype=dtype)
        ops.smplx_fk(po, betas, ex, transl, FK_ALL_JOINTS, tables, joints, rel, feat, planes)
        check_rule(planes.t[:, 0, :, :FK_COEF], feat[:, :FK_COEF], fmt, tag)
        only = ops._new_planes(nsplit, (1, rows), FK_COEF, poses.device, dtype=dtype)
        ops.smplx_fk(po, betas, ex, transl, FK_ALL_JOINTS, tables, joints, rel, None, only)
        assert _same_bits(only.t[..., :FK_COEF], planes.t[..., :FK_COEF]), tag
        if bad:
            _nonfinite_reaches(feat[40:42, :FK_COEF], tag)


def _attention_tc_into(ops, args, planes, out):
    """pm_attention_tc writing fp32 `out` and the given planes (any row stride) in one call."""
    from pantomatrix_b200 import _lib
    q, q_col0, k, k_col0, v, v_col0, batch, heads, tq, tk, hd = args
    _lib.call("pm_attention_tc",
              q.t.data_ptr(), q.t.stride(0), q.t.stride(1), q.t.stride(2), q.ch, q_col0,
              k.t.data_ptr(), k.t.stride(0), k.t.stride(1), k.t.stride(2), k.ch, k_col0,
              v.t.data_ptr(), v.t.stride(0), v.t.stride(1), v.t.stride(2), v.ch, v_col0,
              out.data_ptr(), heads * hd, batch, heads, tq, tk, hd, *ops._pargs(planes),
              torch.cuda.current_stream().cuda_stream)


@pytest.mark.parametrize("bs,tq,tk", [(3, 64, 64), (2, 11, 12), (2, 1, 1)])
@pytest.mark.parametrize("nsplit", [1, 2])
def test_attention_tc_planes(ops, nsplit, bs, tq, tk):
    """Tensor-core attention (fp16 planes only, at most two): planes with an even row stride take the pair store, an
    odd row stride the scalar store; both, and the planes-only call, follow the rule."""
    E, H, hd = 768, 4, 192
    ops.set_plane_format("fp16")
    qkv = _rand(bs, tq, 3 * E + 8, seed=60, scale=2.0)
    kv = _rand(bs, tk, 2 * E + 8, seed=61, scale=2.0)
    for bad in (True, False):
        qq = _with_nonfinite(qkv, tq // 2, cols=(13, 400)) if bad else qkv          # heads 0 and 2 of Q
        qp, kvp = ops.split_bf16(qq, 2), ops.split_bf16(kv, 2)
        args = (qp, 8, kvp, 0, kvp, E, bs, H, tq, tk, hd)
        for ld in (E, E + 1):
            tag = f"attention_tc x{nsplit} {bs}x{tq}x{tk} ld {ld}{' nan/inf' if bad else ''}"
            pl = ops.Planes(torch.full((nsplit, bs, tq, ld), 7.0, device="cuda", dtype=torch.float16), tq, E)
            out = torch.empty(bs * tq, E, device="cuda")
            _attention_tc_into(ops, args, pl, out)
            check_rule(pl.t[..., :E].reshape(nsplit, bs * tq, E), out, ps.FP16, tag)
            if bad:
                _nonfinite_reaches(out[tq // 2], tag)
        only = ops.attention_tc(*args, nsplit=nsplit, f32=False)
        assert _same_bits(only.p.t[..., :E], pl.t[..., :E]), tag


@pytest.mark.parametrize("nsplit", SPLITS)
def test_tapgemm_tc_epilogue_planes(ops, fmt, nsplit):
    """The tap-GEMM epilogue: out_nsplit from 1 up to the operand split, ragged cout (the per-element tail), an fp32 `out`
    column view with an odd row stride (every element through the scalar store), both forced N tiles, zeroed slack rows
    after the last clip."""
    from pantomatrix_b200 import ops as o
    batch, rows, cin, taps, pad = 3, 45, 96, 3, 1
    rows_out = rows + 2 * pad - taps + 1
    for cout in (61, 70, 200):
        x = _rand(batch, rows, cin, seed=70, scale=4.0)
        w = _rand(taps, cout, cin, seed=71, scale=8.0 / math.sqrt(cin * taps))
        bias, res = _rand(cout, seed=72), _rand(batch, rows_out, cout, seed=73)
        pw = o.PackedW(w, nsplit)
        ldo = cout + 2 + (1 - cout % 2)                           # odd
        for bad in (False, True):
            a = o.split_bf16(_with_nonfinite(x, rows + 7) if bad else x, nsplit)
            for out_ns in range(1, nsplit + 1):
                for tile in ((64, 128) if cout > 64 else (64,)):
                    for view in (False, True):
                        tag = (f"tapgemm_tc {fmt} x{nsplit} -> x{out_ns} cout {cout} tile {tile}"
                               f"{' odd ldo view' if view else ''}{' nan/inf' if bad else ''}")
                        out = (torch.zeros(batch, rows_out, ldo, device="cuda")[..., 1:1 + cout] if view else None)
                        kw = dict(rows_out=rows_out, pad=pad, act=o.ACT_LEAKY, slope=0.2, residual=res, tile=tile)
                        f, p = o.tapgemm_tc(a, pw, bias, out_nsplit=out_ns, out=out, out_slack=3, **kw)
                        check_rule(p.t[..., :cout], f, fmt, tag)
                        assert not bool(slack_rows(p).view(torch.int16).any()), f"{tag}: slack rows were written"
                        _, p_only = o.tapgemm_tc(a, pw, bias, out_nsplit=out_ns, want_f32=False, **kw)
                        assert _same_bits(p_only.t[..., :cout], p.t[..., :cout]), tag
                        if bad:
                            _nonfinite_reaches(f[1], tag)

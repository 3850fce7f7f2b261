"""The tensor-core tap-GEMM's two epilogues give the same bytes.  Where every output view has a 16-byte aligned base
and strides, the epilogue finishes each value in registers and stores the tile by TMA; any other view, and every call
with ops.tapgemm_tc(..., store_loop=True), takes the per-element store loop.  Each case runs both and compares the fp32
output and the planes bit for bit, NaN positions included, at both N tiles and in both plane formats.

The cases are the EMAGE step's shapes (the window loop's 2048-row Linears, the k = 3 convs of 32 clips x 64 rows that
pack two clips per tile, the WavEncoder's k = 15 convs and its stride-6 view), ragged rows and columns, every operand
and output split, in-place residuals, outputs written into a window's rows and into a column slice of a wider
tensor, an unaligned column slice (which must fall back) and an fp16 overflow that must still come out as NaN."""
import math

import pytest
import torch

from helpers import bf16_planes_by_default  # noqa: F401

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ops():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    from pantomatrix_b200 import _lib, ops as o
    _lib.load()
    return o


def _rand(*shape, seed=0, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(*shape, generator=g) * scale).cuda()


def _bits(t):
    return t.view(torch.int32) if t.dtype == torch.float32 else t.view(torch.int16)


def _same(got, want, tag):
    assert got.shape == want.shape, tag
    diff = _bits(got) != _bits(want)
    assert not bool(diff.any()), f"{tag}: {int(diff.sum())} of {diff.numel()} elements differ"


def _run(ops, a, pw, bias, make_out=None, **kw):
    """(TMA-store result, store-loop result), each (fp32 buffer or None, valid plane region or None)."""
    res = []
    for loop in (False, True):
        buf = make_out() if make_out is not None else None
        view = buf[1] if buf is not None else None
        f, pl = ops.tapgemm_tc(a, pw, bias, store_loop=loop, out=view, **kw)
        torch.cuda.synchronize()
        whole = buf[0] if buf is not None else f
        planes = None if pl is None else pl.t[:, :, :kw["rows_out"], :pw.cout]
        res.append((whole, planes))
    return res


def _compare(res, tag):
    (f0, p0), (f1, p1) = res
    assert (f0 is None) == (f1 is None) and (p0 is None) == (p1 is None), tag
    if f0 is not None:
        _same(f0, f1, tag + " fp32")
    if p0 is not None:
        _same(p0, p1, tag + " planes")


def _problem(batch, rows, cin, cout, taps, pad, seed=0):
    x = _rand(batch, rows, cin, seed=seed + 1)
    w = _rand(taps, cout, cin, seed=seed + 2, scale=1 / math.sqrt(cin * taps))
    bias = _rand(cout, seed=seed + 3, scale=0.1)
    rows_out = rows + 2 * pad - taps + 1
    res = _rand(batch, rows_out, cout, seed=seed + 4)
    return x, w, bias, res, rows_out


FORMATS = [("bf16", 1), ("bf16", 3), ("fp16", 2)]

SHAPES = [
    # batch, rows, cin, cout, taps, pad
    (1, 2048, 768, 768, 1, 0),         # window loop: attention out projection / FFN
    (1, 2048, 768, 1536, 1, 0),
    (1, 2048, 768, 2304, 1, 0),        # packed q|k|v
    (1, 2048, 1536, 768, 1, 0),        # FFN linear2
    (32, 64, 256, 256, 3, 1),          # k = 3 conv, 32 clips x 64 rows: two clips per 128-row tile
    (7, 13, 256, 61, 3, 1),            # 8 clips per tile, ragged batch and cout
    (128, 1241, 64, 64, 15, 7),        # WavEncoder k = 15 conv, 64 -> 64
    (1, 300, 256, 200, 1, 0),          # ragged rows, ragged last N tile
    (3, 150, 64, 96, 15, 7),           # ragged cout at BN = 64
]


def _tiles(cout):
    return (64, 128) if cout > 64 else (64,)


@pytest.mark.parametrize("fmt,ns", FORMATS)
@pytest.mark.parametrize("shape", SHAPES, ids=lambda s: "x".join(map(str, s)))
def test_shapes(ops, shape, fmt, ns):
    ops.set_plane_format(fmt)
    batch, rows, cin, cout, taps, pad = shape
    x, w, bias, res, rows_out = _problem(*shape)
    a, pw = ops.split_bf16(x, ns), ops.PackedW(w, ns)
    for tile in _tiles(cout):
        if tile == 128 and pw.w_rows % 128:
            continue
        for mode in ("f32", "planes", "both"):
            kw = dict(rows_out=rows_out, pad=pad, act=ops.ACT_LEAKY, slope=0.2, act_cols=cout // 2 + 1, residual=res,
                      want_f32=mode != "planes", out_nsplit=0 if mode == "f32" else ns, tile=tile)
            _compare(_run(ops, a, pw, bias, **kw), f"{shape} {fmt}x{ns} BN={tile} {mode}")
            kw.update(residual=None, act=ops.ACT_RELU)
            _compare(_run(ops, a, pw, None, **kw), f"{shape} {fmt}x{ns} BN={tile} {mode} no bias / residual")


@pytest.mark.parametrize("fmt", ["bf16", "fp16"])
@pytest.mark.parametrize("ns", [1, 2, 3])
@pytest.mark.parametrize("out_ns", [1, 2, 3])
def test_splits(ops, fmt, ns, out_ns):
    """Every operand split against every output split, fp32 beside the planes and planes alone.  Three planes
    beside fp32 and a residual do not fit the ring at BN = 128 and take the store loop either way."""
    ops.set_plane_format(fmt)
    shape = (2, 300, 320, 200, 3, 1)
    x, w, bias, res, rows_out = _problem(*shape, seed=10)
    a, pw = ops.split_bf16(x, ns), ops.PackedW(w, ns)
    for tile in (64, 128):
        for want_f32 in (True, False):
            kw = dict(rows_out=rows_out, pad=1, act=ops.ACT_LEAKY, slope=0.1, residual=res, want_f32=want_f32,
                      out_nsplit=out_ns, tile=tile)
            _compare(_run(ops, a, pw, bias, **kw), f"{fmt} {ns}->{out_ns} BN={tile} f32={want_f32}")


@pytest.mark.parametrize("fmt,ns", FORMATS)
@pytest.mark.parametrize("tile", [64, 128])
def test_inplace_residual(ops, fmt, ns, tile):
    """out is the residual: each tile's residual is in shared memory before any of its stores."""
    ops.set_plane_format(fmt)
    x, w, bias, res, rows_out = _problem(1, 2048, 768, 768, 1, 0, seed=20)
    a, pw = ops.split_bf16(x, ns), ops.PackedW(w, ns)
    got = []
    for loop in (False, True):
        y = res.clone()
        ops.tapgemm_tc(a, pw, bias, rows_out=rows_out, residual=y, out=y, out_nsplit=ns, tile=tile, store_loop=loop)
        torch.cuda.synchronize()
        got.append(y)
    _same(got[0], got[1], f"in place {fmt}x{ns} BN={tile}")


@pytest.mark.parametrize("fmt,ns", FORMATS)
@pytest.mark.parametrize("tile", [64, 128])
def test_output_views(ops, fmt, ns, tile):
    """fp32 output written into views of a larger tensor, whose other elements must stay as they were: a window's
    rows of an accumulated result (TMA path), a 16-byte aligned column slice (TMA path) and a column slice at a
    4-byte offset with an odd row stride (store loop)."""
    ops.set_plane_format(fmt)
    batch, rows, cin, cout = 4, 64, 256, 256
    x, w, bias, res, rows_out = _problem(batch, rows, cin, cout, 3, 1, seed=30)
    a, pw = ops.split_bf16(x, ns), ops.PackedW(w, ns)
    total = 5 * rows_out

    def window():
        big = torch.full((batch, total, cout), float("nan"), device="cuda")
        return big, big[:, 2 * rows_out:3 * rows_out]

    def columns():
        big = torch.full((batch, rows_out, cout + 192), -7.0, device="cuda")
        return big, big[:, :, 128:128 + cout]

    def unaligned():
        big = torch.full((batch, rows_out, cout + 5), -7.0, device="cuda")
        return big, big[:, :, 1:1 + cout]

    for name, make in (("window", window), ("columns", columns), ("unaligned", unaligned)):
        for resid in (None, res):
            kw = dict(rows_out=rows_out, pad=1, act=ops.ACT_RELU, residual=resid, out_nsplit=ns, tile=tile)
            _compare(_run(ops, a, pw, bias, make_out=make, **kw), f"{name} {fmt}x{ns} BN={tile} res={resid is not None}")


@pytest.mark.parametrize("fmt,ns", FORMATS)
def test_strided_view(ops, fmt, ns):
    """The WavEncoder's stride-6 conv: a stride-1 GEMM over the (rows / 6, 6 C) view of its input planes."""
    ops.set_plane_format(fmt)
    batch, rows, c, cout, s = 8, 6 * 400, 64, 64, 6
    x = _rand(batch, rows, c, seed=40)
    w = _rand(-(-15 // s), cout, s * c, seed=41, scale=1 / math.sqrt(15 * c))
    bias = _rand(cout, seed=42, scale=0.1)
    a, pw = ops.split_bf16(x, ns, slack_rows=s), ops.PackedW(w, ns)
    rows_out = (rows - 15) // s + 1
    res = _rand(batch, rows_out, cout, seed=43)
    kw = dict(rows_out=rows_out, act=ops.ACT_LEAKY, slope=0.3, residual=res, out_nsplit=ns,
              a_view=(-(-rows // s), s * c, s * c))
    _compare(_run(ops, a, pw, bias, **kw), f"stride 6 {fmt}x{ns}")


@pytest.mark.parametrize("tile", [64, 128])
def test_fp16_overflow_is_nan(ops, tile):
    """Operands past the fp16 range leave inf - inf = NaN in the accumulators: both epilogues must keep every NaN
    (the compare-select activation does not turn it into 0) in the fp32 output and the planes."""
    ops.set_plane_format("fp16")
    x, w, bias, res, rows_out = _problem(1, 512, 256, 256, 1, 0, seed=50)
    x[0, 10:20] *= 1e4                      # x 64 pre-scale: past 65504
    a, pw = ops.split_bf16(x, 2), ops.PackedW(w, 2)
    kw = dict(rows_out=rows_out, act=ops.ACT_RELU, residual=res, out_nsplit=2, tile=tile)
    res_ = _run(ops, a, pw, bias, **kw)
    assert bool(torch.isnan(res_[0][0]).any()), "the overflow must surface as NaN"
    _compare(res_, f"fp16 overflow BN={tile}")

"""Residual sources of the tensor-core tap-GEMM's epilogue.  A residual view TMA can describe (16-byte base, row and
clip strides a multiple of 4 floats) is loaded as one tile into the operand ring while the last k-blocks compute;
any other view is read per element from global memory.  The arithmetic is the same, so both must give the same bits:
each case runs the GEMM once on a misaligned copy of the residual (the per-element reference) and holds the
TMA-loaded contiguous, row-and-clip-strided and in-place (residual is out) views to it, fp32 output and planes.

The cases vary the k-block count against every ring depth (the residual tile takes the ring slots of the oldest
k-blocks in flight), pack several clips per tile (a 3-D box clipped at the batch) and leave ragged rows and a
ragged last N tile (zero-filled box)."""
import math

import pytest
import torch

from helpers import bf16_planes_by_default  # noqa: F401
from test_tapgemm_tc_gpu import _rand

pytestmark = pytest.mark.gpu

FORMATS = [("bf16", 1), ("bf16", 2), ("bf16", 3), ("fp16", 2)]

CASES = [
    # batch, rows, cin, cout, taps, pad
    (1, 300, 256, 200, 1, 0),      # ragged rows, ragged last N tile
    (7, 16, 128, 96, 3, 1),        # 8 clips per 128-row tile, batch not a multiple of 8
    (3, 150, 64, 64, 15, 7),       # WavEncoder conv2 (64-column tiles only)
    (2, 200, 64, 128, 1, 0),       # one k-block: the residual load runs beside the only MMAs
    (2, 200, 320, 128, 1, 0),      # 5 k-blocks
    (1, 256, 448, 256, 1, 0),      # 7 k-blocks
    (2, 90, 192, 256, 3, 1),       # 9 k-blocks over 3 taps
]


@pytest.fixture(scope="module")
def ops():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    from pantomatrix_b200 import _lib, ops as o
    _lib.load()
    return o


@pytest.fixture
def fmt_ops(ops, request):
    ops.set_plane_format(request.param)
    return ops


def _misaligned(t):
    """t's values in a column view at a 4-byte offset of a tensor with an odd row stride: TMA cannot describe it."""
    b, r, c = t.shape
    big = torch.zeros(b, r, c + 1, device=t.device)             # c % 4 == 0: odd row stride
    v = big[:, :, 1:1 + c]
    v.copy_(t)
    return v


def _strided(t):
    """t's values in a row-and-column view of a larger tensor: row stride c + 8, clip stride (r + 3) (c + 8), both
    multiples of 4 floats, and a 16-byte aligned base (c % 4 == 0)."""
    b, r, c = t.shape
    big = torch.full((b, r + 3, c + 8), float("nan"), device=t.device)
    v = big[:, 2:2 + r, 4:4 + c]
    v.copy_(t)
    return v


@pytest.mark.parametrize("fmt_ops,nsplit", FORMATS, indirect=["fmt_ops"])
@pytest.mark.parametrize("case", CASES)
def test_tma_residual_matches_per_element(fmt_ops, case, nsplit):
    ops = fmt_ops
    batch, rows, cin, cout, taps, pad = case
    assert cout % 4 == 0
    x = _rand(batch, rows, cin, seed=41)
    pw = ops.PackedW(_rand(taps, cout, cin, seed=42, scale=1 / math.sqrt(cin * taps)), nsplit)
    rows_out = rows + 2 * pad - taps + 1
    res = _rand(batch, rows_out, cout, seed=44)
    a = ops.split_bf16(x, nsplit)
    kw = dict(rows_out=rows_out, pad=pad, act=ops.ACT_LEAKY, slope=0.2, out_nsplit=nsplit)
    tiles = (64, 128) if pw.w_rows % 128 == 0 else (64,)
    for bias in (_rand(cout, seed=43, scale=0.1), None):
        for tile in tiles:
            tag = f"{case} nsplit={nsplit} BN={tile} bias={bias is not None}"
            want_f, want_p = ops.tapgemm_tc(a, pw, bias, residual=_misaligned(res), tile=tile, **kw)
            for name, r in (("contiguous", res), ("strided", _strided(res))):
                f, p = ops.tapgemm_tc(a, pw, bias, residual=r, tile=tile, **kw)
                assert torch.equal(f, want_f), f"{tag}: {name} residual, fp32 output differs from the per-element path"
                assert torch.equal(p.t[..., :cout], want_p.t[..., :cout]), f"{tag}: {name} residual, planes differ"
            inplace = res.clone()
            f, p = ops.tapgemm_tc(a, pw, bias, residual=inplace, out=inplace, tile=tile, **kw)
            assert f.data_ptr() == inplace.data_ptr()
            assert torch.equal(inplace, want_f), f"{tag}: in-place residual, fp32 output differs"
            assert torch.equal(p.t[..., :cout], want_p.t[..., :cout]), f"{tag}: in-place residual, planes differ"

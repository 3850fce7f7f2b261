"""N tile of the tensor-core tap-GEMM: 64- and 128-column tiles (and the automatic choice between them) must give
the same bits.  Each output element is summed by the same wgmma k16 steps in the same order whatever the tile width,
so a difference means the accumulation order changed.  Every shape of test_tapgemm_tc_gpu is run with the tile
forced both ways, and each result is also held to helpers.check_tapgemm's per-element bounds."""
import pytest
import torch

from helpers import bf16_planes_by_default, check_tapgemm, slack_rows  # noqa: F401
from test_tapgemm_tc_gpu import CASES, _inputs, _outside, _rand

pytestmark = pytest.mark.gpu

FORMATS = [("bf16", 1), ("bf16", 2), ("bf16", 3), ("fp16", 2)]


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


@pytest.mark.parametrize("fmt_ops,nsplit", FORMATS, indirect=["fmt_ops"])
@pytest.mark.parametrize("case", CASES)
def test_tiles_bit_identical(fmt_ops, case, nsplit):
    ops = fmt_ops
    x, w, bias, res, rows_out = _inputs(case)
    a = ops.split_bf16(x, nsplit)
    pw = ops.PackedW(w, nsplit)
    kw = dict(rows_out=rows_out, pad=case[5], act=ops.ACT_LEAKY, slope=0.2, residual=res, out_nsplit=nsplit)
    tiles = (0, 64, 128) if pw.w_rows % 128 == 0 else (0, 64)
    got = {tile: ops.tapgemm_tc(a, pw, bias, tile=tile, **kw) for tile in tiles}
    f64, p64 = got[64]
    kw.pop("out_nsplit")
    check_tapgemm(a, pw, bias, f64, p64, tag=f"{case} nsplit={nsplit} BN=64", **kw)
    for tile in tiles:
        f, p = got[tile]
        assert torch.equal(f, f64), f"tile {tile}: fp32 output differs from BN=64"
        assert torch.equal(p.t[..., :pw.cout], p64.t[..., :pw.cout]), f"tile {tile}: planes differ from BN=64"


@pytest.mark.parametrize("fmt_ops,nsplit", [("bf16", 3), ("fp16", 2)], indirect=["fmt_ops"])
def test_wide_tile_writes_only_its_views(fmt_ops, nsplit):
    """out= / residual= column views of wider tensors with odd row strides (ldo 301, ldr 277: the per-element
    epilogue), a ragged last 128-column tile (cout 200): both tiles write the view only, leave slack rows zero and
    agree bit for bit."""
    ops = fmt_ops
    batch, rows, cout = 3, 150, 200
    x = _rand(batch, rows, 128, seed=31)
    pw = ops.PackedW(_rand(3, cout, 128, seed=32, scale=0.05), nsplit)
    bias = _rand(cout, seed=33, scale=0.1)
    results = []
    for tile in (64, 128):
        big_out = _rand(batch, rows + 5, 301, seed=34)
        big_res = _rand(batch, rows + 2, 277, seed=35)
        out, res = big_out[:, 2:2 + rows, 13:13 + cout], big_res[:, 1:1 + rows, 3:3 + cout]
        base, mask = _outside(out)
        keep = base[mask].clone()
        res_before = big_res.clone()
        a = ops.split_bf16(x, nsplit)
        kw = dict(rows_out=rows, pad=1, act=ops.ACT_RELU, residual=res)
        got, pl = ops.tapgemm_tc(a, pw, bias, out=out, out_nsplit=nsplit, out_slack=8, tile=tile, **kw)
        assert torch.equal(base[mask], keep), f"BN={tile}: epilogue wrote outside the out= view"
        assert torch.equal(big_res, res_before)
        assert int(torch.count_nonzero(slack_rows(pl))) == 0
        check_tapgemm(a, pw, bias, out, pl, tag=f"strided views BN={tile}", **kw)
        results.append((out.clone(), pl.t[..., :cout].clone()))
    assert torch.equal(results[0][0], results[1][0]) and torch.equal(results[0][1], results[1][1])


def test_forced_wide_tile_needs_padded_weights(ops):
    """A 128-column tile reads 128 weight rows per tap: PackedW pads only cout > 64 to that, so forcing it on a
    64-row pack is refused instead of reading the next tap's rows."""
    from pantomatrix_b200._lib import PmError
    x = _rand(2, 50, 64, seed=36)
    pw = ops.PackedW(_rand(3, 64, 64, seed=37, scale=0.1), 2)
    assert pw.w_rows == 64
    a = ops.split_bf16(x, 2)
    with pytest.raises(PmError):
        ops.tapgemm_tc(a, pw, None, rows_out=50, pad=1, tile=128)
    auto, _ = ops.tapgemm_tc(a, pw, None, rows_out=50, pad=1)
    narrow, _ = ops.tapgemm_tc(a, pw, None, rows_out=50, pad=1, tile=64)
    assert torch.equal(auto, narrow)

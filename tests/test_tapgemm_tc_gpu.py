"""Tensor-core tap-GEMM (pm_tapgemm_tc) against a float64 restatement, for every split mode and the shapes the
EMAGE schedule issues: tall Linears, k=3 / k=15 convs with zero padding, clips packed 2..8 per 128-row tile,
ragged channel counts, fused bias / residual / partial activation, bf16 plane outputs.

Every output element is held to its own bound (helpers.tapgemm_reference): c_mode * (|A| @ |W|)_ij plus fp32 ulps
of bias, residual and result, so an error confined to small columns, one clip of a packed tile or a clip edge
cannot hide behind the largest value of the output."""
import math

import pytest
import torch

from helpers import bf16_planes_by_default, check_tapgemm, slack_rows  # noqa: F401

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


def _check(a, pw, bias, got, planes=None, tag="", **kw):
    used = check_tapgemm(a, pw, bias, got, planes, tag=tag, **kw)
    print(f"[{tag}] largest fraction of the per-element bound used: GEMM {used[0]:.3f}, plane split {used[1]:.3f}")
    return used


CASES = [
    # batch, rows, cin, cout, taps, pad[, decades the output columns' weight scales span]
    (1, 2048, 768, 2304, 1, 0),        # packed qkv projection
    (1, 2048, 1536, 768, 1, 0),        # FFN linear2 (K = 1536)
    (1, 1920, 256, 768, 1, 0),         # T=60 window
    (1, 37, 768, 256, 1, 0),           # ragged rows
    (32, 64, 337, 256, 3, 1),          # motion-encoder stem: ragged cin, 2 clips per tile
    (32, 64, 256, 256, 3, 1),
    (7, 16, 256, 61, 3, 1),            # seed decode: 8 clips per tile, ragged cout, batch not a multiple of NB
    (3, 300, 256, 106, 3, 1),          # full-length decode
    (5, 700, 64, 64, 15, 7),           # WavEncoder conv2 (BN = 64 tile)
    (4, 205, 128, 128, 15, 7),
    (2, 11, 256, 256, 3, 1),           # 11-frame tail window
    (4, 700, 32, 32, 15, 7),           # CaMN / DisCo WavEncoder: cin < one 64-channel k-block (TMA box wider than the tensor)
    (2, 45, 512, 78, 1, 0),            # CaMN body head (ragged cout)
    (2, 45, 403, 4096, 1, 0),          # LSTM input projection, both directions (ragged cin)
    (6, 40, 256, 192, 3, 1, 6),        # column weight scales over six decades, 2 clips per tile
    (1, 300, 768, 320, 1, 0, 6),       # ... tall Linear, ragged last N tile
    (1, 256, 4096, 128, 1, 0),         # long K: 64 k-blocks wrap the 8 / 4 / 2-stage ring 8 / 16 / 32 times
    (2, 100, 1024, 64, 15, 7),         # 240 k-blocks over 15 taps
]


def _inputs(case):
    batch, rows, cin, cout, taps, pad = case[:6]
    decades = case[6] if len(case) > 6 else 0
    x = _rand(batch, rows, cin, seed=1)
    w = _rand(taps, cout, cin, seed=2, scale=1 / math.sqrt(cin * taps))
    bias = _rand(cout, seed=3, scale=0.1)
    rows_out = rows + 2 * pad - taps + 1
    res = _rand(batch, rows_out, cout, seed=4)
    if decades:                       # column n scaled by 10^(-decades * (n % 7) / 6): every N tile spans all scales
        col = 10.0 ** (-decades * torch.arange(cout, device="cuda").remainder(7) / 6)
        w, bias, res = w * col[None, :, None], bias * col, res * col
    return x, w, bias, res, rows_out


def _run_case(ops, case, nsplit):
    taps, pad = case[4], case[5]
    x, w, bias, res, rows_out = _inputs(case)
    a = ops.split_bf16(x, nsplit)
    pw = ops.PackedW(w, nsplit)
    kw = dict(rows_out=rows_out, pad=pad, act=ops.ACT_LEAKY, slope=0.2, residual=res)
    got, planes = ops.tapgemm_tc(a, pw, bias, out_nsplit=nsplit, **kw)
    _check(a, pw, bias, got, planes, tag=f"{case} nsplit={nsplit} {ops.plane_format()}", **kw)


@pytest.mark.parametrize("nsplit", [1, 2, 3])
@pytest.mark.parametrize("case", CASES)
def test_tapgemm_tc_matches_fp64(ops, case, nsplit):
    _run_case(ops, case, nsplit)


@pytest.mark.parametrize("case", CASES)
def test_tapgemm_tc_fp16_planes(ops, case):
    """Two IEEE fp16 planes, 3 products: the accuracy class of bf16x6 (weights packed pre-scaled by a power of two,
    undone by acc_scale in the epilogue)."""
    ops.set_plane_format("fp16")
    _run_case(ops, case, 2)


def test_partial_activation_and_column_slices(ops):
    """conv1 | downsample fused along N: activation on the first half only; consumers read column slices."""
    x = _rand(3, 200, 128, seed=5)
    w = _rand(1, 128, 128, seed=6, scale=0.1)
    pw = ops.PackedW(w, 3)
    a = ops.split_bf16(x, 3)
    got, _ = ops.tapgemm_tc(a, pw, None, rows_out=200, act=ops.ACT_RELU, act_cols=64)
    _check(a, pw, None, got, rows_out=200, act=ops.ACT_RELU, act_cols=64, tag="act_cols")
    # a column slice of a wider fp32 tensor as the A operand
    a2 = ops.split_bf16(got[:, :, 64:], 3)
    pw2 = ops.PackedW(_rand(1, 64, 64, seed=7, scale=0.1), 3)
    got2, _ = ops.tapgemm_tc(a2, pw2, None, rows_out=200)
    _check(a2, pw2, None, got2, rows_out=200, tag="column slice")


@pytest.mark.parametrize("C,cout", [(64, 64), (32, 64)])
def test_strided_conv_as_reshaped_stride1(ops, C, cout):
    """k=15 stride-6 conv == 3-tap stride-1 conv over the (L/6, 6*C) view with zero-padded taps."""
    b, L, s = 3, 745, 6
    x = _rand(b, L, C, seed=8)
    w = _rand(cout, C, 15, seed=9, scale=1 / math.sqrt(C * 15))
    taps = -(-15 // s)
    wp = torch.zeros(taps, cout, s * C, device="cuda")
    for k in range(15):
        wp[k // s, :, (k % s) * C:(k % s + 1) * C] = w[:, :, k]
    a = ops.split_bf16(x, 3, slack_rows=s)
    rows_v = -(-L // s)
    rows_out = (L - 15) // s + 1
    pw = ops.PackedW(wp, 3)
    got, _ = ops.tapgemm_tc(a, pw, None, rows_out=rows_out, a_view=(rows_v, s * C, s * C))
    _check(a, pw, None, got, rows_out=rows_out, a_view=(rows_v, s * C, s * C), tag=f"stride-6 view C={C}")
    want = torch.nn.functional.conv1d(x.double().transpose(1, 2), w.double(), stride=s).transpose(1, 2)
    assert (got.double() - want).abs().max() <= 5e-6 * want.abs().max()     # the view is the strided conv


@pytest.mark.parametrize("scale,tol", [(1.0, 5e-6), (0.05, 5e-6), (1e-3, 3e-4)])
def test_fp16_planes_small_activations(ops, scale, tol):
    """Tensor cores may flush fp16 SUBNORMAL operands, so the second plane of an element would be lost once it drops
    below 2^-14.  Activation planes are therefore pre-scaled by 64 (exact): LayerNorm-sized
    and 20x smaller activations keep the fp32-class accuracy; only tensors that are tiny as a whole (1e-3) degrade to
    single-plane fp16 accuracy (2^-11) - no tensor of this model is that small (smallest GEMM input: ~0.05)."""
    ops.set_plane_format("fp16")
    x = _rand(1, 256, 768, seed=11, scale=scale)
    w = _rand(1, 256, 768, seed=12, scale=1 / math.sqrt(768))
    want = torch.nn.functional.linear(x.double(), w[0].double())
    a, pw = ops.split_bf16(x, 2), ops.PackedW(w, 2)
    got, _ = ops.tapgemm_tc(a, pw, None, rows_out=256)
    err = (got.double() - want).abs().max().item()
    assert err <= tol * float(want.abs().max()), err
    _check(a, pw, None, got, rows_out=256, tag=f"fp16 activations x{scale}")


@pytest.mark.parametrize("fmt,nsplit", [("bf16", 1), ("bf16", 2), ("bf16", 3), ("fp16", 2)])
def test_clips_are_independent(ops, fmt, nsplit):
    """7 clips packed 8 per 128-row tile (R = 16) give bit-identical rows to each clip alone (R = 128) and to the batch
    in reverse order; a Linear over the clips as one tall matrix (Planes.flat) equals the per-clip call."""
    ops.set_plane_format(fmt)
    x = _rand(7, 16, 256, seed=13)
    pw = ops.PackedW(_rand(3, 96, 256, seed=14, scale=1 / 28), nsplit)
    bias, res = _rand(96, seed=15, scale=0.1), _rand(7, 16, 96, seed=16)
    kw = dict(rows_out=16, pad=1, act=ops.ACT_LEAKY, slope=0.2)
    a = ops.split_bf16(x, nsplit)
    got, pl = ops.tapgemm_tc(a, pw, bias, residual=res, out_nsplit=nsplit, **kw)
    _check(a, pw, bias, got, pl, residual=res, tag="7 packed clips", **kw)
    rev, pl_rev = ops.tapgemm_tc(ops.split_bf16(x.flip(0), nsplit), pw, bias, residual=res.flip(0), out_nsplit=nsplit, **kw)
    assert torch.equal(rev.flip(0), got) and torch.equal(pl_rev.t.flip(1)[..., :96], pl.t[..., :96])
    for b in range(7):
        one, _ = ops.tapgemm_tc(ops.split_bf16(x[b:b + 1], nsplit), pw, bias, residual=res[b:b + 1], **kw)
        assert torch.equal(one, got[b:b + 1]), b
    # 1x1 Linear: the flat tall matrix against the per-clip (packed) call
    pl1 = ops.PackedW(_rand(1, 80, 256, seed=17, scale=1 / 16), nsplit)
    per_clip, _ = ops.tapgemm_tc(a, pl1, bias[:80], rows_out=16)
    flat, _ = ops.tapgemm_tc(a.flat(), pl1, bias[:80], rows_out=7 * 16)
    assert torch.equal(flat.view(7, 16, 80), per_clip)
    _check(a.flat(), pl1, bias[:80], flat, rows_out=7 * 16, tag="flat Linear")


def test_prefetch_does_not_change_results(ops):
    """The producer warp's L2 prefetch of the next GEMM's weights (per-CTA byte shares) must not touch the result:
    byte counts 0, 16, 4 KB + 48, a whole PackedW, and fewer than 128 bytes per CTA (most CTAs get an empty share)."""
    x = _rand(1, 1024, 768, seed=18)
    pw = ops.PackedW(_rand(1, 768, 768, seed=19, scale=1 / 28), 3)
    nxt = ops.PackedW(_rand(1, 2304, 768, seed=20, scale=1 / 28), 3)
    a = ops.split_bf16(x, 3)
    want, pl = ops.tapgemm_tc(a, pw, None, rows_out=1024, out_nsplit=3)
    ncta = (1024 // 128) * (768 // 64)
    raw = nxt.t.view(-1).view(torch.uint8)
    for n in (0, 16, 4096 + 48, raw.numel(), 128 * ncta - 16, 48):
        got, pl2 = ops.tapgemm_tc(a, pw, None, rows_out=1024, out_nsplit=3, prefetch=raw[:n])
        assert torch.equal(got, want) and torch.equal(pl2.t[..., :768], pl.t[..., :768]), n
    got, _ = ops.tapgemm_tc(a, pw, None, rows_out=1024, prefetch=nxt.t)
    assert torch.equal(got, want)
    _check(a, pw, None, want, pl, rows_out=1024, tag="prefetch")


def _outside(view):
    """(base, mask) of the storage behind `view`: mask is True outside the view (what a call writing `view` must keep)."""
    base = torch.empty(0, dtype=view.dtype, device=view.device).set_(view.untyped_storage())
    mask = torch.ones(base.numel(), dtype=torch.bool, device=view.device)
    mask.as_strided(view.shape, view.stride(), view.storage_offset()).fill_(False)
    return base, mask


@pytest.mark.parametrize("fmt,nsplit", [("bf16", 3), ("fp16", 2)])
def test_strided_out_and_residual_views(ops, fmt, nsplit):
    """out= and residual= as column views of wider tensors with odd row strides (ldo 101, ldr 77: the per-element
    epilogue), clip stride != rows * ld: the result lands in the view only, every other element is untouched."""
    ops.set_plane_format(fmt)
    for batch, rows, taps, pad in ((3, 40, 3, 1), (2, 150, 1, 0)):
        cout = 70
        x = _rand(batch, rows, 128, seed=21)
        pw = ops.PackedW(_rand(taps, cout, 128, seed=22, scale=0.05), nsplit)
        bias = _rand(cout, seed=23, scale=0.1)
        big_out = _rand(batch, rows + 5, 101, seed=24)
        big_res = _rand(batch, rows + 2, 77, seed=25)
        out, res = big_out[:, 2:2 + rows, 13:13 + cout], big_res[:, 1:1 + rows, 3:3 + cout]
        base, mask = _outside(out)
        keep = base[mask].clone()
        res_before = big_res.clone()
        a = ops.split_bf16(x, nsplit)
        kw = dict(rows_out=rows, pad=pad, act=ops.ACT_RELU, residual=res)
        got, pl = ops.tapgemm_tc(a, pw, bias, out=out, out_nsplit=nsplit, out_slack=8, **kw)
        assert got.data_ptr() == out.data_ptr()
        assert torch.equal(base[mask], keep), "epilogue wrote outside the out= view"
        assert torch.equal(big_res, res_before)
        assert int(torch.count_nonzero(slack_rows(pl))) == 0
        _check(a, pw, bias, out, pl, tag=f"strided out/residual {(batch, rows, taps)} {fmt}", **kw)


@pytest.mark.parametrize("fmt,nsplit", [("bf16", 1), ("bf16", 2), ("bf16", 3), ("fp16", 2)])
def test_plane_only_output_with_slack(ops, fmt, nsplit):
    """want_f32=False: the planes are the only result (checked against float64 directly), with out_nsplit below the
    operand split and out_slack zeroed rows after the last clip."""
    ops.set_plane_format(fmt)
    for batch, rows, taps, pad, out_ns in ((5, 33, 3, 1, nsplit), (2, 300, 15, 7, max(1, nsplit - 1))):
        x = _rand(batch, rows, 64, seed=26)
        pw = ops.PackedW(_rand(taps, 64, 64, seed=27, scale=1 / math.sqrt(64 * taps)), nsplit)
        bias, res = _rand(64, seed=28, scale=0.1), _rand(batch, rows, 64, seed=29)
        a = ops.split_bf16(x, nsplit)
        kw = dict(rows_out=rows, pad=pad, act=ops.ACT_LEAKY, slope=0.01, residual=res)
        f, pl = ops.tapgemm_tc(a, pw, bias, want_f32=False, out_nsplit=out_ns, out_slack=8, **kw)
        assert f is None and pl.nsplit == out_ns and pl.slack == 8
        assert int(torch.count_nonzero(slack_rows(pl))) == 0
        _check(a, pw, bias, None, pl, tag=f"planes only {(batch, rows, taps)} out_nsplit={out_ns} {fmt}", **kw)

"""Tensor-core tap-GEMM (pm_tapgemm_tc) against a float64 restatement, for every split mode and the shapes the
EMAGE schedule issues: tall Linears, k=3 / k=15 convs with zero padding, clips packed 2..8 per 128-row tile,
ragged channel counts, fused bias / residual / partial activation, bf16 plane outputs."""
import math

import pytest
import torch
import torch.nn.functional as F


pytestmark = pytest.mark.gpu

# relative-to-row-scale tolerances per split mode: bf16 (8-bit mantissa), bf16x3 (~2^-16), bf16x6 (~fp32)
TOL = {1: 2e-2, 2: 2e-4, 3: 5e-6}


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


def _check(got, want, nsplit, scale):
    err = (got.double() - want).abs().max().item()
    assert err <= TOL[nsplit] * scale, f"nsplit={nsplit}: max err {err:.3e} > {TOL[nsplit] * scale:.3e}"


CASES = [
    # batch, rows, cin, cout, taps, pad
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
]


def _run_case(ops, case, nsplit, tol, plane_bits=8):
    batch, rows, cin, cout, taps, pad = case
    x = _rand(batch, rows, cin, seed=1)
    w = _rand(taps, cout, cin, seed=2, scale=1 / math.sqrt(cin * taps))
    bias = _rand(cout, seed=3, scale=0.1)
    rows_out = rows + 2 * pad - taps + 1
    res = _rand(batch, rows_out, cout, seed=4)
    want = F.conv1d(x.double().transpose(1, 2), w.double().permute(1, 2, 0), bias.double(), padding=pad).transpose(1, 2)
    want = F.leaky_relu(want + res.double(), 0.2)
    a = ops.split_bf16(x, nsplit)
    pw = ops.PackedW(w, nsplit)
    got, planes = ops.tapgemm_tc(a, pw, bias, rows_out=rows_out, pad=pad, act=ops.ACT_LEAKY, slope=0.2, residual=res,
                                 out_nsplit=nsplit)
    scale = float(want.abs().max())
    err = (got.double() - want).abs().max().item()
    assert err <= tol * scale, f"nsplit={nsplit}: max err {err:.3e} > {tol * scale:.3e}"
    rebuilt = planes.t[:, :, :, :cout].float().sum(0)          # the emitted planes re-assemble the fp32 result
    if planes.t.dtype == torch.float16:
        rebuilt = rebuilt / ops.F16_ACT_SCALE                  # fp16 planes hold 64 * x (exact)
    assert (rebuilt - got).abs().max().item() <= max(2.0 ** (-plane_bits * nsplit), 2.0 ** -24) * scale * 1.01


@pytest.mark.parametrize("nsplit", [1, 2, 3])
@pytest.mark.parametrize("case", CASES)
def test_tapgemm_tc_matches_fp64(ops, case, nsplit):
    _run_case(ops, case, nsplit, TOL[nsplit])


@pytest.mark.parametrize("case", CASES)
def test_tapgemm_tc_fp16_planes(ops, case):
    """Two IEEE fp16 planes, 3 products: the accuracy class of bf16x6 (weights packed pre-scaled by a power of two,
    undone by acc_scale in the epilogue)."""
    ops.set_plane_format("fp16")
    try:
        _run_case(ops, case, 2, TOL[3], plane_bits=11)
    finally:
        ops.set_plane_format("bf16")


def test_partial_activation_and_column_slices(ops):
    """conv1 | downsample fused along N: activation on the first half only; consumers read column slices."""
    x = _rand(3, 200, 128, seed=5)
    w = _rand(1, 128, 128, seed=6, scale=0.1)
    pw = ops.PackedW(w, 3)
    got, _ = ops.tapgemm_tc(ops.split_bf16(x, 3), pw, None, rows_out=200, act=ops.ACT_RELU, act_cols=64)
    want = F.linear(x.double(), w[0].double())
    want[:, :, :64] = F.relu(want[:, :, :64])
    _check(got, want, 3, float(want.abs().max()))
    # a column slice of a wider fp32 tensor as the A operand
    a = ops.split_bf16(got[:, :, 64:], 3)
    w2 = _rand(1, 64, 64, seed=7, scale=0.1)
    got2, _ = ops.tapgemm_tc(a, ops.PackedW(w2, 3), None, rows_out=200)
    _check(got2, F.linear(got[:, :, 64:].double(), w2[0].double()), 3, float(got2.abs().max()))


@pytest.mark.parametrize("C,cout", [(64, 64), (32, 64)])
def test_strided_conv_as_reshaped_stride1(ops, C, cout):
    """k=15 stride-6 conv == 3-tap stride-1 conv over the (L/6, 6*C) view with zero-padded taps."""
    b, L, s = 3, 745, 6
    x = _rand(b, L, C, seed=8)
    w = _rand(cout, C, 15, seed=9, scale=1 / math.sqrt(C * 15))
    want = F.conv1d(x.double().transpose(1, 2), w.double(), stride=s).transpose(1, 2)
    taps = -(-15 // s)
    wp = torch.zeros(taps, cout, s * C, device="cuda")
    for k in range(15):
        wp[k // s, :, (k % s) * C:(k % s + 1) * C] = w[:, :, k]
    a = ops.split_bf16(x, 3, slack_rows=s)
    rows_v = -(-L // s)
    got, _ = ops.tapgemm_tc(a, ops.PackedW(wp, 3), None, rows_out=want.shape[1], a_view=(rows_v, s * C, s * C))
    _check(got, want, 3, float(want.abs().max()))


@pytest.mark.parametrize("scale,tol", [(1.0, 5e-6), (0.05, 5e-6), (1e-3, 3e-4)])
def test_fp16_planes_small_activations(ops, scale, tol):
    """Tensor cores may flush fp16 SUBNORMAL operands, so the second plane of an element would be lost once it drops
    below 2^-14.  Activation planes are therefore pre-scaled by 64 (exact): LayerNorm-sized
    and 20x smaller activations keep the fp32-class accuracy; only tensors that are tiny as a whole (1e-3) degrade to
    single-plane fp16 accuracy (2^-11) - no tensor of this model is that small (smallest GEMM input: ~0.05)."""
    ops.set_plane_format("fp16")
    try:
        x = _rand(1, 256, 768, seed=11, scale=scale)
        w = _rand(1, 256, 768, seed=12, scale=1 / math.sqrt(768))
        want = F.linear(x.double(), w[0].double())
        got, _ = ops.tapgemm_tc(ops.split_bf16(x, 2), ops.PackedW(w, 2), None, rows_out=256)
        err = (got.double() - want).abs().max().item()
        assert err <= tol * float(want.abs().max()), err
    finally:
        ops.set_plane_format("bf16")

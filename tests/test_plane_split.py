"""The CPU restatement of the split-plane rule (tests/plane_split.py) against torch's own conversions, ops.PackedW's
weight planes and the per-element bound the GEMM tests use (helpers.plane_bound).  No GPU needed."""
import numpy as np
import pytest
import torch

import plane_split as ps
from helpers import F16_MIN_NORMAL, plane_bound

pytestmark = pytest.mark.filterwarnings("ignore::RuntimeWarning")      # the sweeps overflow and carry NaNs on purpose

DTYPE = {ps.BF16: torch.bfloat16, ps.FP16: torch.float16}


def _sweep():
    """Every fp32 exponent (subnormals and the inf / NaN exponent included) with the low-bit patterns where rounding
    to 8 / 11 significant bits turns (0x0FFF, 0x1000 = fp16 head tie, 0x1001, 0x1FFF, 0x8000 = bf16 tie) over even and
    odd kept bits, both signs."""
    e = np.arange(256, dtype=np.uint32)[:, None, None]
    low = np.array([0x0FFF, 0x1000, 0x1001, 0x1FFF, 0x8000, 0x8001, 0x7FFF, 0x0000], dtype=np.uint32)[None, :, None]
    kept = np.array([0x000000, 0x002000, 0x010000, 0x7FE000, 0x7F0000, 0x555000], dtype=np.uint32)[None, None, :]
    b = ((e << np.uint32(23)) | kept | low).reshape(-1)
    b = np.concatenate([b, b | np.uint32(0x80000000)])
    return b.view(np.float32)


@pytest.mark.parametrize("fmt", [ps.BF16, ps.FP16])
def test_one_plane_is_torch_round_to_nearest_even(fmt):
    x = np.concatenate([_sweep(), ps.edge_values()])
    want = torch.from_numpy(x).to(DTYPE[fmt]).view(torch.int16).numpy().view(np.uint16)
    got = ps.split(x, 1, fmt, act=False)[0]
    nan = np.isnan(x)
    assert np.array_equal(got[~nan], want[~nan])
    assert np.isnan(ps.bits_to_f32(got[nan], fmt)).all()
    if fmt == ps.FP16:                        # activation planes: the same conversion of 64 x
        want = torch.from_numpy(x * np.float32(64)).to(torch.float16).view(torch.int16).numpy().view(np.uint16)
        assert np.array_equal(ps.split(x, 1, fmt)[0][~nan], want[~nan])


@pytest.mark.parametrize("fmt", [ps.BF16, ps.FP16])
@pytest.mark.parametrize("nsplit", [1, 2, 3])
def test_matches_packed_weight_planes(fmt, nsplit):
    from pantomatrix_b200 import ops
    old = ops.plane_format()
    ops.set_plane_format(fmt)
    try:
        g = torch.Generator().manual_seed(3)
        w = torch.randn(3, 70, 45, generator=g) * torch.logspace(-6, 2, 45)       # columns over eight decades
        w[0, 0, :8] = torch.from_numpy(ps.edge_values()[:8])
        pw = ops.PackedW(w, nsplit)
    finally:
        ops.set_plane_format(old)
    full = torch.zeros(3, pw.w_rows, pw.ldw)
    full[:, :70, :45] = w
    scale = 1.0 / (pw.acc_scale * ps.F16_ACT_SCALE) if fmt == ps.FP16 else 1.0     # the exact power of two it applied
    want = ps.split((full * scale).numpy(), nsplit, fmt, act=False)
    assert np.array_equal(pw.t.view(torch.int16).numpy().view(np.uint16), want)


@pytest.mark.parametrize("fmt", [ps.BF16, ps.FP16])
@pytest.mark.parametrize("nsplit", [1, 2, 3])
def test_split_meets_plane_bound(fmt, nsplit):
    """Wherever the planes are finite, their sum is within helpers.plane_bound of x (bf16: where every plane is a
    normal number, the range the engine's activations live in)."""
    x = np.concatenate([_sweep(), ps.edge_values()])
    bits = ps.split(x, nsplit, fmt)
    vals = ps.bits_to_f32(bits, fmt)
    ok = np.isfinite(x) & np.isfinite(vals).all(0)
    if fmt == ps.BF16:
        ok &= (np.abs(x) >= 2.0 ** -100) | (x == 0)
    err = np.abs(ps.plane_sum(bits, fmt) - x.astype(np.float64))
    bound = plane_bound(nsplit, DTYPE[fmt], torch.from_numpy(x.astype(np.float64))).numpy()
    assert ok.sum() > 10000
    bad = ok & ~(err <= bound)
    assert not bad.any(), f"{bad.sum()} elements outside the bound, e.g. x = {x[bad][:4]}"


def test_fp16_head_is_exact_in_the_normal_range():
    """The two-plane fp16 head (half away from zero on the bit pattern) is an fp16 number wherever |64 x| >= 2^-14 and
    it does not overflow, so plane 1 is the exact remainder there; ties go away from zero, not to even."""
    v = np.concatenate([_sweep(), ps.edge_values()]) * np.float32(64)
    v = v[np.isfinite(v)]
    head = ps.f16_head(v)
    normal = (np.abs(v) >= F16_MIN_NORMAL) & (np.abs(head) <= 65504)
    assert normal.sum() > 1000
    back = ps.bits_to_f32(ps.rne_fp16(head[normal]), ps.FP16)
    assert np.array_equal(back, head[normal])
    tie = np.float32(1.0 + 2.0 ** -11)               # halfway between 1 and 1 + 2^-10 (even neighbour: 1)
    assert ps.f16_head(np.array([tie, -tie]))[0] == np.float32(1.0 + 2.0 ** -10)
    assert ps.f16_head(np.array([-tie]))[0] == -np.float32(1.0 + 2.0 ** -10)
    assert ps.bits_to_f32(ps.rne_fp16(np.array([tie])), ps.FP16)[0] == 1.0


def test_non_finite_inputs_by_class():
    x = np.array([np.nan, np.inf, -np.inf], dtype=np.float32)
    x = np.concatenate([x, np.uint32([0x7FFFFFFF, 0xFFFFFFFF]).view(np.float32)])
    for fmt in (ps.BF16, ps.FP16):
        for nsplit in (1, 2, 3):
            s = ps.plane_sum(ps.split(x, nsplit, fmt), fmt)
            assert np.isnan(s[[0, 3, 4]]).all() and not np.isfinite(s[1:3]).any(), (fmt, nsplit, s)
    # the two-plane fp16 head of the canonical NaN wraps to a zero: plane 1 alone carries the NaN
    canon = np.uint32([0x7FFFFFFF]).view(np.float32)
    assert ps.f16_head(canon)[0] == 0.0
    planes = ps.split(canon, 2, ps.FP16)
    assert ps.bits_to_f32(planes[0], ps.FP16)[0] == 0.0 and np.isnan(ps.bits_to_f32(planes[1], ps.FP16)[0])


def test_mismatches_flags_a_wrong_plane():
    """The comparison the GPU tests use: a one-ulp change of any plane, a lost NaN or a finite sum at an inf is seen."""
    x = ps.edge_values()
    for fmt in (ps.BF16, ps.FP16):
        for nsplit in (1, 2, 3):
            good = ps.split(x, nsplit, fmt)
            assert not ps.mismatches(good, x, fmt).any()
            bad = good.copy()
            bad[nsplit - 1, 5] ^= np.uint16(1)
            assert ps.mismatches(bad, x, fmt)[5]
            i = int(np.flatnonzero(np.isnan(x))[0])
            bad = good.copy()
            bad[:, i] = 0
            assert ps.mismatches(bad, x, fmt)[i]
    one = ps.split(x, 1, ps.FP16)
    head = ps.rne_fp16(ps.f16_head(x * np.float32(64)))[None]
    assert ps.mismatches(head, x, ps.FP16).sum() > 10         # half-away ties and a lost NaN differ from the rule
    assert not ps.mismatches(one, x, ps.FP16).any()

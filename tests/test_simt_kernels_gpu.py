"""The CUDA-core (SIMT) fp32 kernels swept over the shapes where they can go wrong, every output element against its
own float64 bound (tests/simt_bounds.py): the persistent BiLSTM (teacher-forced, per step), fp32 attention, the fp32
tap-GEMM, the residual LayerNorm and the WavEncoder stem.  Each sweep prints the largest fraction of the bound used."""
import math
import time

import pytest
import torch

import simt_bounds as sb

pytestmark = pytest.mark.gpu
DEV = "cuda"
H = 512


@pytest.fixture(scope="module")
def ops():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    from pantomatrix_b200 import _lib, ops as o
    assert _lib.load().pm_device_cc() == 90, "sm_90a kernels need a Hopper (H100) device"
    return o


def _rand(*shape, seed, scale=1.0):
    return (torch.randn(*shape, generator=torch.Generator().manual_seed(seed)) * scale).to(DEV)


class Used:
    """Largest fraction of the per-element bound used over a sweep; each check asserts its own elements."""

    def __init__(self, name):
        self.name, self.worst, self.where = name, 0.0, None

    def check(self, got, want, bound, tag):
        f = sb.bound_fraction(got, want, bound)
        assert f <= 1.0, f"{self.name} {tag}: uses {f:.3g} of its per-element bound"
        if f >= self.worst:
            self.worst, self.where = f, tag

    def report(self, extra=""):
        print(f"[{self.name}] largest fraction of the per-element bound used: {self.worst:.3g} ({self.where}){extra}")


def _sentinel(*shape):
    """A float32 tensor of a bit pattern no kernel writes (a NaN payload), to check that nothing outside a view changes."""
    return torch.full(shape, -1, dtype=torch.int32, device=DEV).view(torch.float32)


# ------------------------------------------------------------------------------------------------------------------
# BiLSTM
# ------------------------------------------------------------------------------------------------------------------


def _lstm_operands(batch, t, x_scale, seed):
    xproj = _rand(batch, t, 8 * H, seed=seed, scale=x_scale)
    whh = _rand(2, 4 * H, H, seed=seed + 1, scale=1.2 / math.sqrt(H))   # the synthetic checkpoints' scale
    return xproj, whh


@pytest.mark.parametrize("batch", [1, 31, 32, 33, 40, 63, 64, 65, 129])
def test_lstm_bidir_per_step(ops, batch):
    """One or two 32-row halves, partial halves, and 1 to 3 launches of 64 clips with partial tails; t = 1 (no
    recurrent product), 2, 9, 149; production-scale inputs and a saturated case (xproj x8: gates at 0 or 1, c grows
    over 149 steps).  One barrier tensor serves every call."""
    used = Used(f"lstm_bidir batch {batch}")
    barrier = torch.zeros(4, dtype=torch.int32, device=DEV)
    t_ref = 0.0
    for t in (1, 2, 9, 149):
        for x_scale in (1.0, 8.0):
            xproj, whh = _lstm_operands(batch, t, x_scale, seed=batch * 10 + t)
            y = ops.lstm_bidir(xproj, whh, barrier, H)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            want, bound = sb.lstm_bidir_f32(xproj, whh, y)
            torch.cuda.synchronize()
            t_ref += time.perf_counter() - t0
            used.check(y, want, bound, f"t {t} x{x_scale:g}")
    used.report(f"; float64 reference {t_ref:.2f} s")


def test_lstm_bidir_strided_views_write_nothing_else(ops):
    """Through the C entry point: xproj rows wider than 8H (ldx > 8H) and y a column range of a wider tensor
    (ldy > 2H, as the BiLSTM halves written in place): the view matches the dense call bit for bit, and not one byte
    outside it changes."""
    from pantomatrix_b200 import _lib
    batch, t = 40, 9
    xproj, whh = _lstm_operands(batch, t, 1.0, seed=5)
    barrier = torch.zeros(4, dtype=torch.int32, device=DEV)
    dense = ops.lstm_bidir(xproj, whh, barrier, H)
    xw = _rand(batch, t, 8 * H + 36, seed=6)
    xw[:, :, 20:20 + 8 * H] = xproj
    x_v = xw[:, :, 20:20 + 8 * H]
    yw = _sentinel(batch, t, 2 * H + 200)
    before = yw.clone()
    y_v = yw[:, :, 96:96 + 2 * H]
    _lib.call("pm_lstm_bidir_f32", x_v.data_ptr(), x_v.stride(0), x_v.stride(1), whh.data_ptr(), y_v.data_ptr(),
              y_v.stride(0), y_v.stride(1), barrier.data_ptr(), batch, t, H, torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    assert torch.equal(y_v.view(torch.int32), dense.view(torch.int32))
    outside = torch.ones_like(yw, dtype=torch.bool)
    outside[:, :, 96:96 + 2 * H] = False
    assert torch.equal(yw.view(torch.int32)[outside], before.view(torch.int32)[outside])
    want, bound = sb.lstm_bidir_f32(x_v, whh, y_v)
    assert sb.within(y_v, want, bound)


def test_lstm_bidir_clip_alone_is_bit_identical(ops):
    """A clip computed alone gives the same bits as its row in a batch of 129 (3 launches): every row's 8 K-slices are
    combined by the same xor-4/2/1 shuffle tree whatever its position in the CTA, half or launch."""
    batch, t = 129, 30
    xproj, whh = _lstm_operands(batch, t, 1.0, seed=7)
    barrier = torch.zeros(4, dtype=torch.int32, device=DEV)
    full = ops.lstm_bidir(xproj, whh, barrier, H)
    for b in range(batch):
        alone = ops.lstm_bidir(xproj[b:b + 1].contiguous(), whh, barrier, H)
        assert torch.equal(alone.view(torch.int32), full[b:b + 1].view(torch.int32)), b


# ------------------------------------------------------------------------------------------------------------------
# attention
# ------------------------------------------------------------------------------------------------------------------

T_EDGES = (1, 2, 31, 32, 33, 63, 64)


def test_attention_f32_sweep(ops):
    """Every (tq, tk) in {1, 2, 31, 32, 33, 63, 64}^2 with 1 and 4 heads; q, k, v read as column ranges of wider packed
    q|k|v and k|v tensors, as the engine passes them."""
    used = Used("attention_f32")
    bs, hd = 3, 192
    for heads in (1, 4):
        E = heads * hd
        q0, k0 = 8, 20                                      # first column of Q inside q|k|v, of K inside k|v
        for tq in T_EDGES:
            for tk in T_EDGES:
                qkv = _rand(bs * tq, q0 + 3 * E + 12, seed=tq * 100 + tk)
                kv = _rand(bs * tk, k0 + 2 * E + 4, seed=tq * 100 + tk + 7)
                q, k, v = qkv[:, q0:q0 + E], kv[:, k0:k0 + E], kv[:, k0 + E:k0 + 2 * E]
                got = ops.attention(q, k, v, bs, heads, tq, tk, hd)
                used.check(got, *sb.attention_f32(q, k, v, bs, heads, tq, tk, hd), f"heads {heads} {tq}x{tk}")
    used.report()


def test_attention_f32_peaked_rows_and_independence(ops):
    """Peaked rows (scores ~ N(0, 10^2), the scale-3.2 case of the tensor-core test), and each clip alone and each
    head alone bit-identical to the batched call."""
    used = Used("attention_f32 peaked")
    E, heads, hd, bs, t = 768, 4, 192, 6, 64
    qkv = _rand(bs * t, 3 * E, seed=75, scale=3.2)
    q, k, v = qkv[:, :E], qkv[:, E:2 * E], qkv[:, 2 * E:]
    got = ops.attention(q, k, v, bs, heads, t, t, hd)
    used.check(got, *sb.attention_f32(q, k, v, bs, heads, t, t, hd), "peaked")
    for b in range(bs):
        rows = slice(b * t, (b + 1) * t)
        alone = ops.attention(q[rows], k[rows], v[rows], 1, heads, t, t, hd)
        assert torch.equal(alone.view(torch.int32), got[rows].view(torch.int32)), b
    for h in range(heads):
        cols = slice(h * hd, (h + 1) * hd)
        alone = ops.attention(q[:, cols], k[:, cols], v[:, cols], bs, 1, t, t, hd)
        assert torch.equal(alone.view(torch.int32), got[:, cols].view(torch.int32)), h
    used.report()


# ------------------------------------------------------------------------------------------------------------------
# tap-GEMM
# ------------------------------------------------------------------------------------------------------------------

GEOMETRIES = [(15, 1, 7), (15, 6, 0), (3, 1, 1), (1, 1, 0)]             # taps, stride, pad


def _tap_operands(batch, rows_in, cin, cout, taps, seed):
    a = _rand(batch, rows_in, cin, seed=seed)
    decades = 10.0 ** torch.linspace(-3, 3, cout, device=DEV)[:, None]  # output columns over six decades
    w = _rand(taps, cout, cin, seed=seed + 1, scale=1 / math.sqrt(taps * cin)) * decades
    return a, w.contiguous(), _rand(cout, seed=seed + 2, scale=0.1) * decades[:, 0]


@pytest.mark.parametrize("taps,stride,pad", GEOMETRIES)
def test_tapgemm_f32_sweep(ops, taps, stride, pad):
    """rows_out in {1, 127, 128, 129} (one, a partial and two 128-row tiles), cout in {1, 63, 64, 65} (64-column
    tiles), cin in {1, 15, 16, 17, 337} (partial 16-channel K tiles), and a rows_out below the natural one; bias,
    residual and activation varied across the cases."""
    used = Used(f"tapgemm_f32 taps {taps} stride {stride} pad {pad}")
    n = 0
    for rows_out in (1, 127, 128, 129):
        for cout in (1, 63, 64, 65):
            for cin in (1, 15, 16, 17, 337):
                n += 1
                rows_in = (rows_out - 1) * stride + taps - 2 * pad + (5 if n % 5 == 0 else 0)  # % 5: rows_out short
                batch = 2
                a, w, bias = _tap_operands(batch, rows_in, cin, cout, taps, seed=n)
                act = (ops.ACT_NONE, ops.ACT_LEAKY, ops.ACT_RELU)[n % 3]
                res = _rand(batch, rows_out, cout, seed=n + 9) if n % 2 else None
                b = bias if n % 4 != 3 else None
                kw = dict(stride=stride, pad=pad, rows_out=rows_out, act=act, slope=0.2, residual=res)
                got = ops.tapgemm(a, w, b, **kw)
                used.check(got, *sb.tapgemm_f32(a, w, b, **kw), f"rows_out {rows_out} cout {cout} cin {cin}")
    used.report()


def test_tapgemm_f32_views_write_nothing_else(ops):
    """out= and residual= column views of wider tensors, A a column range with a clip gap: every element within its
    bound, nothing outside the out view written."""
    batch, rows_in, cin, cout = 3, 129, 17, 65
    for taps, stride, pad in GEOMETRIES:
        a_w = _rand(batch, rows_in + 3, cin + 11, seed=40)
        a = a_w[:, :rows_in, 5:5 + cin]
        _, w, bias = _tap_operands(1, 1, cin, cout, taps, seed=41)
        rows_out = (rows_in + 2 * pad - taps) // stride + 1
        r_w = _rand(batch, rows_out, cout + 30, seed=42)
        res = r_w[:, :, 7:7 + cout]
        o_w = _sentinel(batch, rows_out, cout + 30)
        before = o_w.clone()
        out = o_w[:, :, 9:9 + cout]
        kw = dict(stride=stride, pad=pad, act=ops.ACT_LEAKY, slope=0.2, residual=res)
        ops.tapgemm(a, w, bias, out=out, **kw)
        assert sb.within(out, *sb.tapgemm_f32(a, w, bias, rows_out=rows_out, **kw))
        outside = torch.ones_like(o_w, dtype=torch.bool)
        outside[:, :, 9:9 + cout] = False
        assert torch.equal(o_w.view(torch.int32)[outside], before.view(torch.int32)[outside]), (taps, stride, pad)


def test_tapgemm_f32_flat_linear_path_is_per_clip_order(ops):
    """ops.tapgemm runs a Linear over contiguous clips as one tall matrix; a clip gap in A forces the per-clip grid.
    Both run the same fma chain per output, so they agree bit for bit (and with each clip alone)."""
    batch, rows, cin, cout = 5, 77, 337, 65
    a_gap = _rand(batch, rows + 2, cin, seed=50)
    a_dense = a_gap[:, :rows].contiguous()
    _, w, bias = _tap_operands(1, 1, cin, cout, 1, seed=51)
    res = _rand(batch, rows, cout, seed=52)
    kw = dict(act=ops.ACT_LEAKY, slope=0.1, residual=res)
    flat = ops.tapgemm(a_dense, w, bias, **kw)
    per_clip = ops.tapgemm(a_gap[:, :rows], w, bias, **kw)
    assert torch.equal(flat.view(torch.int32), per_clip.view(torch.int32))
    for b in (0, 2, 4):
        alone = ops.tapgemm(a_dense[b:b + 1], w, bias, act=ops.ACT_LEAKY, slope=0.1, residual=res[b:b + 1])
        assert torch.equal(alone.view(torch.int32), flat[b:b + 1].view(torch.int32)), b
    assert sb.within(flat, *sb.tapgemm_f32(a_dense, w, bias, **kw))


def test_tapgemm_f32_linear_with_fewer_output_rows(ops):
    """A Linear over contiguous clips asked for fewer output rows than input rows: clip b's outputs come from clip b's
    first rows, so this call must not take the tall-matrix path, which would read them from row b * rows_out of the
    flattened input."""
    batch, rows_in, rows_out, cin, cout = 3, 40, 33, 17, 65
    a, w, bias = _tap_operands(batch, rows_in, cin, cout, 1, seed=53)
    got = ops.tapgemm(a, w, bias, rows_out=rows_out)
    assert sb.within(got, *sb.tapgemm_f32(a, w, bias, rows_out=rows_out))
    for b in range(batch):
        alone = ops.tapgemm(a[b:b + 1], w, bias, rows_out=rows_out)
        assert torch.equal(alone.view(torch.int32), got[b:b + 1].view(torch.int32)), b


# ------------------------------------------------------------------------------------------------------------------
# LayerNorm
# ------------------------------------------------------------------------------------------------------------------


def _ln_rows(kind, rows, ch, seed):
    if kind == "normal":
        return _rand(rows, ch, seed=seed, scale=3.0), _rand(rows, ch, seed=seed + 1)
    if kind == "offset":                                                # mean 1e3, std 1e-2
        return 1e3 + _rand(rows, ch, seed=seed, scale=1e-2), _rand(rows, ch, seed=seed + 1, scale=1e-2)
    c = _rand(rows, 1, seed=seed, scale=300.0) + 0.1234567              # constant rows: var 0
    return c.expand(rows, ch).contiguous(), _rand(rows, 1, seed=seed + 1).expand(rows, ch).contiguous()


@pytest.mark.parametrize("ch", [256, 512, 768, 1024])
def test_add_layernorm_sweep(ops, ch):
    """rows in {1, 7, 8, 9, 301} (one warp per row, 8 rows per CTA), normal, offset and constant rows, with and
    without the residual r."""
    used = Used(f"add_layernorm ch {ch}")
    g, b = _rand(ch, seed=60), _rand(ch, seed=61)
    for rows in (1, 7, 8, 9, 301):
        for kind in ("normal", "offset", "constant"):
            x, r = _ln_rows(kind, rows, ch, seed=rows + ch)
            for rr in (r, None):
                got = ops.add_layernorm(x, rr, g, b)
                used.check(got, *sb.add_layernorm_f32(x, rr, g, b), f"rows {rows} {kind} r={rr is not None}")
    used.report()


# ------------------------------------------------------------------------------------------------------------------
# WavEncoder stem
# ------------------------------------------------------------------------------------------------------------------


@pytest.mark.parametrize("cout,stride,pad", [(64, 5, 1600), (32, 5, 1600), (32, 4, 3), (64, 3, 7)])
def test_wav_stem_sweep(ops, cout, stride, pad):
    """rows_out = 1, 190 and 191 (mod 192): a lone row, and tiles whose three-row groups end inside the tile; the
    stride-5 fast path and the generic path; each window's span (offset, padding) reaching past its n_samples into
    audio that exists but must read as zero."""
    used = Used(f"wav_stem cout {cout} stride {stride} pad {pad}")
    bs, windows, offset = 3, 2, 37
    w1, wd = _rand(cout, 15, seed=70, scale=0.5), _rand(cout, 15, seed=71, scale=0.5)
    b1, bd = _rand(cout, seed=72, scale=0.1), _rand(cout, seed=73, scale=0.1)
    for k, m in ((0, 1), (6, 1), (5, 190), (6, 191), (0, 190)):
        rows_out = 192 * k + m
        n = (rows_out - 1) * stride + 15 - 2 * pad + (stride - 1)
        if n <= 0:
            continue
        a_ws = n // 2 + 3
        audio = _rand(bs, offset + a_ws * (windows - 1) + n + 401, seed=rows_out, scale=0.1)
        args = (audio, audio.shape[1], a_ws, bs, windows, n, w1, b1, wd, bd)
        kw = dict(stride=stride, pad=pad, slope=0.01, offset=offset)
        y1, sc = ops.wav_stem(*args, **kw)
        assert y1.shape[1] == rows_out
        (wy, by), (ws, bs_) = sb.wav_stem_f32(*args, **kw)
        used.check(y1, wy, by, f"rows_out {rows_out} y1")
        used.check(sc, ws, bs_, f"rows_out {rows_out} sc")
    used.report()

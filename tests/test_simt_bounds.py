"""The per-element checks of tests/simt_bounds.py can fail: each is fed a CPU fp32 restatement of its kernel (in the
kernel's reduction order where that order matters), which it must accept, and small copies of plausible kernel bugs
applied to that restatement, each of which it must reject.  No GPU needed."""
import math

import pytest
import torch

import simt_bounds as sb

H = 512


def _rand(*shape, seed, scale=1.0):
    return torch.randn(*shape, generator=torch.Generator().manual_seed(seed)) * scale


# ------------------------------------------------------------------------------------------------------------------
# tap-GEMM
# ------------------------------------------------------------------------------------------------------------------


def _tapgemm32(a, w, bias, *, stride, pad, rows_out, act, slope, residual, drop_cin_tail=False, read_past_end=False):
    """fp32 restatement of tapgemm_f32_kernel: the (tap, channel) products summed by one fp32 matmul per output, then
    + bias, + residual and the activation in fp32.  drop_cin_tail: the last, partial 16-channel K tile is skipped.
    read_past_end: row `rows_in` is taken as data (the next clip's first row) instead of padding."""
    batch, rows_in, cin = a.shape
    taps, cout, _ = w.shape
    if drop_cin_tail:
        a = a.clone()
        a[..., cin - cin % 16:] = 0
    ext = torch.cat([a, a.roll(-1, 0)[:, :1]], 1) if read_past_end else a
    hi = rows_in + 1 if read_past_end else rows_in
    l = torch.arange(rows_out)[:, None] * stride + torch.arange(taps)[None] - pad
    ok = (l >= 0) & (l < hi)
    g = (ext[:, l.clamp(0, hi - 1)] * ok[None, :, :, None]).reshape(batch, rows_out, taps * cin)
    v = g @ w.permute(0, 2, 1).reshape(taps * cin, cout)
    if bias is not None:
        v = v + bias
    if residual is not None:
        v = v + residual
    if act == sb.ACT_LEAKY:
        v = torch.where(v > 0, v, v * slope)
    elif act == sb.ACT_RELU:
        v = torch.where(v > 0, v, torch.zeros_like(v))
    return v


TAP_CASES = [
    # batch, rows_out, cin, cout, taps, stride, pad, act, residual
    (2, 129, 17, 65, 15, 1, 7, sb.ACT_LEAKY, True),
    (3, 127, 337, 64, 3, 1, 1, sb.ACT_NONE, False),
    (2, 1, 15, 63, 15, 6, 0, sb.ACT_RELU, True),
    (2, 128, 33, 1, 3, 1, 1, sb.ACT_LEAKY, False),
]


@pytest.mark.parametrize("case", TAP_CASES)
def test_tapgemm_bound_accepts_fp32_and_rejects_bugs(case):
    batch, rows_out, cin, cout, taps, stride, pad, act, use_res = case
    rows_in = (rows_out - 1) * stride + taps - 2 * pad
    a = _rand(batch, rows_in, cin, seed=1)
    decades = 10.0 ** torch.linspace(-3, 3, cout)[:, None]          # output columns over six decades
    w = _rand(taps, cout, cin, seed=2, scale=1 / math.sqrt(taps * cin)) * decades
    bias = _rand(cout, seed=3, scale=0.1)
    res = _rand(batch, rows_out, cout, seed=4) if use_res else None
    kw = dict(stride=stride, pad=pad, rows_out=rows_out, act=act, slope=0.2, residual=res)
    want, bound = sb.tapgemm_f32(a, w, bias, **kw)
    assert sb.within(_tapgemm32(a, w, bias, **kw), want, bound)
    if cin % 16:
        assert not sb.within(_tapgemm32(a, w, bias, drop_cin_tail=True, **kw), want, bound)
    if pad:
        assert not sb.within(_tapgemm32(a, w, bias, read_past_end=True, **kw), want, bound)


# ------------------------------------------------------------------------------------------------------------------
# WavEncoder stem
# ------------------------------------------------------------------------------------------------------------------


def _stem32(audio, a_bs, a_ws, batch, windows, n, w1, b1, wd, bd, *, stride, pad, slope, offset, drop=None):
    """fp32 restatement of wav_stem_kernel; drop = output row that misses its last tap (in every sequence)."""
    flat = audio.reshape(-1)
    seqs = torch.stack([flat[offset + b * a_bs + w * a_ws:][:n] for w in range(windows) for b in range(batch)])
    ks = w1.shape[1]
    rows_out = (n + 2 * pad - ks) // stride + 1
    xp = torch.nn.functional.pad(seqs, (pad, pad + stride))
    win = xp.unfold(1, ks, stride)[:, :rows_out]                     # (seq, rows_out, ks)
    if drop is not None:
        win = win.clone()
        win[:, drop, ks - 1] = 0
    y1 = win @ w1.t() + b1
    return torch.where(y1 > 0, y1, y1 * slope), win @ wd.t() + bd


@pytest.mark.parametrize("cout,stride,pad", [(64, 5, 1600), (32, 4, 3)])
def test_wav_stem_bound_accepts_fp32_and_rejects_a_missing_tap(cout, stride, pad):
    bs, windows, a_ws, n, offset = 2, 2, 1300, 2900, 37
    audio = _rand(bs, offset + a_ws + n + 50, seed=7, scale=0.1)
    w1, wd = _rand(cout, 15, seed=8, scale=0.5), _rand(cout, 15, seed=9, scale=0.5)
    b1, bd = _rand(cout, seed=10, scale=0.1), _rand(cout, seed=11, scale=0.1)
    args = (audio, audio.shape[1], a_ws, bs, windows, n, w1, b1, wd, bd)
    kw = dict(stride=stride, pad=pad, slope=0.01, offset=offset)
    (wy, by), (ws, bs_) = sb.wav_stem_f32(*args, **kw)
    y1, sc = _stem32(*args, **kw)
    assert sb.within(y1, wy, by) and sb.within(sc, ws, bs_)
    row = 2 * 192 - 1                                                  # the last row of the second 192-row tile
    assert (row * stride + 14 - pad) in range(n)                       # its last tap reads a sample, not padding
    y1m, scm = _stem32(*args, drop=row, **kw)
    assert not sb.within(y1m, wy, by) and not sb.within(scm, ws, bs_)


# ------------------------------------------------------------------------------------------------------------------
# LayerNorm
# ------------------------------------------------------------------------------------------------------------------


def _layernorm32(x, r, g, b, eps=1e-5, one_pass=False):
    """fp32 restatement of add_layernorm_kernel in its order: per-lane sums over float4 chunks lane + 32 i, the
    5-level xor butterfly, two-pass variance.  one_pass: variance as E[v^2] - mean^2."""
    rows, n = x.shape
    vec = n // 128
    v = x + r if r is not None else x.clone()
    lanes = v.reshape(rows, vec, 32, 4)                               # chunk i of lane l: columns (l + 32 i) * 4 ..

    def warp_sum(fn):
        s = torch.zeros(rows, 32)
        for i in range(vec):
            q = fn(lanes[:, i])
            s = s + ((q[..., 0] + q[..., 1]) + (q[..., 2] + q[..., 3]))
        for o in (16, 8, 4, 2, 1):
            s = s + s[:, torch.arange(32) ^ o]
        return s[:, :1]

    inv = torch.tensor(1.0 / n, dtype=torch.float32)
    mean = warp_sum(lambda c: c) * inv
    if one_pass:
        var = warp_sum(lambda c: c * c) * inv - mean * mean
    else:
        var = warp_sum(lambda c: (c - mean[:, :, None]) ** 2) * inv
    rstd = torch.rsqrt(var + eps)
    return (v - mean) * rstd * g + b


@pytest.mark.parametrize("ch", [256, 768, 1024])
def test_layernorm_bound_accepts_fp32_and_rejects_one_pass_variance(ch):
    rows = 9
    g, b = _rand(ch, seed=12), _rand(ch, seed=13)
    x, r = _rand(rows, ch, seed=14, scale=3.0), _rand(rows, ch, seed=15)
    for rr in (r, None):
        want, bound = sb.add_layernorm_f32(x, rr, g, b)
        assert sb.within(_layernorm32(x, rr, g, b), want, bound)
    # offset rows: mean 1e3, std 1e-2 - a one-pass variance loses everything there
    xo = 1e3 + _rand(rows, ch, seed=16, scale=1e-2)
    ro = _rand(rows, ch, seed=17, scale=1e-2)
    for rr in (ro, None):
        want, bound = sb.add_layernorm_f32(xo, rr, g, b)
        assert sb.within(_layernorm32(xo, rr, g, b), want, bound)
        assert not sb.within(_layernorm32(xo, rr, g, b, one_pass=True), want, bound)
        assert float((bound / (want - b).abs().clamp_min(1e-3)).median()) < 0.25     # still says something
    # constant rows: var 0, rstd = eps^-1/2
    xc = (_rand(rows, 1, seed=18, scale=300.0) + 0.1234567).expand(rows, ch).contiguous()
    want, bound = sb.add_layernorm_f32(xc, None, g, b)
    assert sb.within(_layernorm32(xc, None, g, b), want, bound)


# ------------------------------------------------------------------------------------------------------------------
# attention
# ------------------------------------------------------------------------------------------------------------------


def _attention32(q, k, v, batch, heads, tq, tk, hd=192, drop_last=False, max_over=None):
    """fp32 restatement of attention_f32_kernel: fp32 scores times fl(1/sqrtf(192)), the row max, expf, the row sum
    (e0 + e1 then the butterfly), p = e * (1 / sum), O = P V.  drop_last: key tk - 1 left out of the row sum.
    max_over: the row max taken over the first max_over keys only."""
    E = heads * hd
    Q, K, V = (x[:, :E].reshape(batch, -1, heads, hd).transpose(1, 2) for x in (q, k, v))
    scale = torch.tensor(1.0, dtype=torch.float32) / torch.sqrt(torch.tensor(float(hd), dtype=torch.float32))
    s = (Q @ K.transpose(-1, -2)) * scale
    m = s[..., :max_over].amax(-1, keepdim=True) if max_over else s.amax(-1, keepdim=True)
    e = torch.exp(s - m)
    e64 = torch.zeros(*e.shape[:-1], 64)
    e64[..., :tk] = e
    if drop_last:
        e64[..., tk - 1] = 0
    lane = e64[..., :32] + e64[..., 32:]
    for o in (16, 8, 4, 2, 1):
        lane = lane + lane[..., torch.arange(32) ^ o]
    p = e * (1.0 / lane[..., :1])
    return (p @ V).transpose(1, 2).reshape(-1, E)


@pytest.mark.parametrize("tq,tk", [(33, 64), (64, 33), (1, 1), (31, 2)])
def test_attention_bound_accepts_fp32_and_rejects_softmax_bugs(tq, tk):
    batch, heads, E = 2, 2, 384
    q, k, v = _rand(batch * tq, E, seed=19), _rand(batch * tk, E, seed=20), _rand(batch * tk, E, seed=21)
    want, bound = sb.attention_f32(q, k, v, batch, heads, tq, tk)
    assert sb.within(_attention32(q, k, v, batch, heads, tq, tk), want, bound)
    assert not sb.within(_attention32(q, k, v, batch, heads, tq, tk, drop_last=True), want, bound)
    if tk > 32:
        # a key past the first 32 that dominates its row (scaled score ~ 200): the row max of 32 keys overflows expf
        k2 = k.clone().reshape(batch, tk, E)
        k2[:, tk - 1] = 15 * q.reshape(batch, tq, E)[:, 0]
        k2 = k2.reshape(batch * tk, E)
        want, bound = sb.attention_f32(q, k2, v, batch, heads, tq, tk)
        assert sb.within(_attention32(q, k2, v, batch, heads, tq, tk), want, bound)
        assert not sb.within(_attention32(q, k2, v, batch, heads, tq, tk, max_over=32), want, bound)


def test_attention_bound_peaked_rows():
    batch, heads, t, E = 2, 2, 64, 384
    qkv = _rand(batch * t, 3 * E, seed=22, scale=3.2)
    q, k, v = qkv[:, :E], qkv[:, E:2 * E], qkv[:, 2 * E:]
    want, bound = sb.attention_f32(q, k, v, batch, heads, t, t)
    assert sb.within(_attention32(q, k, v, batch, heads, t, t), want, bound)
    assert not sb.within(_attention32(q, k, v, batch, heads, t, t, drop_last=True), want, bound)


# ------------------------------------------------------------------------------------------------------------------
# BiLSTM
# ------------------------------------------------------------------------------------------------------------------

SLICE_COLS = [torch.tensor([4 * kq + 32 * j + c for j in range(H // 32) for c in range(4)]) for kq in range(8)]


def _lstm32(xproj, whh, drop=None, stale=None, swap_row=None):
    """fp32 restatement of lstm_bidir_kernel: per step the 8 K-slices of h_{t-1} . W_hh (columns 4 kq + 32 j + c) as
    fp32 matmuls, combined ((s0 + s4) + (s2 + s6)) + ((s1 + s5) + (s3 + s7)), + x, the gates in fp32.
    drop = (dir, step, unit, row, slice): that K-slice is missing from the unit's four gates at that step and row.
    stale = (dir, step, unit0): units unit0 .. unit0 + 15 of batch rows 0..31 read h_{t-2} instead of h_{t-1}.
    swap_row: forward and backward outputs of that batch row are exchanged."""
    B, T, _ = xproj.shape
    y = torch.zeros(B, T, 2 * H)
    for d in range(2):
        W = whh[d]
        c = torch.zeros(B, H)
        for s in range(T):
            t = s if d == 0 else T - 1 - s
            tp, tpp = (t - 1, t - 2) if d == 0 else (t + 1, t + 2)
            pre = xproj[:, t, d * 4 * H:(d + 1) * 4 * H].clone()
            if s > 0:
                def slices(hp):
                    return [hp[:, SLICE_COLS[k]] @ W[:, SLICE_COLS[k]].t() for k in range(8)]
                p = slices(y[:, tp, d * H:(d + 1) * H])
                if stale is not None and stale[:2] == (d, s):
                    old = slices(y[:, tpp, d * H:(d + 1) * H])
                    cols = torch.cat([torch.arange(stale[2], stale[2] + 16) + g * H for g in range(4)])
                    for k in range(8):
                        p[k][:32, cols] = old[k][:32, cols]
                if drop is not None and drop[:2] == (d, s):
                    _, _, u, row, k = drop
                    p[k][row, torch.arange(4) * H + u] = 0
                pre = pre + (((p[0] + p[4]) + (p[2] + p[6])) + ((p[1] + p[5]) + (p[3] + p[7])))
            i, f, g, o = pre.split(H, -1)
            c = torch.sigmoid(f) * c + torch.sigmoid(i) * torch.tanh(g)
            y[:, t, d * H:(d + 1) * H] = torch.sigmoid(o) * torch.tanh(c)
    if swap_row is not None:
        y[swap_row] = torch.cat([y[swap_row, :, H:], y[swap_row, :, :H]], -1)
    return y


def _lstm_inputs(B, T, x_scale=1.0, seed=23):
    xproj = _rand(B, T, 8 * H, seed=seed, scale=x_scale)
    whh = _rand(2, 4 * H, H, seed=seed + 1, scale=1.2 / math.sqrt(H))
    return xproj, whh


@pytest.mark.parametrize("x_scale", [1.0, 8.0])
def test_lstm_bound_accepts_fp32_and_rejects_bugs(x_scale):
    B, T = 40, 6                                                      # two halves, the second partial (rows 32..39)
    xproj, whh = _lstm_inputs(B, T, x_scale)
    good = _lstm32(xproj, whh)
    want, bound = sb.lstm_bidir_f32(xproj, whh, good)
    assert sb.within(good, want, bound)
    for mutant in (dict(drop=(0, 3, 17, 5, 6)), dict(drop=(1, 1, 500, 39, 0)),
                   dict(stale=(0, 4, 48)), dict(stale=(1, 2, 0)),
                   dict(swap_row=31), dict(swap_row=39)):
        bad = _lstm32(xproj, whh, **mutant)
        assert not sb.within(bad, *sb.lstm_bidir_f32(xproj, whh, bad)), mutant


def test_lstm_bound_first_step_and_single_step():
    """t = 1 (no recurrent product at all) and the first step of each direction: h = o tanh(i g) from x alone."""
    xproj, whh = _lstm_inputs(3, 1, seed=31)
    good = _lstm32(xproj, whh)
    want, bound = sb.lstm_bidir_f32(xproj, whh, good)
    assert sb.within(good, want, bound)
    bad = good.clone()
    bad[1, 0, 7] += 64 * sb.U * max(abs(float(bad[1, 0, 7])), 1e-3)
    assert not sb.within(bad, want, bound)

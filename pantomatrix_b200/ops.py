"""Thin torch-tensor wrappers over the C ABI (include/pm_emage.h).

torch is used only for device memory (torch.empty), the current CUDA stream and tensor views; every
arithmetic op of the hot path is a kernel of libpm_emage.so.  All functions require CUDA tensors and
raise (PmError) on any failure - there is no fallback.
"""
from __future__ import annotations

import math

import torch

from . import _lib

ACT_NONE, ACT_RELU, ACT_LEAKY = 0, 1, 2
ROW_NONE, ROW_PE, ROW_SPK = 0, 1, 2

# number of kernel launches issued through this module (bench.py reports it as gpu_launches)
launch_count = 0

# Element format of the tensor-core operand planes: bf16 (default) or IEEE fp16.  Two fp16 planes (3 products)
# match three bf16 planes (6 products) in accuracy while magnitudes stay below 65504 (include/pm_emage.h).
FMT_F16 = 0x100
TC_TILE_SHIFT = 16           # pm_tapgemm_tc: N tile override in bits 16-23 of nsplit (PM_TC_TILE_SHIFT)
TC_STORE_LOOP = 1 << 24      # pm_tapgemm_tc: force the per-element store loop (PM_TC_STORE_LOOP)
# fp16 activation planes hold F16_ACT_SCALE * x (csrc/pm_common.cuh PM_F16_ACT_SCALE: the tensor core flushes fp16
# subnormal operands, the exact pre-scale keeps second planes normal down to |x| = 2^-9); PackedW.acc_scale undoes it.
F16_ACT_SCALE = 64.0
_PLANE_DTYPE = torch.bfloat16


def set_plane_format(name: str) -> None:
    global _PLANE_DTYPE
    _PLANE_DTYPE = {"bf16": torch.bfloat16, "fp16": torch.float16}[name]


def plane_format() -> str:
    return "fp16" if _PLANE_DTYPE == torch.float16 else "bf16"


def _fmt_bit(t) -> int:
    return FMT_F16 if t.dtype == torch.float16 else 0


def _stream() -> int:
    return torch.cuda.current_stream().cuda_stream


def _ptr(t) -> int | None:
    return None if t is None else t.data_ptr()


def _chk(t: torch.Tensor, dtype=torch.float32):
    if not t.is_cuda:
        raise _lib.PmError("pantomatrix_b200 ops need CUDA tensors (no CPU fallback)")
    if t.dtype != dtype:
        raise _lib.PmError(f"expected {dtype}, got {t.dtype}")
    if t.dim() and t.stride(-1) != 1 and t.shape[-1] != 1:
        raise _lib.PmError("innermost dimension must be contiguous")
    return t


def _call(name, *args):
    global launch_count
    launch_count += 1
    _lib.call(name, *args)


def _bs_ld(t: torch.Tensor):
    """(batch stride, row stride) in elements of a (batch, rows, ch) view."""
    return (t.stride(0) if t.shape[0] > 1 else t.shape[1] * t.stride(1)), t.stride(1)


def tapgemm(a, w, bias, *, rows_out=None, stride=1, pad=0, act=ACT_NONE, slope=0.0, residual=None, out=None):
    """out[b,l,:] = act(bias + sum_t A[b, l*stride+t-pad, :] @ W[t].T + residual[b,l,:]).

    a: (batch, rows_in, cin); w: (taps, cout, cin) contiguous; returns (batch, rows_out, cout)."""
    _chk(a), _chk(w)
    batch, rows_in, cin = a.shape
    taps, cout, cin_w = w.shape
    assert cin_w == cin and w.is_contiguous(), (w.shape, a.shape)
    if rows_out is None:
        rows_out = (rows_in + 2 * pad - taps) // stride + 1
    if out is None:
        out = torch.empty(batch, rows_out, cout, device=a.device, dtype=torch.float32)
    else:
        assert out.shape == (batch, rows_out, cout), (out.shape, (batch, rows_out, cout))
    _chk(out)
    if residual is not None:
        _chk(residual)
        assert residual.shape == out.shape
    # a Linear (taps == 1, no padding) over contiguous batches is one tall matrix: better tile use.  Only when every
    # input row has its output row: with rows_out < rows_in, clip b's rows would start at b * rows_out of the tall A.
    if (taps == 1 and pad == 0 and stride == 1 and batch > 1 and rows_out == rows_in
            and a.stride(0) == rows_in * a.stride(1)
            and out.stride(0) == rows_out * out.stride(1)
            and (residual is None or residual.stride(0) == rows_out * residual.stride(1))):
        a = a.reshape(1, batch * rows_in, cin) if a.is_contiguous() else a.as_strided(
            (1, batch * rows_in, cin), (0, a.stride(1), 1), a.storage_offset())
        flat = lambda t: t.as_strided((1, batch * rows_out, cout), (0, t.stride(1), 1), t.storage_offset())
        out_v = flat(out)
        res_v = flat(residual) if residual is not None else None
        batch_k, rows_in_k, rows_out_k = 1, batch * rows_in, batch * rows_out
    else:
        out_v, res_v, batch_k, rows_in_k, rows_out_k = out, residual, batch, rows_in, rows_out
    a_bs, lda = _bs_ld(a)
    o_bs, ldo = _bs_ld(out_v)
    r_bs, ldr = _bs_ld(res_v) if res_v is not None else (0, 0)
    _call("pm_tapgemm_f32", a.data_ptr(), a_bs, lda, batch_k, rows_in_k, cin,
          w.data_ptr(), _ptr(bias), taps, stride, pad, rows_out_k, cout,
          _ptr(res_v), r_bs, ldr, act, float(slope), out_v.data_ptr(), o_bs, ldo, _stream())
    return out


def wav_stem(audio, a_bs, a_ws, batch, windows, n_samples, w1, b1, wd, bd, *, stride, pad, slope, offset=0, nsplit=0):
    """First WavEncoder block's two convolutions on the raw waveform.  `audio` is the flat (bs, n)
    tensor; sequence (b, w) starts at element offset + b*a_bs + w*a_ws and is n_samples long.
    Returns (y1, sc): y1 as fp32 tensor (nsplit 0) or as the operand Planes of the conv that follows."""
    _chk(audio)
    cout, ks = w1.shape
    rows_out = (n_samples + 2 * pad - ks) // stride + 1
    sc = torch.empty(batch * windows, rows_out, cout, device=audio.device, dtype=torch.float32)
    if nsplit:
        y1 = _new_planes(nsplit, (batch * windows, rows_out), cout, audio.device)
        y_ptr, pa = 0, (y1.t.data_ptr(), y1.t.stride(0), y1.t.stride(2), nsplit | _fmt_bit(y1.t))
    else:
        y1 = torch.empty_like(sc)
        y_ptr, pa = y1.data_ptr(), (0, 0, 0, 0)
    _call("pm_wav_stem_f32", audio.data_ptr() + 4 * offset, a_bs, a_ws, batch, windows, n_samples,
          w1.data_ptr(), b1.data_ptr(), wd.data_ptr(), bd.data_ptr(), cout, ks, stride, pad, rows_out,
          float(slope), y_ptr, sc.data_ptr(), *pa, _stream())
    return y1, sc


def resample_poly(pcm, bank, up, down, n_pre_remove, out=None):
    """Recorded audio -> mono fp32 at up/down times its rate (include/pm_emage.h pm_resample_poly_f32).

    pcm: (batch, n_in, channels) int16 or float32, samples and channels dense (any clip stride); bank: (up, taps)
    float32 polyphase filter (audio_io.Resampler builds it).  Returns out (batch, ceil(n_in*up/down)) float32; a given
    `out` may be a view with any clip stride (e.g. a column range of a wider buffer)."""
    if pcm.dtype not in (torch.int16, torch.float32):
        raise _lib.PmError(f"resample_poly: PCM must be int16 or float32, got {pcm.dtype}")
    if pcm.dim() != 3:
        raise _lib.PmError(f"resample_poly: PCM must be (batch, n_in, channels), got shape {tuple(pcm.shape)}")
    _chk(pcm, pcm.dtype), _chk(bank)
    batch, n_in, channels = pcm.shape
    if n_in > 1 and pcm.stride(1) != channels:
        raise _lib.PmError("resample_poly: the samples of a clip must be dense (interleaved channels)")
    if not bank.is_contiguous() or bank.dim() != 2 or bank.shape[0] != up:
        raise _lib.PmError(f"resample_poly: bank must be a contiguous (up={up}, taps) tensor, got {tuple(bank.shape)}")
    n_out = -(-n_in * up // down)
    if out is None:
        out = torch.empty(batch, n_out, device=pcm.device, dtype=torch.float32)
    elif tuple(out.shape) != (batch, n_out):
        raise _lib.PmError(f"resample_poly: out must be {(batch, n_out)}, got {tuple(out.shape)}")
    _chk(out)
    _call("pm_resample_poly_f32", pcm.data_ptr(), int(pcm.dtype == torch.int16), pcm.stride(0) if batch > 1 else 0,
          batch, n_in, channels, bank.data_ptr(), int(up), int(down), bank.shape[1], int(n_pre_remove),
          out.data_ptr(), out.stride(0) if batch > 1 else 0, _stream())
    return out


class Act:
    """One activation as fp32 tensor (`f`) and/or split-bf16 planes (`p`); either may be None."""
    __slots__ = ("f", "p")

    def __init__(self, f=None, p=None):
        self.f, self.p = f, p


def _new_planes(nsplit, lead_shape, ch, device, slack_rows=0, dtype=None):
    """Planes for an activation of shape (*lead_shape, ch); lead_shape = (batch, rows)."""
    batch, rows = lead_shape
    dtype = dtype or _PLANE_DTYPE
    ld = _round_up(ch, 8)
    if slack_rows:
        buf = torch.empty(nsplit, batch * rows + slack_rows, ld, device=device, dtype=dtype)
        if buf.is_cuda:
            for i in range(nsplit):               # cudaMemsetAsync: a memset node under graph capture, not a kernel
                _lib.call("pm_memset_async", buf[i, batch * rows:].data_ptr(), 0, slack_rows * ld * buf.element_size(), _stream())
        else:
            buf[:, batch * rows:].zero_()
        t = buf[:, :batch * rows].view(nsplit, batch, rows, ld)
    else:
        t = torch.empty(nsplit, batch, rows, ld, device=device, dtype=dtype)
    return Planes(t, rows, ch, slack_rows)


def _pargs(pl):
    if pl is None:
        return None, 0, 0, 0
    return pl.t.data_ptr(), pl.t.stride(0), pl.t.stride(2), pl.t.shape[0] | _fmt_bit(pl.t)


def _result(f, pl, nsplit):
    return f if nsplit == 0 else Act(f, pl)


def add_layernorm(x, r, gamma, beta, eps=1e-5, nsplit=0, f32=True):
    _chk(x)
    assert x.is_contiguous() and (r is None or (r.is_contiguous() and r.shape == x.shape))
    ch = x.shape[-1]
    rows = x.numel() // ch
    out = torch.empty_like(x) if (f32 or not nsplit) else None
    pl = _new_planes(nsplit, (x.shape[0], rows // x.shape[0]), ch, x.device) if nsplit else None
    _call("pm_add_layernorm_f32", x.data_ptr(), _ptr(r), gamma.data_ptr(), beta.data_ptr(), _ptr(out),
          rows, ch, float(eps), *_pargs(pl), _stream())
    return _result(out, pl, nsplit)


def attention(q, k, v, batch, heads, tq, tk, head_dim, nsplit=0, f32=True):
    """q: (batch*tq, >=heads*head_dim) view, k/v: (batch*tk, ...) views (column slices allowed)."""
    for t in (q, k, v):
        _chk(t)
    E = heads * head_dim
    out = torch.empty(batch * tq, E, device=q.device, dtype=torch.float32) if (f32 or not nsplit) else None
    pl = _new_planes(nsplit, (batch, tq), E, q.device) if nsplit else None
    _call("pm_attention_f32", q.data_ptr(), q.stride(0), k.data_ptr(), k.stride(0), v.data_ptr(), v.stride(0),
          _ptr(out), E, batch, heads, tq, tk, head_dim, *_pargs(pl), _stream())
    return _result(out, pl, nsplit)


def attention_tc(q, q_col0, k, k_col0, v, v_col0, batch, heads, tq, tk, head_dim, nsplit=2, f32=False):
    """Attention on the wgmma tensor cores (fp16x3 engine).  q / k / v: two-plane fp16 Planes whose columns
    [*_col0 + h*head_dim, ...) hold head h (the packed q|k|v or k|v projection output is passed as is)."""
    for pl, rows in ((q, tq), (k, tk), (v, tk)):
        assert pl.t.dtype == torch.float16 and pl.t.shape[0] == 2 and pl.t.shape[1] == batch and pl.rows == rows, \
            "attention_tc needs two-plane fp16 operands of (batch, rows, ch)"
    E = heads * head_dim
    dev = q.t.device
    out = torch.empty(batch * tq, E, device=dev, dtype=torch.float32) if (f32 or not nsplit) else None
    pl = _new_planes(nsplit, (batch, tq), E, dev, dtype=torch.float16) if nsplit else None
    _call("pm_attention_tc",
          q.t.data_ptr(), q.t.stride(0), q.t.stride(1), q.t.stride(2), q.ch, q_col0,
          k.t.data_ptr(), k.t.stride(0), k.t.stride(1), k.t.stride(2), k.ch, k_col0,
          v.t.data_ptr(), v.t.stride(0), v.t.stride(1), v.t.stride(2), v.ch, v_col0,
          _ptr(out), E, batch, heads, tq, tk, head_dim, *_pargs(pl), _stream())
    return _result(out, pl, nsplit)


def add_rows(x, pe, spk, first, second, batch, rows, ch, nsplit=0, f32=True):
    dev = (pe if pe is not None else spk).device
    out = torch.empty(batch, rows, ch, device=dev, dtype=torch.float32) if (f32 or not nsplit) else None
    if x is not None:
        _chk(x)
        assert x.is_contiguous() and x.numel() == batch * rows * ch
    pl = _new_planes(nsplit, (batch, rows), ch, dev) if nsplit else None
    _call("pm_add_rows_f32", _ptr(x), _ptr(pe), _ptr(spk), first, second, _ptr(out), batch, rows, ch, *_pargs(pl), _stream())
    return _result(out, pl, nsplit)


def add2(a, b, nsplit=0, f32=True):
    """a + b (pm_add2_f32).  Dense operands, or (fp32 out only) (..., ch) views with evenly spaced rows - e.g. the two
    column halves of a BiLSTM output, read in place.  Returns a dense tensor / Act."""
    _chk(a), _chk(b)
    assert a.shape == b.shape, (a.shape, b.shape)
    n, ch = a.numel(), a.shape[-1]
    if not (a.is_contiguous() and b.is_contiguous()):
        assert nsplit == 0, "strided add2 writes fp32 only"
        out, pl = torch.empty(a.shape, device=a.device, dtype=torch.float32), None
        (rows, lda), ldb, ldo = _rows_ld(a), _rows_ld(b)[1], ch
    else:
        out = torch.empty_like(a) if (f32 or not nsplit) else None
        pl = _new_planes(nsplit, (a.shape[0], n // ch // a.shape[0]), ch, a.device) if nsplit else None
        # planes are written per row of ch; fp32 alone is one row of n, so 16-byte access does not depend on ch
        rows, lda = (n // ch, ch) if nsplit else (1, n)
        ch = ldb = ldo = lda
    _call("pm_add2_f32", a.data_ptr(), lda, b.data_ptr(), ldb, _ptr(out), ldo, rows, ch, *_pargs(pl), _stream())
    return _result(out, pl, nsplit)


def _rows_ld(t):
    """(rows, row stride) of a (..., ch) view whose rows all lie one stride apart (e.g. a column range)."""
    ch = t.shape[-1]
    rows = t.numel() // ch if ch else 0
    lead = [(n, s) for n, s in zip(t.shape[:-1], t.stride()[:-1]) if n > 1]
    ld = lead[-1][1] if lead else ch
    want = ld
    for n, s in reversed(lead):
        if s != want:
            raise _lib.PmError(f"rows of a {tuple(t.shape)} view with strides {t.stride()} are not evenly spaced")
        want = s * n
    return rows, ld


def lstm_cond(spk, speaker_id, seed, seed_len, seed_frames, pose_dims, out):
    """Speaker row + seed columns of the layer-0 LSTM input, written into `out` (batch, t, spk_dim + pose_dims + 1), a
    column range of that input (include/pm_emage.h pm_lstm_cond_f32).  speaker_id int64 (batch,) or (batch, 1), clamped
    into the table; seed (batch, rows, pose_dims) with dense rows or None (zeros); seed_len is the length of the
    sequence the seed stands for (row mapping in the header)."""
    _chk(spk), _chk(speaker_id, torch.int64), _chk(out)
    assert spk.is_contiguous() and speaker_id.is_contiguous()
    batch, t, cols = out.shape
    assert speaker_id.numel() == batch and cols == spk.shape[1] + pose_dims + 1, (speaker_id.shape, out.shape)
    o_bs, ldo = _bs_ld(out)
    s_bs = s_ld = 0
    if seed is not None:
        _chk(seed)
        assert seed.dim() == 3 and seed.shape[0] == batch and seed.shape[2] == pose_dims, (seed.shape, batch, pose_dims)
        if seed.numel() == 0:
            seed = None
        else:
            s_bs, s_ld = _bs_ld(seed)
    _call("pm_lstm_cond_f32", spk.data_ptr(), spk.shape[0], spk.shape[1], speaker_id.data_ptr(), _ptr(seed), s_bs, s_ld,
          int(seed_len), int(seed_frames), int(pose_dims), out.data_ptr(), o_bs, ldo, batch, t, _stream())
    return out


def window_input(motion, mask, seed, mask_embedding, start, win_len, pre, nsplit=0, f32=True, shape=None):
    """motion / mask: (batch, total_len, ch) or None = inference()'s defaults (then `shape` = (batch, total_len, ch));
    seed: (batch, pre, ch) view with dense rows (any clip stride), None when pre == 0."""
    batch, total_len, ch = motion.shape if motion is not None else shape
    for t in (motion, mask):
        if t is not None:
            _chk(t)
            assert t.is_contiguous() and t.shape == (batch, total_len, ch)
    seed_bs = 0
    if seed is not None:
        _chk(seed)
        assert seed.shape == (batch, pre, ch) and (pre <= 1 or seed.stride(1) == ch)
        seed_bs = seed.stride(0)
    dev = mask_embedding.device
    out = torch.empty(batch, win_len, ch, device=dev, dtype=torch.float32) if (f32 or not nsplit) else None
    pl = _new_planes(nsplit, (batch, win_len), ch, dev) if nsplit else None
    _call("pm_window_input_f32", _ptr(motion), _ptr(mask), _ptr(seed), mask_embedding.data_ptr(),
          _ptr(out), batch, total_len, start, win_len, pre, ch, seed_bs, *_pargs(pl), _stream())
    return _result(out, pl, nsplit)


def _batched_rows(x, ld):
    """(rows, rows_per_batch, batch stride) of a (rows, ch) matrix or a (batch, rows, ch) view whose rows are `ld` apart."""
    if x.dim() == 2:
        assert x.stride(0) == ld
        return x.shape[0], 0, 0
    assert x.dim() == 3 and (x.shape[1] == 1 or x.stride(1) == ld)
    return x.shape[0] * x.shape[1], x.shape[1], x.stride(0)


def l2_argmin(z, codebook, e2, engine="auto", max_ctas=0):
    """fp32 argmin_k |z - e_k|^2, first minimum wins.  engine: "auto" (the product path: tensor-core screen + exact fp32
    re-scoring for 256-code codebooks, fp32 SIMT otherwise), "tc" or "simt" (tests / microbenchmarks)."""
    _chk(z), _chk(codebook), _chk(e2)
    assert codebook.is_contiguous()
    n_codes, e_dim = codebook.shape
    if z.dim() > 3:
        z = z.reshape(-1, e_dim)
    rows, rpb, z_bs = _batched_rows(z, e_dim)      # (rows, 256) or a (batch, rows, 256) view, e.g. the tail of a window
    idx = torch.empty(z.shape[:-1], device=z.device, dtype=torch.int64)
    if engine == "tc":
        _call("pm_l2_argmin_tc", z.data_ptr(), rows, rpb, z_bs, codebook.data_ptr(), e2.data_ptr(), n_codes, e_dim,
              idx.data_ptr(), int(max_ctas), _stream())
    elif engine == "simt":
        _call("pm_l2_argmin_simt_f32", z.data_ptr(), rows, rpb, z_bs, codebook.data_ptr(), e2.data_ptr(), n_codes, e_dim,
              idx.data_ptr(), _stream())
    else:
        _call("pm_l2_argmin_f32", z.data_ptr(), rows, rpb, z_bs, codebook.data_ptr(), e2.data_ptr(), n_codes, e_dim,
              idx.data_ptr(), _stream())
    return idx


def row_argmax(x, nonfinite=None):
    """First argmax over the last dim of a (rows, ch) matrix or a (batch, rows, ch) view (any clip stride).
    nonfinite: optional int32[1] device flag, set to 1 when a NaN / inf is read (never cleared here)."""
    _chk(x)
    ch = x.shape[-1]
    if x.dim() > 3:
        x = x.reshape(-1, ch)
    ld = x.stride(-2) if x.shape[-2] > 1 else ch
    rows, rpb, x_bs = _batched_rows(x, ld)
    idx = torch.empty(x.shape[:-1], device=x.device, dtype=torch.int64)
    _call("pm_row_argmax_f32", x.data_ptr(), rows, ch, ld, rpb, x_bs, idx.data_ptr(), _ptr(nonfinite), _stream())
    return idx


def zero_flag(device):
    """int32[1] device flag cleared by a memset node (no kernel)."""
    flag = torch.empty(1, device=device, dtype=torch.int32)
    _lib.call("pm_memset_async", flag.data_ptr(), 0, 4, _stream())
    return flag


def gather_rows(codebook, index, nsplit=0, f32=True):
    _chk(codebook), _chk(index, torch.int64)
    assert index.is_contiguous()
    ch = codebook.shape[1]
    out = torch.empty(*index.shape, ch, device=codebook.device, dtype=torch.float32) if (f32 or not nsplit) else None
    pl = None
    if nsplit:
        lead = (index.shape[0], index.numel() // index.shape[0]) if index.dim() > 1 else (1, index.numel())
        pl = _new_planes(nsplit, lead, ch, codebook.device)
    _call("pm_gather_rows_f32", codebook.data_ptr(), codebook.shape[0], index.data_ptr(), index.numel(), ch, _ptr(out),
          *_pargs(pl), _stream())
    return _result(out, pl, nsplit)


def row_sqnorm(x):
    _chk(x)
    out = torch.empty(x.shape[0], device=x.device, dtype=torch.float32)
    _call("pm_row_sqnorm_f32", x.data_ptr(), x.shape[0], x.shape[1], out.data_ptr(), _stream())
    return out


def pose_compose(face, upper, hands, lower, bs, t, device):
    for ten, dim in ((face, 106), (upper, 78), (hands, 180), (lower, 61)):
        if ten is not None:
            _chk(ten)
            assert ten.is_contiguous() and ten.shape == (bs, t, dim), (ten.shape, dim)
    expression = torch.empty(bs, t, 100, device=device, dtype=torch.float32)
    axis_angle = torch.empty(bs, t, 165, device=device, dtype=torch.float32)
    motion4inf = torch.empty(bs, t, 337, device=device, dtype=torch.float32)
    _call("pm_pose_compose_f32", _ptr(face), _ptr(upper), _ptr(hands), _ptr(lower), expression.data_ptr(),
          axis_angle.data_ptr(), motion4inf.data_ptr(), bs * t, _stream())
    return expression, axis_angle, motion4inf


def global_trans(rec, ref_trans, dt, vel_off=54):
    _chk(rec), _chk(ref_trans)
    assert rec.is_contiguous()
    bs, t, ld = rec.shape
    assert ref_trans.shape == (bs, 3)                      # may be an expanded (stride 0) view of one row
    trans = torch.empty(bs, t, 3, device=rec.device, dtype=torch.float32)
    _call("pm_global_trans_f32", rec.data_ptr(), ld, vel_off, ref_trans.data_ptr(), ref_trans.stride(0), float(dt),
          trans.data_ptr(), bs, t, _stream())
    return trans


# ------------------------------------------------------------------------------------------------------
# wgmma tensor-core engine: split-bf16 planes
# ------------------------------------------------------------------------------------------------------


def _round_up(x, m):
    return (x + m - 1) // m * m


class Planes:
    """`nsplit` bf16 planes of a (batch, rows, ch) activation: tensor (nsplit, batch, rows_alloc, ld) bf16
    with x ~ sum_p planes[p].  Only [:, :, :rows, :ch] is meaningful."""
    __slots__ = ("t", "rows", "ch", "slack")

    def __init__(self, t, rows, ch, slack=0):
        self.t, self.rows, self.ch, self.slack = t, rows, ch, slack   # slack: zeroed rows after the last clip

    def flat(self):
        """(nsplit, 1, batch*rows, ld) view: all clips as one tall matrix (needs clip-contiguous rows)."""
        ns, b, r, ld = self.t.shape
        assert self.t.stride(1) == r * self.t.stride(2)
        return Planes(self.t.as_strided((ns, 1, b * r, ld), (self.t.stride(0), b * r * self.t.stride(2), self.t.stride(2), 1),
                                        self.t.storage_offset()), b * r, self.ch, self.slack)

    @property
    def nsplit(self):
        return self.t.shape[0]

    @property
    def batch(self):
        return self.t.shape[1]


def split_bf16(x, nsplit, slack_rows=0):
    """fp32 (batch, rows, ch) view -> Planes (ld = ch rounded up to 8).  `slack_rows` zeroed rows are
    appended after the last clip for strided-view consumers."""
    _chk(x)
    batch, rows, ch = x.shape
    pl = _new_planes(nsplit, (batch, rows), ch, x.device, slack_rows)
    x_bs, ldx = _bs_ld(x)
    _call("pm_split_bf16", x.data_ptr(), x_bs, ldx, batch, rows, ch, pl.t.data_ptr(), pl.t.stride(0), pl.t.stride(1),
          pl.t.stride(2), nsplit | _fmt_bit(pl.t), _stream())
    return pl


class PackedW:
    """Weights of one tap-GEMM for the tensor-core engine: (nsplit, taps, w_rows, ldw) bf16 (or fp16) planes.
    fp16 planes hold W * 2^k with the largest |W| in [16384, 32768) - small weights keep their second plane out of
    the fp16 subnormals - and `acc_scale` = 2^-k / F16_ACT_SCALE is handed to the kernel's epilogue."""
    __slots__ = ("t", "taps", "cout", "cin", "w_rows", "ldw", "acc_scale")

    def __init__(self, w, nsplit):
        """w: fp32 (taps, cout, cin)."""
        taps, cout, cin = w.shape
        bn = 64 if cout <= 64 else 128
        self.taps, self.cout, self.cin = taps, cout, cin
        self.w_rows, self.ldw = _round_up(cout, bn), _round_up(cin, 8)
        full = torch.zeros(taps, self.w_rows, self.ldw, device=w.device, dtype=torch.float32)
        full[:, :cout, :cin] = w
        self.acc_scale = 1.0
        if _PLANE_DTYPE == torch.float16:
            m = float(full.abs().max())
            if m > 0.0 and math.isfinite(m):
                k = math.floor(math.log2(32768.0 / m))
                full = full * (2.0 ** k)
                self.acc_scale = 2.0 ** -k
            self.acc_scale /= F16_ACT_SCALE                  # activation planes arrive pre-scaled (exact power of two)
        planes, rem = [], full
        for _ in range(nsplit):                       # round-to-nearest-even, same as the device split
            p = rem.to(_PLANE_DTYPE)
            planes.append(p)
            rem = rem - p.float()
        self.t = torch.stack(planes).contiguous()


def tapgemm_tc(a: Planes, w: PackedW, bias, *, rows_in=None, rows_out, pad=0, act=ACT_NONE, act_cols=0, slope=0.0,
               residual=None, want_f32=True, out_nsplit=0, out=None, a_view=None, out_slack=0, prefetch=None, tile=0,
               store_loop=False):
    """Tensor-core tap-GEMM.  `prefetch`: a tensor (the next GEMM's packed weights) to pull into L2 meanwhile.
    `a_view` = (rows_in, cin, lda) overrides the logical view of the A planes
    (strided convs pass the (rows/s, s*C) view of the same memory).  `tile` forces the kernel's N tile (64 or 128
    columns; 0 = chosen from the shape), for tests and A/B runs: results are bit-identical either way.  `store_loop`
    forces the epilogue's per-element store loop instead of its TMA stores (tests, A/B runs; the same bits).
    Returns (fp32 out | None, Planes | None)."""
    t = a.t
    nsplit, batch = t.shape[0], t.shape[1]
    assert nsplit == w.t.shape[0] and t.dtype == w.t.dtype, "A and W must use the same split and plane format"
    fmt = _fmt_bit(t)
    rows_a, cin, lda = (a.rows, a.ch, t.stride(2)) if a_view is None else a_view
    if rows_in is not None:
        rows_a = rows_in
    assert cin == w.cin, (cin, w.cin)
    assert tile in (0, 64, 128), tile
    cout = w.cout
    dev = t.device
    out_f = None
    if want_f32:
        out_f = out if out is not None else torch.empty(batch, rows_out, cout, device=dev, dtype=torch.float32)
        assert out_f.shape == (batch, rows_out, cout)
    o_bs, ldo = _bs_ld(out_f) if out_f is not None else (0, 0)
    out_p = None
    if out_nsplit:
        out_p = _new_planes(out_nsplit, (batch, rows_out), cout, dev, out_slack, dtype=t.dtype)
    r_bs, ldr = _bs_ld(residual) if residual is not None else (0, 0)
    if residual is not None:
        _chk(residual)
        assert residual.shape == (batch, rows_out, cout)
    _call("pm_tapgemm_tc", t.data_ptr(), t.stride(0), t.stride(1), lda, batch, rows_a, cin,
          w.t.data_ptr(), w.t.stride(0), w.w_rows, w.ldw, w.taps, pad, nsplit | fmt | (tile // 64) << TC_TILE_SHIFT | (TC_STORE_LOOP if store_loop else 0),
          _ptr(bias), rows_out, cout, _ptr(residual), r_bs, ldr, act, act_cols, float(slope), float(w.acc_scale),
          _ptr(out_f), o_bs, ldo,
          None if out_p is None else out_p.t.data_ptr(), 0 if out_p is None else out_p.t.stride(0),
          0 if out_p is None else out_p.t.stride(1), 0 if out_p is None else out_p.t.stride(2),
          out_nsplit | (fmt if out_nsplit else 0),
          None if prefetch is None else prefetch.data_ptr(),
          0 if prefetch is None else prefetch.numel() * prefetch.element_size(), _stream())
    return out_f, out_p


# ------------------------------------------------------------------------------------------------------
# CaMN / DisCo
# ------------------------------------------------------------------------------------------------------


def lstm_bidir(xproj, whh, barrier, hidden):
    """One bidirectional LSTM layer.  xproj (batch, t, 8*hidden) = W_ih x + b for [forward | backward] (gates
    i,f,g,o), whh (2, 4*hidden, hidden).  Returns (batch, t, 2*hidden) = [forward h | backward h]."""
    _chk(xproj), _chk(whh)
    assert xproj.is_contiguous() and whh.is_contiguous() and whh.shape == (2, 4 * hidden, hidden)
    batch, t, w = xproj.shape
    assert w == 8 * hidden
    y = torch.empty(batch, t, 2 * hidden, device=xproj.device, dtype=torch.float32)
    _call("pm_lstm_bidir_f32", xproj.data_ptr(), xproj.stride(0), xproj.stride(1), whh.data_ptr(), y.data_ptr(),
          y.stride(0), y.stride(1), barrier.data_ptr(), batch, t, hidden, _stream())
    return y


def rot6d_to_aa(rot6d, slot, n_sel):
    """rot6d (..., n_sel*6) -> axis-angle (..., 165); slot: int32[55] device tensor (position among the selected
    joints or -1)."""
    _chk(rot6d), _chk(slot, torch.int32)
    assert rot6d.is_contiguous() and rot6d.shape[-1] == n_sel * 6
    if slot.shape != (55,) or slot.device != rot6d.device:
        raise _lib.PmError(f"slot must be a dense int32 [55] tensor on {rot6d.device}, got {tuple(slot.shape)} on {slot.device}")
    rows = rot6d.numel() // (n_sel * 6)
    out = torch.empty(*rot6d.shape[:-1], 165, device=rot6d.device, dtype=torch.float32)
    _call("pm_rot6d_to_aa_f32", rot6d.data_ptr(), rows, n_sel, slot.data_ptr(), out.data_ptr(), _stream())
    return out


# ------------------------------------------------------------------------------------------------------
# SMPL-X body model
# ------------------------------------------------------------------------------------------------------


def _clip_frame_strides(x):
    """(clip stride, frame stride) of a (batch, t, ch) view."""
    return (x.stride(0), x.stride(1)) if x is not None else (0, 0)


def smplx_fk(poses, betas, expression, transl, joint_mask, tables, joints, rel=None, feat=None, planes=None):
    """Rest joints + Rodrigues + forward kinematics (include/pm_emage.h pm_smplx_fk_f32).  poses (batch, t, 165),
    betas (batch, 300), expression (batch, t, 100), transl (batch, t, 3): views with a dense last dim, the last three
    nullable.  tables = (j_template, j_dirs, pose_mean, parents, level_order, level_start) device tensors.  Writes
    joints (batch*t, 55, 3), rel (batch*t, 55, 12) and the GEMM operand row as fp32 `feat` (rows, ld) and / or Planes."""
    for x in (poses, betas, expression, transl, joints, rel, feat):
        if x is not None:
            _chk(x)
    jt, jd, pm, par, order, lstart = tables
    batch, t, _ = poses.shape
    pb, pt = _clip_frame_strides(poses)
    eb, et = _clip_frame_strides(expression)
    tb, tt = _clip_frame_strides(transl)
    _call("pm_smplx_fk_f32", poses.data_ptr(), pb, pt, _ptr(betas), 0 if betas is None else betas.stride(0),
          _ptr(expression), eb, et, _ptr(transl), tb, tt, int(joint_mask), batch, t,
          jt.data_ptr(), jd.data_ptr(), pm.data_ptr(), par.data_ptr(), order.data_ptr(), lstart.data_ptr(),
          lstart.numel() - 1, joints.data_ptr(), _ptr(rel), _ptr(feat), 0 if feat is None else feat.stride(0),
          *_pargs(planes), _stream())
    return joints


def smplx_skin(verts, n_verts, csr, rel, transl, t):
    """Linear blend skinning in place over verts (rows, ld) = v_posed (pm_smplx_skin_f32); csr = (row_ptr, col, val)."""
    _chk(verts), _chk(rel)
    row_ptr, col, val = csr
    tb, tt = _clip_frame_strides(transl)
    if transl is not None:
        _chk(transl)
    _call("pm_smplx_skin_f32", verts.data_ptr(), verts.stride(0), verts.shape[0], int(n_verts), row_ptr.data_ptr(),
          col.data_ptr(), val.data_ptr(), rel.data_ptr(), _ptr(transl), tb, tt, int(t), _stream())
    return verts


def motion_rep(poses, joints, dt, two_dt, out):
    """rep15d (batch, t, 825) of get_motion_rep_tensor from poses (batch, t, 165) and joints (batch, t, 55, 3)."""
    _chk(poses), _chk(joints), _chk(out)
    assert joints.is_contiguous() and out.is_contiguous()
    if poses.dim() != 3 or poses.shape[-1] != 165:
        raise _lib.PmError(f"poses must be a (batch, t, 165) view, got {tuple(poses.shape)}")
    batch, t, _ = poses.shape
    if joints.numel() != batch * t * 165 or tuple(out.shape) != (batch, t, 825):
        raise _lib.PmError(f"joints must hold (batch, t, 55, 3) and out be (batch, t, 825) for poses {tuple(poses.shape)}, "
                           f"got {tuple(joints.shape)} and {tuple(out.shape)}")
    pb, pt = _clip_frame_strides(poses)
    _call("pm_motion_rep_f32", poses.data_ptr(), pb, pt, joints.data_ptr(), batch, t, float(dt), float(two_dt),
          out.data_ptr(), _stream())
    return out


# ------------------------------------------------------------------------------------------------------
# SMPL-X mesh render
# ------------------------------------------------------------------------------------------------------


def mesh_vertex(verts, views, faces, vf_csr, xy, depth, normal):
    """View transform, projection, snapping and vertex normals of a chunk of xy.shape[1] (1 or 2) image views per frame
    (pm_mesh_vertex_f32).  verts: one (frames, V, 3) tensor per view, frames any stride apart; views: one (scale, (ox,
    oy, oz)) per view.  Writes xy (frames, views, V, 2) int32, depth (frames, views, V) and normal (frames, views, V,
    3)."""
    nviews = xy.shape[1]
    if len(verts) != nviews or len(views) != nviews:
        raise _lib.PmError(f"mesh_vertex: {nviews} views need {nviews} vertex tensors and transforms")
    for v in verts:
        _chk(v)
    _chk(xy, torch.int32), _chk(depth), _chk(normal), _chk(faces, torch.int32)
    v0, (s0, o0) = verts[0], views[0]
    v1, (s1, o1) = (verts[1], views[1]) if nviews == 2 else (None, (0.0, (0.0, 0.0, 0.0)))
    vf_ptr, vf_face = vf_csr
    _call("pm_mesh_vertex_f32", v0.data_ptr(), v0.stride(0), _ptr(v1), 0 if v1 is None else v1.stride(0),
          v0.shape[1], v0.shape[0], float(s0), float(o0[0]), float(o0[1]), float(o0[2]), float(s1), float(o1[0]),
          float(o1[1]), float(o1[2]), faces.data_ptr(), vf_ptr.data_ptr(), vf_face.data_ptr(), xy.data_ptr(),
          depth.data_ptr(), normal.data_ptr(), nviews, _stream())


def mesh_raster(xy, depth, faces, vis):
    """Visibility keys of a chunk (pm_mesh_raster) into vis (frames, views, 720, 480) int64, views = xy.shape[1],
    cleared here to all ones by a memset (a memset node under graph capture)."""
    _chk(xy, torch.int32), _chk(depth), _chk(faces, torch.int32), _chk(vis, torch.int64)
    assert xy.is_contiguous() and depth.is_contiguous() and vis.is_contiguous() and vis.shape[1] == xy.shape[1]
    _lib.call("pm_memset_async", vis.data_ptr(), 0xFF, vis.numel() * 8, _stream())
    _call("pm_mesh_raster", xy.data_ptr(), depth.data_ptr(), xy.shape[2], faces.data_ptr(), faces.shape[0],
          xy.shape[0], vis.data_ptr(), xy.shape[1], _stream())


def mesh_shade(vis, xy, normal, faces, out):
    """Shaded RGB of a chunk (pm_mesh_shade_u8) into out (frames, 720, views * 480, 3) uint8, views = vis.shape[1],
    frames any stride apart."""
    _chk(vis, torch.int64), _chk(xy, torch.int32), _chk(normal), _chk(faces, torch.int32), _chk(out, torch.uint8)
    if out.shape[2] != vis.shape[1] * vis.shape[3]:
        raise _lib.PmError(f"mesh_shade: {vis.shape[1]} views need out {vis.shape[1] * vis.shape[3]} wide, "
                           f"got {out.shape[2]}")
    assert out[0].is_contiguous() and normal.is_contiguous()
    _call("pm_mesh_shade_u8", vis.data_ptr(), xy.data_ptr(), normal.data_ptr(), xy.shape[2], faces.data_ptr(),
          vis.shape[0], out.data_ptr(), out.stride(0), vis.shape[1], _stream())


def time_upsample(x, k, out=None):
    """motion_io.time_upsample_numpy in float32 (pm_time_upsample_f32): x (batch, t, ch), any clip / frame strides with
    a dense last dimension -> out (batch, k*t, ch) dense."""
    _chk(x)
    batch, t, ch = x.shape
    if out is None:
        out = torch.empty(batch, k * t, ch, device=x.device, dtype=torch.float32)
    _chk(out)
    assert tuple(out.shape) == (batch, k * t, ch) and out.is_contiguous()
    xb, xt = _clip_frame_strides(x)
    _call("pm_time_upsample_f32", x.data_ptr(), xb, xt, batch, t, ch, int(k), out.data_ptr(), _stream())
    return out


# ------------------------------------------------------------------------------------------------------
# PNG encoding
# ------------------------------------------------------------------------------------------------------


def png_encode(frames, data, nbytes, row_bits, row_adler):
    """The PNG files of frames (N, H, W, 3) uint8, each frame dense, any stride apart, into the slots of data (N, cap)
    uint8 with their sizes in nbytes (N,) int64 (include/pm_emage.h pm_png_*).  row_bits / row_adler: (N, H) int64
    workspace.  The slots are cleared first by a memset (a memset node under graph capture), then four launches."""
    _chk(frames, torch.uint8), _chk(data, torch.uint8), _chk(nbytes, torch.int64)
    _chk(row_bits, torch.int64), _chk(row_adler, torch.int64)
    n, h, w, _ = frames.shape
    assert data.is_contiguous() and row_bits.is_contiguous() and row_adler.is_contiguous() and nbytes.is_contiguous()
    cap, fs = data.shape[1], frames.stride(0) if n > 1 else 3 * h * w
    _lib.call("pm_memset_async", data.data_ptr(), 0, data.numel(), _stream())
    _call("pm_png_count", frames.data_ptr(), fs, n, h, w, row_bits.data_ptr(), row_adler.data_ptr(), _stream())
    _call("pm_png_scan", n, h, w, row_bits.data_ptr(), row_adler.data_ptr(), data.data_ptr(), cap, nbytes.data_ptr(),
          _stream())
    _call("pm_png_emit", frames.data_ptr(), fs, n, h, w, row_bits.data_ptr(), data.data_ptr(), cap, _stream())
    _call("pm_png_crc", n, h, w, data.data_ptr(), cap, nbytes.data_ptr(), _stream())


# ------------------------------------------------------------------------------------------------------
# H.264 encoding
# ------------------------------------------------------------------------------------------------------


H264_I4X4 = 0x100                         # include/pm_emage.h PM_H264_I4X4: the qp flag that adds Intra 4x4


def h264_encode(frames, clip_len, qp, data, nbytes, scratch, sizes, gop=1, recon=None, search=0, mv=None,
                intra4x4=False):
    """The H.264 samples of frames (N, H, W, 3) uint8, each frame dense, any stride apart, frame i at index i % clip_len
    of its clip, into the slots of data (N, cap) uint8 with their sizes in nbytes (N,) int64 (include/pm_emage.h
    pm_h264_*).  scratch (N, H / 16, slice_cap) uint8 and sizes (N, H / 16) int32: workspace, one slice per row.
    gop: frames per group of pictures, 1 <= gop <= clip_len; gop > 1 needs recon (GOPs, H / 16, >= 24 W) uint8, one macroblock row's
    reconstruction per (GOP, row), written by each GOP's IDR frame before its P frames read it.  search: the motion
    search range in whole pixels, 0..32; search > 0 with gop > 1 runs pm_h264_encode_me and needs recon (GOPs, >= 3 H W)
    uint8, two whole-frame reconstructions per GOP, and mv (GOPs, H / 16, W / 16, 2) int16, the searched vectors.
    intra4x4: add Intra 4x4 macroblocks (qp | PM_H264_I4X4 on every path).  The slots are cleared first by a memset (a
    memset node under graph capture), then the launches."""
    _chk(frames, torch.uint8), _chk(data, torch.uint8), _chk(nbytes, torch.int64)
    _chk(scratch, torch.uint8), _chk(sizes, torch.int32)
    n, h, w, _ = frames.shape
    assert data.is_contiguous() and nbytes.is_contiguous() and scratch.is_contiguous() and sizes.is_contiguous()
    cap, fs, slice_cap = data.shape[1], frames.stride(0) if n > 1 else 3 * h * w, scratch.shape[2]
    assert 0 <= qp <= 51
    qp = qp | H264_I4X4 if intra4x4 else qp
    _lib.call("pm_memset_async", data.data_ptr(), 0, data.numel(), _stream())
    if gop == 1:
        _call("pm_h264_encode", frames.data_ptr(), fs, n, clip_len, h, w, qp, scratch.data_ptr(), slice_cap,
              sizes.data_ptr(), _stream())
    elif search > 0:
        _chk(recon, torch.uint8), _chk(mv, torch.int16)
        chains = n // clip_len * -(-clip_len // gop)
        assert 1 < gop <= clip_len and 0 < search <= 32 and n % clip_len == 0
        assert recon.is_contiguous() and recon.shape[0] >= chains and recon.shape[1] >= 3 * h * w
        assert mv.is_contiguous() and mv.shape[0] >= chains and mv.shape[1:] == (h // 16, w // 16, 2)
        _call("pm_h264_encode_me", frames.data_ptr(), fs, n, clip_len, h, w, qp, scratch.data_ptr(), slice_cap,
              sizes.data_ptr(), gop, recon.data_ptr(), recon.stride(0), search, mv.data_ptr(), mv.numel() // 2,
              _stream())
    else:
        _chk(recon, torch.uint8)
        chains = n // clip_len * -(-clip_len // gop)
        assert 1 < gop <= clip_len and n % clip_len == 0 and recon.is_contiguous()
        assert recon.shape[0] >= chains and recon.shape[1] == h // 16 and recon.shape[2] >= 24 * w
        _call("pm_h264_encode_gop", frames.data_ptr(), fs, n, clip_len, h, w, qp, scratch.data_ptr(), slice_cap,
              sizes.data_ptr(), gop, recon.data_ptr(), recon.stride(1), _stream())
    _call("pm_h264_gather", n, h, w, scratch.data_ptr(), slice_cap, sizes.data_ptr(), data.data_ptr(), cap,
          nbytes.data_ptr(), _stream())


# ------------------------------------------------------------------------------------------------------
# FLAC encoding
# ------------------------------------------------------------------------------------------------------


def flac_encode(pcm, bps, rate, data, nbytes, rec):
    """The FLAC frames of pcm (B, n, C) int16 (bps 16) or int32 (bps 24), each clip dense, clips any stride apart,
    into the slots of data (B F, cap) uint8 with their sizes in nbytes (B F,) int64 (include/pm_emage.h pm_flac_*).
    rec (B F K, 66) int32: workspace, one analysis record per (clip, frame, channel candidate).  The slots are cleared
    first by a memset (a memset node under graph capture), then two launches."""
    _chk(pcm, torch.int16 if bps == 16 else torch.int32), _chk(data, torch.uint8), _chk(nbytes, torch.int64)
    _chk(rec, torch.int32)
    b, n, c = pcm.shape
    assert data.is_contiguous() and nbytes.is_contiguous() and rec.is_contiguous()
    cs = pcm.stride(0) if b > 1 else n * c
    _lib.call("pm_memset_async", data.data_ptr(), 0, data.numel(), _stream())
    _call("pm_flac_analyse", pcm.data_ptr(), cs, b, n, c, bps, rec.data_ptr(), _stream())
    _call("pm_flac_emit", pcm.data_ptr(), cs, b, n, c, bps, rate, rec.data_ptr(), data.data_ptr(), data.shape[1],
          nbytes.data_ptr(), _stream())


def softmax2_mix(sel, c1, c2, out=None):
    """out[..., :] = softmax(sel[..., 0:2])[0] * c1 + [1] * c2 (out may be a column slice of a wider tensor)."""
    _chk(sel), _chk(c1), _chk(c2)
    assert sel.is_contiguous() and c1.is_contiguous() and c2.is_contiguous() and sel.shape[-1] == 2
    assert c2.shape == c1.shape and sel.shape[:-1] == c1.shape[:-1]
    ch = c1.shape[-1]
    rows = c1.numel() // ch
    if out is None:
        out = torch.empty_like(c1)
    _chk(out)
    if out.shape != c1.shape:
        raise _lib.PmError(f"out must be {tuple(c1.shape)}, got {tuple(out.shape)}")
    _call("pm_softmax2_mix_f32", sel.data_ptr(), c1.data_ptr(), c2.data_ptr(), out.data_ptr(), rows, ch, _row_stride(out),
          _stream())
    return out


def _row_stride(x):
    """The one row stride of a (..., ch) view whose rows lie evenly spaced, as in a (rows, ld) matrix - the layout a
    kernel taking a single leading dimension can address.  Raises PmError for any other view, e.g. a [:, :T] slice of
    a (B, T', ch) buffer with T' > T, whose clips lie T' rows apart."""
    lead = [(n, st) for n, st in zip(x.shape[:-1], x.stride()[:-1]) if n != 1]
    ld = lead[-1][1] if lead else x.shape[-1]
    step = ld
    for n, st in reversed(lead):
        if st != step:
            raise _lib.PmError(f"rows of a {tuple(x.shape)} view with strides {x.stride()} are not evenly spaced")
        step *= n
    return ld

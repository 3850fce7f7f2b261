"""Shared test helpers: product-side model construction with the synthetic checkpoints, and the float64 references
with per-element error bounds that the tensor-core kernel tests (tests/test_tapgemm_tc_gpu.py, tests/test_kernels_gpu.py,
tests/test_kernel_shadow_gpu.py) check every output element against."""
import functools
import math

import pytest
import torch

from synthetic_models import build_lstm_product, build_product  # noqa: F401  (construction lives at the repo root)

F16_ACT_SCALE = 64.0                 # fp16 activation planes hold 64 x (pantomatrix_b200.ops.F16_ACT_SCALE)
F16_MIN_NORMAL = 2.0 ** -14          # nonzero fp16 operands below this are subnormal: the tensor core may flush them
UNIT = {torch.bfloat16: 2.0 ** -8, torch.float16: 2.0 ** -11}     # relative size of plane p + 1 to plane p
ULP32 = 2.0 ** -24
STEP = 2.0 ** -22                    # error of one wgmma instruction relative to its accumulator's magnitude bound


@pytest.fixture(autouse=True)
def bf16_planes_by_default():
    """For the kernel test modules that import it: each test starts on bf16 operand planes (ops' default) unless it
    selects fp16 itself, and leaves the plane format - half of the engine's precision mode - as it found it."""
    from pantomatrix_b200 import ops
    found = ops.plane_format()
    ops.set_plane_format("bf16")
    yield
    ops.set_plane_format(found)


def use_precision(request, name: str) -> None:
    """engine.set_precision(name) for the requesting test; the mode it found is selected again afterwards."""
    from pantomatrix_b200.emage_audio import engine
    request.addfinalizer(functools.partial(engine.set_precision, engine.get_precision()))
    engine.set_precision(name)


def geodesic_deg(aa_a: torch.Tensor, aa_b: torch.Tensor) -> torch.Tensor:
    """Angle (degrees) of the relative rotation between two axis-angle tensors (..., 3): the error measure
    that is meaningful across the axis-angle discontinuity at pi."""
    from oracle.emage_oracle import axis_angle_to_quat, quat_to_matrix
    ra = quat_to_matrix(axis_angle_to_quat(aa_a.double()))
    rb = quat_to_matrix(axis_angle_to_quat(aa_b.double()))
    tr = (ra.transpose(-1, -2) @ rb).diagonal(dim1=-2, dim2=-1).sum(-1)
    return torch.rad2deg(torch.acos(torch.clamp((tr - 1) / 2, -1, 1)))


# ------------------------------------------------------------------------------------------------------------------
# split planes
# ------------------------------------------------------------------------------------------------------------------


def planes_f64(t: torch.Tensor, act: bool = True) -> torch.Tensor:
    """float64 value of split planes t (nsplit, ...): their exact sum, divided by the x64 pre-scale for fp16
    activation planes (act=True)."""
    v = t.double().sum(0)
    return v / F16_ACT_SCALE if (act and t.dtype == torch.float16) else v


def flushable_f64(t: torch.Tensor, scale: float) -> torch.Tensor | None:
    """Sum over planes of |x| * scale for the nonzero fp16 subnormal plane elements (the tensor core may read them as
    zero), None for bf16 planes (no tensor of this model reaches the bf16 subnormals)."""
    if t.dtype != torch.float16:
        return None
    a = t.double().abs()
    return (a * ((a > 0) & (a < F16_MIN_NORMAL))).sum(0) * scale


def plane_bound(nsplit: int, dtype, value: torch.Tensor) -> torch.Tensor:
    """Largest |planes - value| when `value` (fp32) is split into `nsplit` planes: each plane holds the rounded running
    remainder, so the split keeps 8 (bf16) or 11 (fp16) more bits per plane, at most the 24 of fp32.  Below 2^-14 (after
    the x64 pre-scale) fp16 planes are subnormals with an absolute resolution of 2^-24: each of two planes may round
    by 2^-25 there (pm_f16_head forms an 11-bit head that is only exact in the normal range), 2^-24 / 64 in activation
    units."""
    rel = 1.01 * max(UNIT[dtype] ** nsplit, ULP32)
    floor = 2.0 ** -24 / F16_ACT_SCALE if dtype == torch.float16 else 0.0
    return rel * value.abs() + floor


def slack_rows(pl) -> torch.Tensor:
    """The zeroed rows a Planes object carries after its last clip (ops._new_planes), as a (nsplit, slack, ld) view."""
    ns, b, r, ld = pl.t.shape
    return pl.t.as_strided((ns, pl.slack, ld), (pl.t.stride(0), ld, 1), pl.t.storage_offset() + b * r * ld)


# ------------------------------------------------------------------------------------------------------------------
# tap-GEMM (pm_tapgemm_tc)
# ------------------------------------------------------------------------------------------------------------------


def tapgemm_c(nsplit: int, dtype, n_iter: int) -> float:
    """Relative bound c_mode of the tensor-core tap-GEMM: |err_ij| <= c_mode * (|A_eff| @ |W_eff|)_ij + (fp32 ulps of
    the epilogue, tapgemm_reference).  A_eff and W_eff are the plane sums the kernel received, so only what the kernel
    itself does enters:

    * Dropped products.  With u = 2^-8 (bf16) or 2^-11 (fp16) plane p of x is at most (1.01 u)^p |x|.  The kernel
      computes the products of planes (i, j) with i + j < nsplit, so it drops (1,1) for nsplit 2 (<= u^2) and
      (1,2), (2,1), (2,2) for nsplit 3 (<= 2 u^3 + u^4); nsplit 1 drops nothing.  bf16x3: ~2^-16, fp16x3: ~2^-22,
      bf16x6: ~2^-23 (times 1.01^k).
    * fp32 accumulation (mma_kblock).  The p0*p0 products of a 64-channel k-block (4 wgmma k16 instructions) go
      alternately into two main accumulators, so each main chain is L = 4 ceil(n_iter / 2) ~ K / 32 instructions long
      (n_iter = taps * ceil(cin / 64), K = 64 n_iter).  One instruction aligns its 16 exact products to the largest
      exponent and truncates: it errs by at most STEP = 2^-22 of the running |sum|, which is <= |A_eff| @ |W_eff|.
      The cross products (at most 2.1 u of it in total) go into the correction accumulator, (#products - 1) * 4
      instructions per k-block: STEP * Lc * 2.1 u.
    * Epilogue: acc0 + acc1 + accc, + bias, + residual are four fp32 roundings, 4 * 2^-24 = STEP of the partial sums
      (the |A||W| part is here, the bias / residual / result parts are added by tapgemm_reference).
    """
    u = 1.01 * UNIT[dtype]
    dropped = {1: 0.0, 2: u ** 2, 3: 2 * u ** 3 + u ** 4}[nsplit]
    chain = 4 * ((n_iter + 1) // 2)
    corr = (nsplit * (nsplit + 1) // 2 - 1) * 4 * n_iter * 2.1 * u
    return dropped + STEP * (chain + corr + 1)


def _tap_sum(a_pad, w, rows_out):
    """sum_t a_pad[:, t : t + rows_out] @ w[t].T for a_pad (batch, rows_out + taps - 1, cin), w (taps, cout, cin)."""
    y = None
    for t in range(w.shape[0]):
        y_t = torch.matmul(a_pad[:, t:t + rows_out], w[t].t())
        y = y_t if y is None else y.add_(y_t)
    return y


def tapgemm_reference(a, w, bias, *, rows_in=None, rows_out, pad=0, act=0, act_cols=0, slope=0.0, residual=None,
                      a_view=None):
    """float64 reference and per-element error bound of ops.tapgemm_tc(a, w, bias, ...) built from the operands the
    kernel receives: the A planes read through the same (rows_in, cin, lda) view as the kernel's TMA map, rows past
    rows_in of each clip (and before row 0) are zero, W = plane sum of the PackedW times its acc_scale.
    Returns (want, bound) as float64 (batch, rows_out, cout)."""
    t = a.t
    nsplit, batch = t.shape[0], t.shape[1]
    rows_a, cin, lda = (a.rows, a.ch, t.stride(2)) if a_view is None else a_view
    if rows_in is not None:
        rows_a = rows_in
    bs = t.stride(1) if batch > 1 else rows_a * lda
    view = t.as_strided((nsplit, batch, rows_a, cin), (t.stride(0), bs, lda, 1), t.storage_offset())
    f16 = t.dtype == torch.float16
    w_scale = w.acc_scale * F16_ACT_SCALE if f16 else 1.0            # fp16 weight planes hold W * 2^k, acc_scale = 2^-k / 64
    taps, cout = w.taps, w.cout
    wp = w.t[:, :, :cout, :cin]
    a_eff = planes_f64(view)
    w_eff = planes_f64(wp, act=False) * w_scale
    span = rows_out + taps - 1

    def padded(x):
        out = torch.zeros(batch, span, cin, dtype=torch.float64, device=x.device)
        hi = min(span, rows_a + pad)
        if hi > pad:
            out[:, pad:hi] = x[:, :hi - pad]
        return out

    a_pad = padded(a_eff)
    want = _tap_sum(a_pad, w_eff, rows_out)
    a_abs, w_abs = a_pad.abs_(), w_eff.abs()
    a_fl = flushable_f64(view, 1.0 / F16_ACT_SCALE)
    w_fl = flushable_f64(wp, w_scale)
    c = tapgemm_c(nsplit, t.dtype, taps * -(-cin // 64))
    lhs = a_abs * c if a_fl is None else a_abs * c + padded(a_fl)
    bound = _tap_sum(lhs, w_abs, rows_out)
    if w_fl is not None:
        bound += _tap_sum(a_abs, w_fl, rows_out)
    extra = torch.zeros_like(want)
    if bias is not None:
        want += bias.double()
        extra += bias.double().abs()
    if residual is not None:
        want += residual.double()
        extra += residual.double().abs()
    if act:
        ncols = cout if act_cols <= 0 else act_cols
        s = 0.0 if act == 1 else float(slope)
        head = want[..., :ncols]
        want[..., :ncols] = torch.where(head < 0, head * s, head)
    extra += want.abs()
    bound += STEP * extra
    return want, bound


def bound_fraction(got, want, bound) -> float:
    """Largest |got - want| / bound over all elements (inf where the bound is 0 and the error is not)."""
    err = (got.double() - want).abs()
    frac = torch.where(bound > 0, err / bound.clamp_min(1e-300), torch.where(err > 0, math.inf, 0.0))
    return float(frac.max()) if frac.numel() else 0.0


def check_tapgemm(a, w, bias, got_f, got_p, tag="", **kw):
    """Every output element of one tapgemm_tc call against tapgemm_reference: the fp32 result within the bound, the
    emitted planes re-assembling the fp32 result (or, without it, the reference within bound + split error).
    Returns the largest fractions of the GEMM bound and of the plane-split bound used."""
    want, bound = tapgemm_reference(a, w, bias, **kw)
    batch, rows_out, cout = want.shape
    used = [0.0, 0.0]
    if got_f is not None:
        used[0] = bound_fraction(got_f, want, bound)
        assert used[0] <= 1.0, f"{tag}: fp32 output uses {used[0]:.3g} of its per-element bound"
    if got_p is not None:
        v = planes_f64(got_p.t[:, :, :rows_out, :cout])
        if got_f is not None:
            used[1] = bound_fraction(v, got_f.double(), plane_bound(got_p.nsplit, got_p.t.dtype, got_f.double()))
        else:
            used[0] = used[1] = bound_fraction(v, want, bound + plane_bound(got_p.nsplit, got_p.t.dtype, want.abs() + bound))
        assert used[1] <= 1.0, f"{tag}: plane output uses {used[1]:.3g} of its per-element bound"
    return tuple(used)


# ------------------------------------------------------------------------------------------------------------------
# attention (pm_attention_tc)
# ------------------------------------------------------------------------------------------------------------------


def attention_reference(q, q_col0, k, k_col0, v, v_col0, batch, heads, tq, tk, head_dim):
    """float64 softmax attention of the two-plane fp16 Q, K, V head slices the kernel reads, and a per-element bound
    (batch * tq, heads * head_dim) of the tensor-core kernel's error:

    * S = Q K^T: 3 products (drops p1 p1 <= (1.01 u)^2, u = 2^-11) over one accumulator chain of 3 * 12 instructions,
      so |dS| <= cs (|Q| @ |K|^T) / sqrt(hd), cs = 1.03 u^2 + 36 STEP.
    * P = exp(S - rowmax): ex2.approx (2 ulp) of an fp32 argument whose rounding costs 2^-24 |arg| ln 2, a 64-term fp32
      row sum: relative error e_i = 2^-21 + 2^-24 max_j(|t_ij| + |m_i|) + 64 * 2^-24 per probability, t in log2 units.
      A perturbation d of the scores moves softmax by p_ij (d_ij - sum_k p_ik d_ik), so the output moves by at most
      2 (max_j dS_ij + e_i) (P @ |V|)_i.
    * P as two fp16 planes of 1024 p: 2^-22 relative, and probabilities below 2^-24 (fp16 subnormal after the x1024)
      may be flushed: 2^-24 (1 @ |V|) absolute.
    * O = P V: 3 products and one chain of 12 instructions: (1.03 u^2 + 13 STEP) (P @ |V|), then two fp32 roundings of
      the normalisation, 2^-23 |O|.
    Returns (want, bound) as float64."""
    u = 1.01 * UNIT[torch.float16]
    E = heads * head_dim

    def heads_of(x, rows):                                                 # (batch, rows, E) -> (batch, heads, rows, hd)
        return x.reshape(batch, rows, heads, head_dim).transpose(1, 2)

    def operand(pl, col0, rows):
        sl = pl.t[:, :, :rows, col0:col0 + E]
        return heads_of(planes_f64(sl), rows), heads_of(flushable_f64(sl, 1.0 / F16_ACT_SCALE), rows)

    (Q, Qf), (K, Kf), (V, Vf) = operand(q, q_col0, tq), operand(k, k_col0, tk), operand(v, v_col0, tk)
    sc = 1.0 / math.sqrt(head_dim)
    s = Q @ K.transpose(-1, -2) * sc
    p = torch.softmax(s, -1)
    want = p @ V
    # flushed fp16 subnormal plane elements of Q / K / V count in full
    ds = ((1.03 * u ** 2 + 36 * STEP) * Q.abs() + Qf) @ K.abs().transpose(-1, -2) * sc + Q.abs() @ Kf.transpose(-1, -2) * sc
    t2 = s / math.log(2.0)
    m = t2.max(-1, keepdim=True).values
    e = 2.0 ** -21 + ULP32 * (t2.abs() + m.abs()).max(-1, keepdim=True).values + 64 * ULP32
    pv = p @ V.abs()
    bound = (2 * (ds.max(-1, keepdim=True).values + e) + 2.0 ** -22 + 1.03 * u ** 2 + 13 * STEP) * pv
    bound = bound + p @ Vf + ULP32 * V.abs().sum(-2, keepdim=True) + 2.0 ** -23 * want.abs()
    flat = lambda x: x.transpose(1, 2).reshape(batch * tq, E)
    return flat(want), flat(bound)


def check_attention(res, args, tag=""):
    """Every output element of one attention_tc call (res: fp32 tensor or ops.Act) against attention_reference.
    Returns the largest fractions of the attention bound and of the plane-split bound used."""
    want, bound = attention_reference(*args)
    f_t = res if isinstance(res, torch.Tensor) else res.f
    p_t = None if isinstance(res, torch.Tensor) else res.p
    used = [0.0, 0.0]
    if f_t is not None:
        used[0] = bound_fraction(f_t, want, bound)
        assert used[0] <= 1.0, f"{tag}: fp32 output uses {used[0]:.3g} of its per-element bound"
    if p_t is not None:
        batch, tq, E = p_t.batch, p_t.rows, p_t.ch
        v = planes_f64(p_t.t[:, :, :, :E]).reshape(batch * tq, E)
        if f_t is not None:
            used[1] = bound_fraction(v, f_t.double(), plane_bound(p_t.nsplit, p_t.t.dtype, f_t.double()))
        else:
            used[0] = used[1] = bound_fraction(v, want, bound + plane_bound(p_t.nsplit, p_t.t.dtype, want.abs() + bound))
        assert used[1] <= 1.0, f"{tag}: plane output uses {used[1]:.3g} of its per-element bound"
    return tuple(used)


# ------------------------------------------------------------------------------------------------------------------
# VQ lookup (pm_l2_argmin_*)
# ------------------------------------------------------------------------------------------------------------------


def fp64_margins(z, cb):
    """float64 argmin of |z - e_k|^2 (the M.py:64 expression) per row and the gap to the second best code."""
    d = (z.double() ** 2).sum(1, keepdim=True) + (cb.double() ** 2).sum(1) - 2 * z.double() @ cb.double().t()
    top = d.topk(2, dim=1, largest=False)
    return top.indices[:, 0], top.values[:, 1] - top.values[:, 0], d


def check_l2_argmin(got, z, cb, tag=""):
    """Indices of an L2-argmin call: always in [0, 256); equal to the float64 argmin wherever the float64 margin
    exceeds the fp32 noise of that row's distances, 2e-6 (|z|^2 + max |e_k|^2) (the rule of
    test_l2_argmin_tc_any_scale, per row); elsewhere a code whose float64 distance is within that noise of the
    minimum.  Returns (decided rows, rows)."""
    z = z.reshape(-1, cb.shape[1])
    got = got.reshape(-1)
    assert int(got.min()) >= 0 and int(got.max()) < cb.shape[0], f"{tag}: index out of range"
    finite = torch.isfinite(z).all(1)
    want, margin, d = fp64_margins(z.nan_to_num(0.0), cb)
    noise = 2e-6 * ((z.double() ** 2).sum(1).nan_to_num(0.0) + (cb.double() ** 2).sum(1).max())
    decided = (margin > noise) & finite
    assert torch.equal(got[decided], want[decided]), f"{tag}: {int((got[decided] != want[decided]).sum())} decided rows differ"
    gap = d.gather(1, got[:, None])[:, 0] - d.min(1).values
    assert bool((gap[finite] <= noise[finite]).all()), f"{tag}: an undecided row picked a code outside the near-ties"
    return int(decided.sum()), got.numel()

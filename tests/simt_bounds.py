"""float64 references with per-element error bounds for the CUDA-core (SIMT) fp32 kernels: the tap-GEMM
(pm_tapgemm_simt.cu), the WavEncoder stem, the residual LayerNorm (pm_elementwise.cu), attention (pm_attention.cu) and
the persistent BiLSTM (pm_lstm.cu).

Each function takes the operands the kernel actually received (fp32 tensors, on any device) and returns (want, bound)
as float64: |got - want| <= bound must hold for every output element.  Each bound counts the roundings the kernel does,
in its order, from the source named in the docstring.  The library is built without fast-math
(pantomatrix_b200/build.py: -O3 only), so expf, tanhf and rsqrtf are the libdevice functions with the error bounds of
the CUDA math guide (2 ulp each), sqrtf and '/' are correctly rounded, and the only liberty the compiler takes is
contracting a * b + c into one fma - which never adds a rounding, so every bound below allows both forms.

Notation: U = 2^-24 (unit roundoff of fp32); an fp32 op rounds x to x (1 + d), |d| <= U; 2 ulp of a result r is at most
2 * 2^-23 |r| = 4 U |r|.  gamma(n) = n U / (1 - n U) bounds the relative error of an n-step fp32 fma chain against the
sum of its |terms|.  Products of two first-order terms (U^2 and smaller) are covered by the final factor SECOND."""
import math

import torch

U = 2.0 ** -24
SECOND = 1.0 + 2.0 ** -20            # second-order terms: every bound is first order in U times at most 2^4 slack
ACT_NONE, ACT_RELU, ACT_LEAKY = 0, 1, 2


def gamma(n: int) -> float:
    return n * U / (1.0 - n * U)


def bound_fraction(got, want, bound) -> float:
    """Largest |got - want| / bound over all elements; inf where the bound is 0 and the error is not, or where got is
    not finite while want is."""
    err = (got.double() - want).abs()
    err = torch.where(torch.isnan(err), torch.full_like(err, math.inf), err)
    frac = torch.where(bound > 0, err / bound.clamp_min(1e-300), torch.where(err > 0, math.inf, 0.0))
    return float(frac.max()) if frac.numel() else 0.0


def within(got, want, bound) -> bool:
    """Every element of got within its own bound (NaN or inf where want is finite fails)."""
    return bound_fraction(got, want, bound) <= 1.0


# ------------------------------------------------------------------------------------------------------------------
# tap-GEMM (pm_tapgemm_f32) and the WavEncoder stem (pm_wav_stem_f32)
# ------------------------------------------------------------------------------------------------------------------


def _gathered(a, taps, stride, pad, rows_out):
    """(batch, rows_out, taps * cin) float64: A row l * stride + t - pad of tap t, zero outside [0, rows_in)."""
    batch, rows_in, cin = a.shape
    l = torch.arange(rows_out, device=a.device)[:, None] * stride + torch.arange(taps, device=a.device)[None] - pad
    ok = (l >= 0) & (l < rows_in)
    g = a.double()[:, l.clamp(0, max(rows_in - 1, 0))] if rows_in else a.new_zeros(batch, rows_out, taps, cin).double()
    return (g * ok[None, :, :, None]).reshape(batch, rows_out, taps * cin)


def _act_bound(pre, b_pre, act, slope):
    """Output and bound after pm_act (pm_common.cuh): v > 0 ? v : v * slope (ReLU: 0).  The negative side is exact for
    ReLU and one rounding of v * slope for LeakyReLU, so its bound is slope * b_pre plus that rounding; an element whose
    pre-activation interval [pre - b_pre, pre + b_pre] straddles 0 may land on either side, so it gets the larger of
    the two (pm_act is Lipschitz with constant max(1, slope) <= 1 here, so either side's error stays within it)."""
    if act == ACT_NONE:
        return pre, b_pre
    s = 0.0 if act == ACT_RELU else float(slope)
    want = torch.where(pre > 0, pre, pre * s)
    neg = s * b_pre + U * s * (pre.abs() + b_pre)
    side = torch.where(pre > 0, b_pre, neg)
    return want, torch.where(pre.abs() <= b_pre, torch.maximum(b_pre, neg), side)


def tapgemm_f32(a, w, bias=None, *, stride=1, pad=0, rows_out=None, act=ACT_NONE, slope=0.0, residual=None):
    """Reference and bound of ops.tapgemm(a, w, bias, ...) on the fp32 SIMT kernel (pm_tapgemm_simt.cu).

    a (batch, rows_in, cin), w (taps, cout, cin), bias (cout,) or None, residual (batch, rows_out, cout) or None.

    * Mainloop (`for t < taps`, `for c0 < cin step BK`, `for k < BK`): each output is ONE accumulator acc[i][j] updated
      by fmaf for every (tap, channel) pair in order, K_eff = taps * cin products.  The padding channels of the last
      16-wide K tile (c >= cin) and the padding rows (row < 0 or >= rows_in) are loaded as 0, and fmaf(0, w, acc) ==
      acc exactly, so they add no rounding.  A K_eff-step chain errs by at most gamma(K_eff) (|A| @ |W|).
    * Epilogue: v = acc + bias, v += residual: one rounding each, U |acc + bias| <= U (|A| @ |W| + |bias|) (first
      order) and U |v + residual| <= U (|pre| + |residual|) (without a residual only the first).
    * Together: |err_pre| <= (K_eff + 2) U (|A| @ |W| + |bias|) + U (|residual| + |pre|), the +2 holding the bias
      rounding and gamma's second-order part; then pm_act (_act_bound).
    Returns (want, bound) float64 (batch, rows_out, cout)."""
    taps, cout, cin = w.shape
    batch, rows_in, _ = a.shape
    if rows_out is None:
        rows_out = (rows_in + 2 * pad - taps) // stride + 1
    g = _gathered(a, taps, stride, pad, rows_out)
    wk = w.double().permute(0, 2, 1).reshape(taps * cin, cout)
    pre = g @ wk
    b_pre = g.abs_() @ wk.abs_()
    del g
    if bias is not None:
        pre += bias.double()
        b_pre += bias.double().abs()
    b_pre *= (taps * cin + 2) * U
    if residual is not None:
        pre += residual.double()
        b_pre += U * residual.double().abs()
    b_pre += U * pre.abs()
    want, bound = _act_bound(pre, b_pre, act, slope)
    return want, bound * SECOND


def wav_stem_f32(audio, a_bs, a_ws, batch, windows, n_samples, w1, b1, wd, bd, *, stride, pad, slope, offset=0):
    """Reference and bound of ops.wav_stem(...) with fp32 outputs (pm_wav_stem_f32, wav_stem_kernel in
    pm_elementwise.cu): (y1, sc), each (windows * batch, rows_out, cout), window-major.

    Sequence (b, w) is audio.flatten()[offset + b a_bs + w a_ws :][:n_samples]; the tile stages the samples of its span
    with zeros outside [0, n_samples) (`sx[i] = ... ? x[s] : 0`), so samples past n_samples never count even where the
    tensor has data.  Per output both the stride-5 path and the generic path run the 15-step fmaf chain k = 0 .. 14
    (`acc[j][c] = fmaf(v, w[k], acc[j][c])`), then add the bias (one rounding); y1 then goes through
    `a > 0 ? a : a * slope`.  That is the tap-GEMM bound of a 15-tap, 1-channel conv (tapgemm_f32: K_eff = 15, no
    residual): (15 + 2) U (|x| @ |w| + |b|) + U |pre|, LeakyReLU on y1 only."""
    flat = audio.reshape(-1)
    seqs = torch.stack([flat[offset + b * a_bs + w * a_ws: offset + b * a_bs + w * a_ws + n_samples]
                        for w in range(windows) for b in range(batch)]).unsqueeze(-1)
    t1, td = w1.t().unsqueeze(-1), wd.t().unsqueeze(-1)            # (taps, cout, cin = 1)
    y1 = tapgemm_f32(seqs, t1, b1, stride=stride, pad=pad, act=ACT_LEAKY, slope=slope)
    sc = tapgemm_f32(seqs, td, bd, stride=stride, pad=pad)
    return y1, sc


# ------------------------------------------------------------------------------------------------------------------
# LayerNorm (pm_add_layernorm_f32)
# ------------------------------------------------------------------------------------------------------------------


def add_layernorm_f32(x, r, gamma_, beta, eps=1e-5):
    """Reference and bound of ops.add_layernorm(x, r, gamma, beta, eps) (add_layernorm_kernel, pm_elementwise.cu):
    LayerNorm(x + r) over the last dim n = ch = 128 VEC, one warp per row, two-pass mean / variance.  The reference
    uses the fp32 value of eps (the kernel receives a float).

    * v_i = x_i + r_i: one rounding, U |w_i| with w = x + r exact (none without r).
    * Mean: a lane adds its VEC float4 chunks as s += (a + b) + (c + d) - an element passes at most VEC + 2 additions -
      then pm_warp_sum's 5 butterfly levels: depth VEC + 7, so |sum error| <= (VEC + 7) U sum |v|.  `* (1.f / CH)`:
      1/CH is exact for 256, 512, 1024 and one rounding for 768, the product one more.
      E_mu = (VEC + 7 + [r]) U mean|w| + (1 + [1/CH inexact]) U |mu|.
    * Deviation d_i = v_i - mean: E_d,i = [r] U |w_i| + E_mu + U (|dev_i| + E_mu) (the subtraction's rounding).
    * Variance: q += (a a + b b) + (c c + d d) - the squares (or the fma that contracts them), two additions, VEC
      accumulations, 5 butterfly levels: VEC + 8 roundings per term, then `* (1.f / CH)` as above and `+ eps` (one
      rounding, U (var + eps)).  The squares of the deviation errors enter as sum(2 |dev| E_d + E_d^2) / n.  With
      rho = E_V / (var + eps), rsqrtf (2 ulp: 4 U) gives rstd within rel_r = (1 - rho)^-1/2 - 1 + 4 U (1 - rho)^-1/2.
      This stays meaningful for rows whose mean is 10^3 their standard deviation (E_mu is a small part of the std) and
      for constant rows (var = 0, rstd = eps^-1/2: only E_d survives, the deviation the kernel sees is its mean error).
    * Output `(v - mean) * rstd * g + b`: |dev_hat rstd_hat - dev rstd| <= E_t = (E_d (1 + rel_r) + |dev| rel_r) rstd,
      then three roundings (the product, * g, + b; contraction only removes one): 2 U |g| (|dev| rstd + E_t) + U |want|.
    Returns (want, bound) float64 of x's shape."""
    n = x.shape[-1]
    vec = n // 128
    inv_inexact = 0 if (n & (n - 1)) == 0 else 1
    has_r = r is not None
    w = x.double() + (r.double() if has_r else 0.0)
    eps = float(torch.tensor(eps, dtype=torch.float32))
    mu = w.mean(-1, keepdim=True)
    dev = w - mu
    var = (dev * dev).mean(-1, keepdim=True)
    rw = U * w.abs() if has_r else torch.zeros_like(w)
    e_mu = (vec + 7 + int(has_r)) * U * w.abs().mean(-1, keepdim=True) + (1 + inv_inexact) * U * mu.abs()
    e_d = rw + e_mu + U * (dev.abs() + e_mu)
    c_v = (vec + 9 + inv_inexact) * U
    e_v = (2 * dev.abs() * e_d + e_d * e_d).mean(-1, keepdim=True) * (1 + c_v) + c_v * var + U * (var + eps)
    rho = e_v / (var + eps)
    ok = rho < 1
    s = torch.where(ok, (1 - rho).clamp_min(1e-300).rsqrt(), torch.full_like(rho, math.inf))
    rel_r = s - 1 + 4 * U * s
    rstd = (var + eps).rsqrt()
    g, b = gamma_.double(), beta.double()
    want = dev * rstd * g + b
    e_t = (e_d * (1 + rel_r) + dev.abs() * rel_r) * rstd
    bound = g.abs() * e_t + 2 * U * g.abs() * (dev.abs() * rstd + e_t) + U * want.abs()
    return want, bound * SECOND


# ------------------------------------------------------------------------------------------------------------------
# attention (pm_attention_f32)
# ------------------------------------------------------------------------------------------------------------------


def attention_f32(q, k, v, batch, heads, tq, tk, head_dim=192):
    """Reference and bound of ops.attention(q, k, v, ...) with fp32 output (attention_f32_kernel, pm_attention.cu).
    q (batch * tq, >= heads * hd), k, v (batch * tk, ...) are the views the kernel reads (head h = columns h hd ...).

    * Scores (`for d < HD`: acc = fmaf(q, k, acc)): a 192-step fma chain, gamma(192) (|q| @ |k|^T), times `scale` =
      1.0f / sqrtf(192.f) - sqrtf and '/' correctly rounded, so scale is within 2 U of 1/sqrt(192) - and the product
      rounds once more: |dS_ij| <= gamma(192) sc (|q| @ |k|^T)_ij + 3 U |s_ij|.
    * Softmax (warp per row): m = the row max of the computed scores (exact), e = expf(s - m): the subtraction rounds
      (U |t_ij|, t = s - m <= 0) and expf errs by 2 ulp (4 U); the row sum e0 + e1 then 5 butterfly levels is 6
      roundings of positive terms (6 U); inv = 1.f / sum and p = e * inv one rounding each.  So p_hat = p'(1 + eta),
      |eta| <= U (|t_ij| + 2 D_i + 12), where p' = softmax of the computed scores.  A score perturbation of at most
      D_i = max_j |dS_ij| moves p' from the exact p by a factor within exp(+-2 D_i): rel_p = expm1(2 D_i) +
      U (|t| + 2 D_i + 12) exp(2 D_i).  Probabilities whose expf result is subnormal (t < -87) are bounded
      absolutely: 2^-126 per key.
    * Output (`for j < tk`: acc = fmaf(p, v, acc)): a tk-step fma chain over the computed probabilities:
      |err_ic| <= sum_j p_ij |v_jc| (rel_p_ij (1 + gamma(tk)) + gamma(tk)) + 2^-126 sum_j |v_jc|; the tile is then
      copied out unchanged.
    Returns (want, bound) float64 (batch * tq, heads * hd)."""
    hd = head_dim
    E = heads * hd

    def heads_of(x, rows):
        return x[:, :E].double().reshape(batch, rows, heads, hd).transpose(1, 2)

    Q, K, V = heads_of(q, tq), heads_of(k, tk), heads_of(v, tk)
    sc = 1.0 / math.sqrt(hd)
    s = Q @ K.transpose(-1, -2) * sc
    ds = gamma(hd) * sc * (Q.abs() @ K.abs().transpose(-1, -2)) + 3 * U * s.abs()
    d = ds.amax(-1, keepdim=True)
    p = torch.softmax(s, -1)
    t = s - s.amax(-1, keepdim=True)
    rel_p = torch.expm1(2 * d) + U * (t.abs() + 2 * d + 12) * torch.exp(2 * d)
    gt = gamma(tk)
    want = p @ V
    bound = (p * (rel_p * (1 + gt) + gt)) @ V.abs() + 2.0 ** -126 * V.abs().sum(-2, keepdim=True)
    flat = lambda x: x.transpose(1, 2).reshape(batch * tq, E)
    return flat(want), flat(bound * SECOND)


# ------------------------------------------------------------------------------------------------------------------
# BiLSTM (pm_lstm_bidir_f32): teacher-forced, one step at a time
# ------------------------------------------------------------------------------------------------------------------

LSTM_DOT_STEPS = 64 + 3 + 1          # K-slice fma chain + shuffle tree + the input projection add (lstm_bidir_kernel)


def _sig_err(z, e):
    """|sigmoidf_(z_hat) - sigmoid(z)| for |z_hat - z| <= e: sigma' (z + delta) <= exp|delta| sigma'(z) moves it by at
    most e sigma'(z) exp(e); sigmoidf_ = 1.f / (1.f + expf(-z)) adds expf's 4 U (relative to e^-z, so at most 4 U of
    the sum 1 + e^-z), the addition's U and the division's U: 6 U sigma."""
    sg = torch.sigmoid(z)
    return sg, e * sg * (1 - sg) * torch.exp(e) + 6 * U * sg


def _tanh_err(z, e):
    """|tanhf(z_hat) - tanh(z)| for |z_hat - z| <= e: tanh'(z + delta) <= exp(2 |delta|) tanh'(z); tanhf errs by
    2 ulp (4 U)."""
    th = torch.tanh(z)
    return th, e * (1 - th * th) * torch.exp(2 * e) + 4 * U * th.abs()


def lstm_bidir_f32(xproj, whh, y, hidden=512):
    """Teacher-forced reference and bound of one pm_lstm_bidir_f32 call (lstm_bidir_kernel, pm_lstm.cu).
    xproj (B, T, >= 8H) and y (B, T, >= 2H) are the kernel's input and OUTPUT views, whh (2, 4H, H).

    The recurrence amplifies errors through W_hh, so whole-sequence comparison can only use a loose global tolerance.
    Instead every step is checked on its own: the gate pre-activations of step t are formed in float64 from the
    kernel's own h_{t-1} (read from y), so each h_t element is held to the error of ONE step.

    * Pre-activations: K-slice kq of a lane accumulates its 64 columns of h_{t-1} . W_hh (`for j < H / 32` x float4: a
      64-step fmaf chain), the 8 K-slices are combined by the xor-4/2/1 shuffle tree (3 additions) and added to the
      input projection (`pre[r] = x[r] + ...`, 1 rounding): |E_pre| <= (64 + 3 + 1) U (|h_{t-1}| @ |W_hh|^T) + U |pre|
      (first step: pre = x exactly, and h_{t-1} = 0 gives the same formula).
    * Gates: sigmoidf_ / tanhf of the pre-activations: _sig_err, _tanh_err.
    * Cell state (registers, never written): c_t = f c_{t-1} + i g is carried in float64 from the float64 gates, and
      its bound alongside: E_c,t = (f + E_f) E_c,t-1 + E_f |c_{t-1}| + E_i (|g| + E_g) + i E_g + U (f |c_{t-1}| +
      i |g|) + U |c_t| (the two products and the sum: at most two roundings whether or not one is an fma).  The
      recurrence contracts as long as f + E_f < 1.
    * h_t = sigmoidf_(o) * tanhf(c_t): E_h = E_o (|tanh c| + E_tc) + o E_tc + U |h|, E_tc from _tanh_err(c, E_c).
    Returns (want, bound) float64 (B, T, 2H): float64 h_t from the kernel's h_{t-1}, and its bound."""
    H = hidden
    B, T = y.shape[0], y.shape[1]
    want = torch.empty(B, T, 2 * H, dtype=torch.float64, device=y.device)
    bound = torch.empty_like(want)
    for d in range(2):
        x = xproj[:, :, d * 4 * H:(d + 1) * 4 * H].double()
        h = y[:, :, d * H:(d + 1) * H].double()
        hp = torch.zeros_like(h)
        if T > 1:
            if d == 0:
                hp[:, 1:] = h[:, :-1]
            else:
                hp[:, :-1] = h[:, 1:]
        W = whh[d].double()
        pre = x + hp @ W.t()
        e_pre = LSTM_DOT_STEPS * U * (hp.abs() @ W.abs().t()) + U * pre.abs()
        del hp, x
        (pi, pf, pg, po), (ei, ef, eg, eo) = pre.split(H, -1), e_pre.split(H, -1)
        si, e_si = _sig_err(pi, ei)
        sf, e_sf = _sig_err(pf, ef)
        tg, e_tg = _tanh_err(pg, eg)
        so, e_so = _sig_err(po, eo)
        c = torch.zeros(B, H, dtype=torch.float64, device=y.device)
        ec = torch.zeros_like(c)
        cs, ecs = torch.empty_like(si), torch.empty_like(si)
        for s in range(T):
            t = s if d == 0 else T - 1 - s
            f, i, g = sf[:, t], si[:, t], tg[:, t]
            cn = f * c + i * g
            ec = ((f + e_sf[:, t]) * ec + e_sf[:, t] * c.abs() + e_si[:, t] * (g.abs() + e_tg[:, t]) + i * e_tg[:, t]
                  + U * (f * c.abs() + i * g.abs()) + U * cn.abs()) * SECOND
            c = cn
            cs[:, t], ecs[:, t] = c, ec
        tc, e_tc = _tanh_err(cs, ecs)
        hw = so * tc
        want[:, :, d * H:(d + 1) * H] = hw
        bound[:, :, d * H:(d + 1) * H] = (e_so * (tc.abs() + e_tc) + so * e_tc + U * hw.abs()) * SECOND
    return want, bound

"""Per-kernel parity tests (GPU): every C-ABI entry point against a plain torch restatement of the same op
in float64 (or exact equality for integer / copy semantics).  All calls go through pantomatrix_b200.ops,
i.e. through libpm_emage.so."""
import math

import pytest
import torch
import torch.nn.functional as F

from helpers import bf16_planes_by_default, check_attention, check_l2_argmin, fp64_margins  # noqa: F401

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ops():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    from pantomatrix_b200 import _lib, ops as o
    _lib.load()
    assert _lib.load().pm_device_cc() == 90, "sm_90a kernels need a Hopper (H100) device"
    return o


def _rand(*shape, seed=0, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(*shape, generator=g) * scale).cuda()


def _close(got, want, rtol=2e-5, atol=2e-5):
    want = want.to(torch.float64)
    err = (got.double() - want).abs()
    tol = atol + rtol * want.abs()
    assert bool((err <= tol).all()), f"max err {err.max().item():.3e} (tol {tol.max().item():.3e})"


CONV_CASES = [
    # batch, rows_in, cin, cout, k, stride, pad, act, residual
    (3, 700, 64, 64, 15, 1, 7, "leaky", True),       # BasicBlock conv2 + shortcut
    (3, 745, 64, 64, 15, 6, 0, "leaky", False),      # strided conv1
    (2, 205, 128, 256, 15, 3, 0, "none", False),     # downsample branch
    (4, 64, 337, 256, 3, 1, 1, "leaky", False),      # motion encoder stem (ragged cin)
    (4, 11, 256, 61, 3, 1, 1, "none", True),         # ragged cout / short window + ResBlock skip
    (5, 16, 61, 61, 3, 1, 1, "none", False),
]


@pytest.mark.parametrize("case", CONV_CASES)
def test_tapgemm_conv(ops, case):
    b, rows, cin, cout, k, stride, pad, act, use_res = case
    x = _rand(b, rows, cin, seed=1)
    w = _rand(cout, cin, k, seed=2, scale=1 / math.sqrt(cin * k))
    bias = _rand(cout, seed=3, scale=0.1)
    want = F.conv1d(x.double().transpose(1, 2), w.double(), bias.double(), stride=stride, padding=pad).transpose(1, 2)
    res = _rand(*want.shape, seed=4) if use_res else None
    if use_res:
        want = want + res.double()
    if act == "leaky":
        want = F.leaky_relu(want, 0.2)
    got = ops.tapgemm(x, w.permute(2, 0, 1).contiguous(), bias, stride=stride, pad=pad,
                      act=ops.ACT_LEAKY if act == "leaky" else ops.ACT_NONE, slope=0.2, residual=res)
    assert got.shape == want.shape
    _close(got, want)


@pytest.mark.parametrize("m,k,n,act", [(2048, 768, 2304, "none"), (1920, 768, 1536, "relu"), (2048, 1536, 768, "none"),
                                       (37, 256, 768, "leaky"), (2048, 512, 768, "none")])
def test_tapgemm_linear(ops, m, k, n, act):
    x = _rand(32, m // 32 if m % 32 == 0 else 1, k, seed=5) if m % 32 == 0 else _rand(1, m, k, seed=5)
    w = _rand(n, k, seed=6, scale=1 / math.sqrt(k))
    bias = _rand(n, seed=7, scale=0.1)
    res = _rand(*x.shape[:2], n, seed=8)
    want = F.linear(x.double(), w.double(), bias.double()) + res.double()
    want = {"none": want, "relu": F.relu(want), "leaky": F.leaky_relu(want, 0.1)}[act]
    got = ops.tapgemm(x, w.unsqueeze(0), bias, residual=res, slope=0.1,
                      act={"none": ops.ACT_NONE, "relu": ops.ACT_RELU, "leaky": ops.ACT_LEAKY}[act])
    _close(got, want)


def test_tapgemm_strided_views(ops):
    """Column-slice input (packed qkv) and column-slice output, as the attention / concat call sites use."""
    x = _rand(4, 64, 2304, seed=9)
    w = _rand(256, 768, seed=10, scale=0.03)
    out = torch.zeros(4, 64, 512, device="cuda")
    ops.tapgemm(x[:, :, 768:1536], w.unsqueeze(0), None, out=out[:, :, 256:])
    _close(out[:, :, 256:], F.linear(x[:, :, 768:1536].double(), w.double()))
    assert out[:, :, :256].abs().max() == 0


def test_wav_stem(ops):
    bs, n, windows, ws, ns_ = 3, 9000, 2, 3000, 5863
    audio = _rand(bs, n, seed=11, scale=0.1)
    w1, wd = _rand(64, 15, seed=12, scale=0.5), _rand(64, 15, seed=13, scale=0.5)
    b1, bd = _rand(64, seed=14, scale=0.1), _rand(64, seed=15, scale=0.1)
    y1, sc = ops.wav_stem(audio, n, ws, bs, windows, ns_, w1, b1, wd, bd, stride=5, pad=1600, slope=0.01, offset=100)
    for w in range(windows):
        sl = audio[:, 100 + w * ws: 100 + w * ws + ns_].double().unsqueeze(1)
        c1 = F.conv1d(sl, w1.double().unsqueeze(1), b1.double(), stride=5, padding=1600).transpose(1, 2)
        cd = F.conv1d(sl, wd.double().unsqueeze(1), bd.double(), stride=5, padding=1600).transpose(1, 2)
        _close(y1[w * bs:(w + 1) * bs], F.leaky_relu(c1, 0.01))          # window-major layout
        _close(sc[w * bs:(w + 1) * bs], cd)
    # the tensor-core engines take conv1's output as operand planes straight from the stem: same values, split in-kernel
    for ns, fmt in ((2, "fp16"), (3, "bf16"), (2, "bf16")):
        old = ops.plane_format()
        ops.set_plane_format(fmt)
        try:
            pl, sc2 = ops.wav_stem(audio, n, ws, bs, windows, ns_, w1, b1, wd, bd, stride=5, pad=1600, slope=0.01, offset=100, nsplit=ns)
            ref = ops.split_bf16(y1, ns)
            assert torch.equal(pl.t[..., :64], ref.t[..., :64]) and torch.equal(sc2, sc)
        finally:
            ops.set_plane_format(old)
    # CaMN / DisCo stem width, stride != 5 through the generic path
    w1s, wds, b1s, bds = w1[:32].contiguous(), wd[:32].contiguous(), b1[:32].contiguous(), bd[:32].contiguous()
    for stride, pad in ((5, 1600), (4, 3)):
        y, s_ = ops.wav_stem(audio, n, ws, bs, windows, ns_, w1s, b1s, wds, bds, stride=stride, pad=pad, slope=0.01)
        sl = torch.cat([audio[:, w * ws: w * ws + ns_] for w in range(windows)]).double().unsqueeze(1)
        _close(y, F.leaky_relu(F.conv1d(sl, w1s.double().unsqueeze(1), b1s.double(), stride=stride, padding=pad), 0.01).transpose(1, 2))
        _close(s_, F.conv1d(sl, wds.double().unsqueeze(1), bds.double(), stride=stride, padding=pad).transpose(1, 2))


@pytest.mark.parametrize("ch", [256, 768])
def test_add_layernorm(ops, ch):
    x, r = _rand(301, ch, seed=16, scale=3.0), _rand(301, ch, seed=17)
    g, b = _rand(ch, seed=18), _rand(ch, seed=19)
    _close(ops.add_layernorm(x, r, g, b), F.layer_norm((x + r).double(), (ch,), g.double(), b.double(), 1e-5), 1e-5, 1e-5)
    _close(ops.add_layernorm(x, None, g, b), F.layer_norm(x.double(), (ch,), g.double(), b.double(), 1e-5), 1e-5, 1e-5)


@pytest.mark.parametrize("bs,tq,tk", [(5, 64, 64), (3, 60, 60), (2, 11, 12), (2, 1, 1)])
def test_attention(ops, bs, tq, tk):
    E, H, hd = 768, 4, 192
    qkv = _rand(bs * tq, 3 * E, seed=20)
    kv = _rand(bs * tk, 2 * E, seed=21)
    got = ops.attention(qkv[:, :E], kv[:, :E], kv[:, E:], bs, H, tq, tk, hd)
    q = qkv[:, :E].double().view(bs, tq, H, hd).transpose(1, 2)
    k = kv[:, :E].double().view(bs, tk, H, hd).transpose(1, 2)
    v = kv[:, E:].double().view(bs, tk, H, hd).transpose(1, 2)
    want = (torch.softmax(q @ k.transpose(-1, -2) / math.sqrt(hd), -1) @ v).transpose(1, 2).reshape(bs * tq, E)
    _close(got, want, 1e-5, 1e-5)


@pytest.mark.parametrize("bs,tq,tk", [(5, 64, 64), (3, 60, 60), (2, 11, 12), (2, 64, 60), (2, 1, 1), (32, 64, 64),
                                      (3, 64, 11), (3, 11, 64), (1, 64, 64)])
def test_attention_tc_against_float64(ops, bs, tq, tk):
    """Tensor-core attention of the fp16x3 engine: two-plane fp16 operands read in place from the packed q|k|v (self) or
    q + k|v (cross) projection outputs, here at column offsets inside wider planes with columns to spare after the
    last head; fp32, two-plane and one-plane outputs against float64, every element within its own bound
    (helpers.attention_reference), and the one-plane output the round-to-nearest-even split of the fp32 output."""
    E, H, hd = 768, 4, 192
    q0, k0 = 8, 24                                       # first column of Q inside q|k|v, of K inside k|v
    qkv = _rand(bs, tq, q0 + 3 * E + 40, seed=20)
    kv = _rand(bs, tk, k0 + 2 * E + 40, seed=21)
    ops.set_plane_format("fp16")
    qp, kvp = ops.split_bf16(qkv, 2), ops.split_bf16(kv, 2)
    cross_args = (qp, q0, kvp, k0, kvp, k0 + E, bs, H, tq, tk, hd)
    cross = ops.attention_tc(*cross_args, nsplit=2, f32=True)
    one = ops.attention_tc(*cross_args, nsplit=1, f32=False)
    if tq == tk:
        self_args = (qp, q0, qp, q0 + E, qp, q0 + 2 * E, bs, H, tq, tq, hd)
        self_att = ops.attention_tc(*self_args, nsplit=0)

    def ref(q, k, v):
        q, k, v = (x.double().reshape(bs, -1, H, hd).transpose(1, 2) for x in (q, k, v))
        return (torch.softmax(q @ k.transpose(-1, -2) / math.sqrt(hd), -1) @ v).transpose(1, 2).reshape(bs * tq, E)
    want = ref(qkv[..., q0:q0 + E], kv[..., k0:k0 + E], kv[..., k0 + E:k0 + 2 * E])
    _close(cross.f, want, 1e-5, 1e-5)
    used = [check_attention(cross, cross_args, tag="cross")]
    assert one.f is None and one.p.nsplit == 1
    used.append(check_attention(one, cross_args, tag="one plane"))
    # one plane is 64 x rounded to nearest even (the split rule, tests/plane_split.py), not the two-plane head
    one_bits = one.p.t[0, ..., :E].reshape(bs * tq, E).view(torch.int16)
    assert torch.equal(one_bits, (cross.f * ops.F16_ACT_SCALE).half().view(torch.int16))
    if tq == tk:
        _close(self_att, ref(qkv[..., q0:q0 + E], qkv[..., q0 + E:q0 + 2 * E], qkv[..., q0 + 2 * E:q0 + 3 * E]), 1e-5, 1e-5)
        used.append(check_attention(self_att, self_args, tag="self"))
    print(f"[attention_tc {bs}x{tq}x{tk}] largest fraction of the per-element bound used: attention "
          f"{max(u[0] for u in used):.3f}, plane split {max(u[1] for u in used):.3f}")


def test_attention_tc_peaked_rows_and_independence(ops):
    """Peaked softmax rows (scores up to ~40 after scaling, most probabilities far below 2^-24: ex2.approx.ftz and the
    fp16 planes of 1024 p), and clips / heads computed alone are bit-identical to the batched call."""
    E, H, hd, bs, t = 768, 4, 192, 6, 64
    qkv = _rand(bs, t, 3 * E, seed=75, scale=3.2)       # s = q.k / sqrt(192) ~ N(0, 10^2)
    ops.set_plane_format("fp16")
    qp = ops.split_bf16(qkv, 2)
    args = (qp, 0, qp, E, qp, 2 * E, bs, H, t, t, hd)
    got = ops.attention_tc(*args, nsplit=2, f32=True)
    clips = [ops.attention_tc(ops.split_bf16(qkv[b:b + 1], 2), 0, ops.split_bf16(qkv[b:b + 1], 2), E,
                              ops.split_bf16(qkv[b:b + 1], 2), 2 * E, 1, H, t, t, hd, nsplit=0) for b in (0, 3, 5)]
    heads = [ops.attention_tc(qp, h * hd, qp, E + h * hd, qp, 2 * E + h * hd, bs, 1, t, t, hd, nsplit=0) for h in range(H)]
    q = qkv[..., :E].double().reshape(bs, t, H, hd).transpose(1, 2)
    k = qkv[..., E:2 * E].double().reshape(bs, t, H, hd).transpose(1, 2)
    s = q @ k.transpose(-1, -2) / math.sqrt(hd)
    assert s.abs().max() > 35 and (torch.softmax(s, -1) < 2.0 ** -24).double().mean() > 0.3     # the case is peaked
    used = check_attention(got, args, tag="peaked")
    print(f"[attention_tc peaked] largest fraction of the per-element bound used: attention {used[0]:.3f}, "
          f"plane split {used[1]:.3f}")
    for b, c in zip((0, 3, 5), clips):
        assert torch.equal(c, got.f[b * t:(b + 1) * t]), b
    for h, o in enumerate(heads):
        assert torch.equal(o, got.f[:, h * hd:(h + 1) * hd]), h


def test_broadcast_adds_are_exact(ops):
    bs, t, ch = 3, 60, 768
    x, pe, spk = _rand(bs, t, ch, seed=22), _rand(128, ch, seed=23), _rand(bs, ch, seed=24)
    got = ops.add_rows(x, pe, spk, ops.ROW_SPK, ops.ROW_PE, bs, t, ch)
    assert torch.equal(got, (x + spk[:, None]) + pe[None, :t])
    got = ops.add_rows(None, pe, spk, ops.ROW_SPK, ops.ROW_PE, bs, t, ch)
    assert torch.equal(got, (spk[:, None] + pe[None, :t]).expand(bs, t, ch))
    got = ops.add_rows(x, pe, spk, ops.ROW_PE, ops.ROW_SPK, bs, t, ch)
    assert torch.equal(got, (x + pe[None, :t]) + spk[:, None])
    a, b = _rand(7, 13, 5, seed=25), _rand(7, 13, 5, seed=26)
    assert torch.equal(ops.add2(a, b), a + b)


def test_window_input_matches_reference_semantics(ops):
    bs, L, ch, pre, s, t = 3, 130, 337, 4, 60, 64
    motion, seed, emb = _rand(bs, L, ch, seed=27), _rand(bs, pre, ch, seed=28), _rand(ch, seed=29)
    mask = (torch.rand(bs, L, ch, generator=torch.Generator().manual_seed(30)) > 0.5).float().cuda()
    got = ops.window_input(motion, mask, seed, emb, s, t, pre)
    wm, wk = motion[:, s:s + t].clone(), mask[:, s:s + t].clone()          # M.py:384-391
    wm[:, :pre] = torch.where(wk[:, :pre] == 0, motion[:, s:s + pre], seed)
    wk[:, :pre] = 0
    want = torch.where(wk == 1, emb.view(1, 1, ch).expand_as(wm), wm)      # M.py:267-268
    assert torch.equal(got, want)


def _fp64_margins(z, cb):
    return fp64_margins(z, cb)[:2]


ENGINES = ["tc", "simt"]          # tensor-core screen + exact fp32 re-scoring (the product path) | fp32 SIMT kernel


@pytest.mark.parametrize("engine", ENGINES)
@pytest.mark.parametrize("rows", [1, 63, 9600, 128 * 148 * 2 + 77])
def test_l2_argmin_bit_exact(ops, rows, engine):
    z, cb = _rand(rows, 256, seed=31), _rand(256, 256, seed=32)
    got = ops.l2_argmin(z, cb, ops.row_sqnorm(cb), engine=engine)
    want, margin = _fp64_margins(z, cb)
    decided = margin > 1e-3          # fp32 evaluation of d (|d| ~ 500) cannot order closer pairs reliably
    assert decided.float().mean() > 0.99
    assert torch.equal(got[decided], want[decided])
    # the undecided rows must still pick one of the two near-tied codes
    d32 = (z ** 2).sum(1, keepdim=True) + (cb ** 2).sum(1) - 2 * z @ cb.t()
    assert bool(((d32.gather(1, got[:, None])[:, 0] - d32.min(1).values).abs() < 1e-2).all())
    if rows == 9600:                 # the dispatcher the product calls picks the tensor-core kernel for 256 codes
        assert torch.equal(ops.l2_argmin(z, cb, ops.row_sqnorm(cb)), ops.l2_argmin(z, cb, ops.row_sqnorm(cb), engine="tc"))


@pytest.mark.parametrize("engine", ENGINES)
def test_l2_argmin_ties_pick_first(ops, engine):
    cb = _rand(256, 256, seed=33)
    cb[200] = cb[7]                                   # duplicate code: lower index must win (torch.argmin)
    z = cb[[7, 200, 9]].clone() + 1e-3
    got = ops.l2_argmin(z, cb, ops.row_sqnorm(cb), engine=engine)
    assert got.tolist() == [7, 7, 9]


@pytest.mark.parametrize("zs,cs", [(1e-6, 1e-6), (3e4, 3e4), (1.0, 2e3), (1e-3, 1e-4), (300.0, 1.0)])
def test_l2_argmin_tc_any_scale(ops, zs, cs):
    """The fp16 screen scales rows and codebook by exact powers of two: results do not depend on the data's scale
    (3e4 * N(0,1) overflows fp16 unscaled, 1e-6 would vanish in its subnormals).  Latent and codebook scales stay
    within ~10^3 of each other: beyond that |z|^2 swamps the fp32 distance itself (reference formula M.py:64)."""
    z, cb = _rand(4099, 256, seed=43, scale=zs), _rand(256, 256, seed=44, scale=cs)
    got = ops.l2_argmin(z, cb, ops.row_sqnorm(cb), engine="tc")
    want, margin = _fp64_margins(z, cb)
    dscale = float((z.double() ** 2).sum(1).mean() + (cb.double() ** 2).sum(1).mean())
    decided = margin > 2e-6 * dscale
    assert decided.float().mean() > 0.97
    assert torch.equal(got[decided], want[decided])


def test_l2_argmin_tc_near_ties_are_rescored_exactly(ops):
    """Rows placed (almost) on the bisector of two codes: the fp16 screen cannot order them, the fp32 re-scoring must.
    The tensor-core kernel has to agree with the fp32 SIMT kernel wherever fp32 itself can decide."""
    cb = _rand(256, 256, seed=45)
    g = torch.Generator().manual_seed(46)
    a, b = torch.randint(0, 256, (2, 20000), generator=g)
    eps = (torch.rand(20000, generator=g) - 0.5).cuda() * 2e-5          # offset from the bisector: d_a - d_b ~ +-0.01
    z = 0.5 * (cb[a.cuda()] + cb[b.cuda()]) + eps[:, None] * (cb[a.cuda()] - cb[b.cuda()])
    e2 = ops.row_sqnorm(cb)
    tc, simt = ops.l2_argmin(z, cb, e2, engine="tc"), ops.l2_argmin(z, cb, e2, engine="simt")
    want, margin = _fp64_margins(z, cb)
    decided = margin > 2e-3
    assert 0.5 < decided.float().mean() < 0.999                           # the case really is near-tied
    assert torch.equal(tc[decided], want[decided]) and torch.equal(simt[decided], want[decided])
    d64 = (z.double() ** 2).sum(1, keepdim=True) + (cb.double() ** 2).sum(1) - 2 * z.double() @ cb.double().t()
    assert bool((d64.gather(1, tc[:, None])[:, 0] - d64.min(1).values < 2e-3).all())


@pytest.mark.parametrize("engine", ENGINES)
def test_l2_argmin_nan_and_clustered_rows(ops, engine):
    """A NaN latent yields index 0 (what torch.argmin returns for an all-NaN row), never an out-of-range index
    (ADVICE r1); a codebook of near-duplicates makes every code a candidate (the re-score-everything path)."""
    cb = _rand(256, 256, seed=47)
    z = _rand(300, 256, seed=48)
    z[5, 17] = float("nan")
    z[131] = float("nan")
    z[200] = 0.0
    got = ops.l2_argmin(z, cb, ops.row_sqnorm(cb), engine=engine)
    assert got[5].item() == 0 and got[131].item() == 0
    assert int(got.min()) >= 0 and int(got.max()) < 256
    want, margin = _fp64_margins(z.nan_to_num(0.0), cb)
    ok = (margin > 1e-3) & ~torch.isnan(z).any(1)
    assert torch.equal(got[ok], want[ok])
    base = _rand(1, 256, seed=49)
    cbc = (base + 1e-3 * _rand(256, 256, seed=50)).contiguous()           # 256 codes within 1e-3 of each other
    zc = (base + 1e-3 * _rand(500, 256, seed=51)).contiguous()
    gotc = ops.l2_argmin(zc, cbc, ops.row_sqnorm(cbc), engine=engine)
    d64 = ((zc.double()[:, None, :] - cbc.double()[None]) ** 2).sum(-1)
    assert bool((d64.gather(1, gotc[:, None])[:, 0] - d64.min(1).values < 5e-4).all())      # fp32 noise of d ~ 512 * 2^-23


def test_l2_argmin_million_rows_optimality(ops):
    """BASELINE-scale property check: chosen code is a minimiser (within fp32 noise) for 2^20 rows."""
    rows = 1 << 20
    z = torch.randn(rows, 256, device="cuda", generator=torch.Generator(device="cuda").manual_seed(34))
    cb = _rand(256, 256, seed=35)
    got = ops.l2_argmin(z, cb, ops.row_sqnorm(cb))
    assert int(got.min()) >= 0 and int(got.max()) < 256
    for lo in range(0, rows, 1 << 18):
        zz = z[lo:lo + (1 << 18)]
        d = (zz ** 2).sum(1, keepdim=True) + (cb ** 2).sum(1) - 2 * zz @ cb.t()
        picked = d.gather(1, got[lo:lo + (1 << 18), None])[:, 0]
        assert bool((picked - d.min(1).values < 5e-3).all())


@pytest.mark.parametrize("max_ctas", [1, 2, 3, 5])
def test_l2_argmin_tc_persistent_ctas(ops, max_ctas):
    """~40 tiles on 1-5 persistent CTAs: every CTA runs many tiles, so the A-tile handshake, the alternating INFO slots
    and the barrier phases all turn over.  Bit-identical to one tile per CTA, and to the fp32 SIMT kernel wherever fp32
    decides."""
    z, cb = _rand(40 * 128 - 3, 256, seed=76), _rand(256, 256, seed=77)
    e2 = ops.row_sqnorm(cb)
    got = ops.l2_argmin(z, cb, e2, engine="tc", max_ctas=max_ctas)
    assert torch.equal(got, ops.l2_argmin(z, cb, e2, engine="tc"))
    decided, rows = check_l2_argmin(got, z, cb, tag=f"max_ctas={max_ctas}")
    want, margin, _ = fp64_margins(z, cb)
    ok = margin > 1e-3
    assert torch.equal(got[ok], ops.l2_argmin(z, cb, e2, engine="simt")[ok])
    print(f"[l2_argmin max_ctas={max_ctas}] rows decided by float64 {decided}/{rows}")


@pytest.mark.parametrize("clips", [40, 1000])
def test_l2_argmin_tc_strided_tails(ops, clips):
    """The last 13 frames of 300-frame clips read in place (clip stride 300 * 256): 520 rows (5 tiles) and 13 000 rows
    (102 tiles), also with the tiles spread over 3 persistent CTAs."""
    x, cb = _rand(clips, 300, 256, seed=78), _rand(256, 256, seed=79)
    e2 = ops.row_sqnorm(cb)
    tail = x[:, 300 - 13:]
    dense = ops.l2_argmin(tail.contiguous(), cb, e2, engine="tc")
    for mc in (0, 3):
        assert torch.equal(ops.l2_argmin(tail, cb, e2, engine="tc", max_ctas=mc), dense), mc
    check_l2_argmin(dense, tail, cb, tag=f"{clips} strided tails")


@pytest.mark.parametrize("rem", [1, 7, 8, 9, 127])
def test_l2_argmin_tc_partial_last_tile(ops, rem):
    """rows % 128 in {1, 7, 8, 9, 127}: the loaders' last batch of 8 rows is partial; on 2 CTAs the partial tile is a
    CTA's later tile.  A row permutation permutes the indices exactly."""
    rows = 5 * 128 + rem
    z, cb = _rand(rows, 256, seed=80 + rem), _rand(256, 256, seed=81)
    e2 = ops.row_sqnorm(cb)
    got = ops.l2_argmin(z, cb, e2, engine="tc")
    assert torch.equal(ops.l2_argmin(z, cb, e2, engine="tc", max_ctas=2), got)
    check_l2_argmin(got, z, cb, tag=f"rows % 128 = {rem}")
    perm = torch.randperm(rows, generator=torch.Generator().manual_seed(rem)).cuda()
    assert torch.equal(ops.l2_argmin(z[perm].contiguous(), cb, e2, engine="tc", max_ctas=3), got[perm])


def test_window_input_defaults_and_strided_seed(ops):
    """motion / mask = None generate inference()'s defaults in the kernel (identity rot6d + zero trans/contact, all
    masked); the seed is read in place from the tail of a longer decode (clip stride != pre * ch); no seed at all
    (first window) keeps motion[:, :pre]."""
    bs, total, ch, pre = 3, 130, 337, 4
    emb = _rand(ch, seed=70)
    motion = torch.zeros(bs, total, ch, device="cuda")
    motion[:, :, 0:ch - 7:6] = 1.0
    motion[:, :, 4:ch - 7:6] = 1.0
    mask = torch.ones_like(motion)
    dec = _rand(bs, 13, ch, seed=71)                                     # a 13-frame seed decode; its last 4 frames are the seed
    seed = dec[:, 13 - pre:]
    want = ops.window_input(motion, mask, seed.contiguous(), emb, 60, 64, pre)
    got = ops.window_input(None, None, seed, emb, 60, 64, pre, shape=(bs, total, ch))
    assert torch.equal(got, want)
    first = ops.window_input(None, None, None, emb, 0, 64, pre, shape=(bs, total, ch))
    assert torch.equal(first, ops.window_input(motion, mask, motion[:, :pre].contiguous(), emb, 0, 64, pre))
    user = _rand(bs, total, ch, seed=72)                                 # caller-supplied motion with the same strided seed
    assert torch.equal(ops.window_input(user, mask, seed, emb, 60, 64, pre), ops.window_input(user, mask, seed.contiguous(), emb, 60, 64, pre))


def test_strided_tail_views_and_nonfinite_flag(ops):
    """row_argmax / l2_argmin on the last frames of a window read in place (clip stride = whole sequence), and the
    non-finite flag the fp16x3 pipeline relies on."""
    bs, total, nd = 5, 300, 13
    x = _rand(bs, total, 256, seed=73)
    tail = x[:, 64 - nd:64]
    assert torch.equal(ops.row_argmax(tail), tail.contiguous().argmax(-1))
    cb = _rand(256, 256, seed=74)
    e2 = ops.row_sqnorm(cb)
    for engine in ENGINES:
        assert torch.equal(ops.l2_argmin(tail, cb, e2, engine=engine), ops.l2_argmin(tail.contiguous(), cb, e2, engine=engine))
    flag = ops.zero_flag("cuda")
    ops.row_argmax(tail, nonfinite=flag)
    assert int(flag) == 0
    x[2, 60, 7] = float("inf")
    ops.row_argmax(tail, nonfinite=flag)
    assert int(flag) == 1


def test_row_argmax_first_max(ops):
    x = _rand(9600, 256, seed=36)
    x[5, 17] = x[5, 200] = 50.0                      # tie -> first index
    x[6, :] = -3.0                                   # all equal -> 0
    got = ops.row_argmax(x)
    assert torch.equal(got, torch.max(F.log_softmax(x, dim=1), dim=1)[1]) or torch.equal(got, x.argmax(1))
    assert got[5].item() == 17 and got[6].item() == 0


def test_gather_rows(ops):
    cb = _rand(256, 256, seed=37)
    idx = torch.randint(0, 256, (4, 33), generator=torch.Generator().manual_seed(38)).cuda()
    assert torch.equal(ops.gather_rows(cb, idx), cb[idx])
    bad = idx.clone()
    bad[0, 0], bad[1, 1] = 2147483647, -5              # out-of-range ids are clamped, never read out of bounds
    got = ops.gather_rows(cb, bad)
    assert torch.equal(got[0, 0], cb[255]) and torch.equal(got[1, 1], cb[0]) and torch.equal(got[2], cb[idx[2]])


def test_pose_compose_matches_oracle(ops):
    from oracle import emage_oracle as O
    from helpers import geodesic_deg
    bs, t = 3, 50
    parts = dict(face=_rand(bs, t, 106, seed=39), upper=_rand(bs, t, 78, seed=40), hands=_rand(bs, t, 180, seed=41),
                 lower=_rand(bs, t, 61, seed=42))
    expr, aa, m4 = ops.pose_compose(parts["face"], parts["upper"], parts["hands"], parts["lower"], bs, t, "cuda")
    c = {k: v.cpu() for k, v in parts.items()}
    jaw = O.rot6d_to_axis_angle(c["face"][:, :, :6])
    up = O.rot6d_to_axis_angle(c["upper"].reshape(bs, t, -1, 6)).reshape(bs, t, -1)
    ha = O.rot6d_to_axis_angle(c["hands"].reshape(bs, t, -1, 6)).reshape(bs, t, -1)
    lo = O.rot6d_to_axis_angle(c["lower"][:, :, :54].reshape(bs, t, -1, 6)).reshape(bs, t, -1)
    want = (O._scatter_joints(up, O.UPPER_JOINTS, bs, t) + O._scatter_joints(ha, O.HANDS_JOINTS, bs, t)
            + O._scatter_joints(lo, O.LOWER_JOINTS, bs, t))
    want[:, :, 66:69] = jaw
    assert torch.equal(expr.cpu(), c["face"][:, :, 6:])
    assert torch.equal(m4.cpu()[:, :, 330:], c["lower"][:, :, 54:])
    geo = geodesic_deg(aa.cpu().reshape(bs, t, 55, 3), want.reshape(bs, t, 55, 3))
    assert geo.max() < 0.02, geo.max()
    far = (want.reshape(bs, t, 55, 3).norm(dim=-1) < 3.0).unsqueeze(-1).expand(bs, t, 55, 3).reshape(bs, t, 165)
    assert (aa.cpu() - want)[far].abs().max() < 1e-3           # the pose gate; fp32 quaternion route loses ~2e-4
    want6 = O.axis_angle_to_rot6d(want.reshape(bs, t, 55, 3)).reshape(bs, t, 330)
    assert (m4.cpu()[:, :, :330] - want6).abs().max() < 1e-3
    # the reference's zero branches (M.py:143-146,174-178): eyes and missing parts are identity rotations
    expr0, aa0, m40 = ops.pose_compose(None, parts["upper"], None, None, bs, t, "cuda")
    assert expr0.abs().max() == 0 and aa0[:, :, 66:75].abs().max() == 0
    assert torch.equal(m40[0, 0, 0:6].cpu(), torch.tensor([1.0, 0, 0, 0, 1, 0]))


def test_global_trans_sequential_sum(ops):
    bs, t = 4, 300
    rec, ref = _rand(bs, t, 61, seed=43), _rand(bs, 3, seed=44)
    got = ops.global_trans(rec, ref, 1 / 30).cpu()
    assert torch.equal(ops.global_trans(rec, ref[0:1].expand(rec.shape[0], 3), 1 / 30),
                       ops.global_trans(rec, ref[0:1].expand(rec.shape[0], 3).contiguous(), 1 / 30))   # stride-0 ref
    v = rec.cpu()[:, :, 54:57]
    x, z = [ref.cpu()[:, 0:1]], [ref.cpu()[:, 2:3]]
    for i in range(1, t):                                        # P.py:107-115
        x.append(v[:, i - 1, 0:1] * (1 / 30) + x[-1])
        z.append(v[:, i - 1, 2:3] * (1 / 30) + z[-1])
    assert torch.equal(got[:, :, 0], torch.cat(x, 1)) and torch.equal(got[:, :, 2], torch.cat(z, 1))
    assert torch.equal(got[:, :, 1], v[:, :, 1])


def _planes_value(pl):
    """fp32 value the planes stand for (fp16 planes hold ops.F16_ACT_SCALE * x)."""
    from pantomatrix_b200 import ops as o
    return pl.t[:, :, :, :pl.ch].float().sum(0) / (o.F16_ACT_SCALE if pl.t.dtype == torch.float16 else 1.0)


@pytest.fixture()
def plane_format(request, ops):
    ops.set_plane_format(request.param)
    return request.param


@pytest.mark.parametrize("plane_format", ["bf16", "fp16"], indirect=True)
@pytest.mark.parametrize("nsplit", [1, 2, 3])
def test_fused_plane_outputs(ops, nsplit, plane_format):
    """Producers that write their result directly as split planes (the A-operand format of the tensor-core
    GEMM): planes must re-assemble the fp32 result to 2^-8 / 2^-16 / 2^-24 (bf16) or 2^-11 / 2^-22 / 2^-24 (fp16)
    relative accuracy."""
    tol = max(2.0 ** (-(8 if plane_format == "bf16" else 11) * nsplit), 2.0 ** -24) * 1.01
    E = 768
    x, r, g, b = _rand(4, 60, E, seed=50), _rand(4, 60, E, seed=51), _rand(E, seed=52), _rand(E, seed=53)
    ref = ops.add_layernorm(x, r, g, b)
    got = ops.add_layernorm(x, r, g, b, nsplit=nsplit)
    assert torch.equal(got.f, ref) and (_planes_value(got.p) - ref).abs().max() <= tol * ref.abs().max()
    only = ops.add_layernorm(x, r, g, b, nsplit=nsplit, f32=False)
    assert only.f is None and torch.equal(only.p.t[..., :E], got.p.t[..., :E])
    qkv = _rand(4 * 60, 3 * E, seed=54)
    ref = ops.attention(qkv[:, :E], qkv[:, E:2 * E], qkv[:, 2 * E:], 4, 4, 60, 60, 192)
    got = ops.attention(qkv[:, :E], qkv[:, E:2 * E], qkv[:, 2 * E:], 4, 4, 60, 60, 192, nsplit=nsplit, f32=False)
    assert got.f is None and (_planes_value(got.p).reshape(240, E) - ref).abs().max() <= tol * ref.abs().max()
    pe, spk = _rand(128, E, seed=55), _rand(4, E, seed=56)
    ref = ops.add_rows(x, pe, spk, ops.ROW_SPK, ops.ROW_PE, 4, 60, E)
    got = ops.add_rows(x, pe, spk, ops.ROW_SPK, ops.ROW_PE, 4, 60, E, nsplit=nsplit)
    assert torch.equal(got.f, ref) and (_planes_value(got.p) - ref).abs().max() <= tol * ref.abs().max()
    got = ops.add2(x, r, nsplit=nsplit, f32=False)
    assert (_planes_value(got.p) - (x + r)).abs().max() <= tol * (x + r).abs().max()
    cb = _rand(256, 256, seed=57)
    idx = torch.randint(0, 256, (4, 33), generator=torch.Generator().manual_seed(58)).cuda()
    got = ops.gather_rows(cb, idx, nsplit=nsplit)
    assert torch.equal(got.f, cb[idx]) and (_planes_value(got.p) - cb[idx]).abs().max() <= tol * cb.abs().max()
    motion, seed, emb = _rand(3, 130, 337, seed=59), _rand(3, 4, 337, seed=60), _rand(337, seed=61)
    mask = (torch.rand(3, 130, 337, generator=torch.Generator().manual_seed(62)) > 0.5).float().cuda()
    ref = ops.window_input(motion, mask, seed, emb, 60, 64, 4)
    got = ops.window_input(motion, mask, seed, emb, 60, 64, 4, nsplit=nsplit, f32=False)
    assert got.p.t.shape[-1] == 344 and (_planes_value(got.p) - ref).abs().max() <= tol * ref.abs().max()

"""Shadow check of real inferences (GPU): every tensor-core tap-GEMM, attention and VQ-lookup call that
pipeline.generate and the CaMN / DisCo forward make is checked, element by element, against float64 computed from the
operands that call actually received (tests/helpers.py: per-element bounds derived from the products each split mode
drops and the fp32 accumulation chains).  The calls are intercepted by replacing pantomatrix_b200.ops.tapgemm_tc /
attention_tc / l2_argmin inside the test only; the product code is unchanged.

Calls whose out= or residual= is a view into a larger tensor (window outputs written in place into the accumulated
results) must leave everything outside the view bit-for-bit unchanged, and out_slack rows must stay zero.
The pipeline runs uncaptured with the side-stream forks off, so each check runs right after its kernel on one stream."""
import pytest
import torch

from helpers import build_lstm_product, build_product, check_attention, check_l2_argmin, check_tapgemm, slack_rows
from oracle.weights import synth_audio

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def product():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    return build_product(seed=0)


def _outside(view):
    """(storage as a flat tensor, mask of the elements outside `view`, their bytes), or None when the view covers its
    storage.  Compared as bytes: the surroundings may be uninitialised memory holding NaN patterns."""
    base = torch.empty(0, dtype=view.dtype, device=view.device).set_(view.untyped_storage())
    if base.numel() == view.numel():
        return None
    mask = torch.ones(base.numel(), dtype=torch.bool, device=view.device)
    mask.as_strided(view.shape, view.stride(), view.storage_offset()).fill_(False)
    return base, mask, base[mask].view(torch.uint8).clone()


class Shadow:
    """Wrappers around the three tensor-core entry points of ops: call the kernel, then check that call."""

    def __init__(self, ops):
        self.ops = ops
        self.real = {name: getattr(ops, name) for name in ("tapgemm_tc", "attention_tc", "l2_argmin")}
        self.calls = {name: 0 for name in self.real}
        self.sigs = {name: set() for name in self.real}
        self.used = {name: (0.0, 0.0) for name in self.real}        # (kernel bound, plane-split bound)
        self.rows = [0, 0]                               # l2_argmin: rows decided by float64, rows

    def install(self, monkeypatch):
        for name in self.real:
            monkeypatch.setattr(self.ops, name, getattr(self, name))

    def _note(self, name, sig, used):
        self.calls[name] += 1
        self.sigs[name].add(sig)
        self.used[name] = tuple(max(u, v) for u, v in zip(self.used[name], used))

    def tapgemm_tc(self, a, w, bias, *, rows_in=None, rows_out, pad=0, act=0, act_cols=0, slope=0.0, residual=None,
                   want_f32=True, out_nsplit=0, out=None, a_view=None, out_slack=0, prefetch=None):
        shared = out is not None and residual is not None and \
            out.untyped_storage().data_ptr() == residual.untyped_storage().data_ptr()
        guards = [g for g in (_outside(out) if out is not None else None,
                              _outside(residual) if residual is not None and not shared else None) if g is not None]
        res_copy = residual.contiguous().clone() if residual is not None else None
        f, pl = self.real["tapgemm_tc"](a, w, bias, rows_in=rows_in, rows_out=rows_out, pad=pad, act=act, act_cols=act_cols,
                                        slope=slope, residual=residual, want_f32=want_f32, out_nsplit=out_nsplit, out=out,
                                        a_view=a_view, out_slack=out_slack, prefetch=prefetch)
        sig = (tuple(a.t.shape), a_view, rows_in, rows_out, w.taps, w.cout, w.cin, pad, act, act_cols, want_f32, out_nsplit,
               out is not None, residual is not None, out_slack, prefetch is not None)
        for base, mask, before in guards:
            assert torch.equal(base[mask].view(torch.uint8), before), f"tapgemm_tc {sig}: write outside the out= / residual= view"
        if residual is not None:
            assert torch.equal(residual.contiguous().view(torch.uint8), res_copy.view(torch.uint8)), \
                f"tapgemm_tc {sig}: residual modified"
        if pl is not None and out_slack:
            assert int(torch.count_nonzero(slack_rows(pl))) == 0, f"tapgemm_tc {sig}: out_slack rows written"
        used = check_tapgemm(a, w, bias, f, pl, tag=f"tapgemm_tc {sig}", rows_in=rows_in, rows_out=rows_out, pad=pad,
                             act=act, act_cols=act_cols, slope=slope, residual=residual, a_view=a_view)
        self._note("tapgemm_tc", sig, used)
        return f, pl

    def attention_tc(self, q, q_col0, k, k_col0, v, v_col0, batch, heads, tq, tk, head_dim, nsplit=2, f32=False):
        res = self.real["attention_tc"](q, q_col0, k, k_col0, v, v_col0, batch, heads, tq, tk, head_dim, nsplit=nsplit, f32=f32)
        sig = (batch, heads, tq, tk, q_col0, k_col0, v_col0, q.ch, k.ch, v.ch, nsplit, f32)
        used = check_attention(res, (q, q_col0, k, k_col0, v, v_col0, batch, heads, tq, tk, head_dim), tag=f"attention_tc {sig}")
        self._note("attention_tc", sig, used)
        return res

    def l2_argmin(self, z, codebook, e2, engine="auto", max_ctas=0):
        idx = self.real["l2_argmin"](z, codebook, e2, engine=engine, max_ctas=max_ctas)
        sig = (tuple(z.shape), tuple(z.stride()), engine)
        decided, rows = check_l2_argmin(idx, z, codebook, tag=f"l2_argmin {sig}")
        self.rows[0] += decided
        self.rows[1] += rows
        self._note("l2_argmin", sig, (0.0, 0.0))
        return idx

    def report(self, tag, expect):
        for name in self.real:
            extra = f", rows decided by float64 {self.rows[0]}/{self.rows[1]}" if name == "l2_argmin" else \
                f", largest fraction of the per-element bound used {self.used[name][0]:.3f} (plane split {self.used[name][1]:.3f})"
            print(f"[{tag}] {name}: {self.calls[name]} calls, {len(self.sigs[name])} shape signatures{extra}")
        for name in expect:
            assert self.calls[name] > 0 and len(self.sigs[name]) > 0, f"{tag}: no {name} call was checked"


@pytest.fixture()
def shadow(monkeypatch):
    from pantomatrix_b200 import ops
    from pantomatrix_b200.emage_audio import engine
    monkeypatch.setitem(engine._STATE, "fork", False)
    s = Shadow(ops)
    s.install(monkeypatch)
    yield s
    engine.set_precision(engine.DEFAULT_PRECISION)


@pytest.mark.parametrize("precision,bs,n_samples", [
    ("fp16x3", 5, 165867),        # 10 s + an 11-frame tail window: 311 frames
    ("bf16x6", 5, 165867),
    ("bf16x3", 5, 165867),
    ("fp16x3", 32, 160000),       # BASELINE: 32 clips x 300 frames (production grid and clip packing)
])
def test_generate_shadow(product, shadow, precision, bs, n_samples):
    from pantomatrix_b200.emage_audio import engine
    from pantomatrix_b200.pipeline import generate
    model, vqm = product
    engine.set_precision(precision)
    audio = torch.from_numpy(synth_audio(bs, n_samples, 4321)).cuda()
    lat, pred = generate(model, vqm, audio)
    torch.cuda.synchronize()
    assert all(bool(torch.isfinite(v).all()) for v in lat.values())
    shadow.report(f"generate {precision} {bs}x{n_samples}",
                  ("tapgemm_tc", "l2_argmin") + (("attention_tc",) if precision == "fp16x3" else ()))


@pytest.mark.parametrize("kind", ["camn", "disco"])
def test_lstm_forward_shadow(shadow, kind):
    """CaMN / DisCo: the WavEncoder convs (cin 32), the LSTM input projections (cin 403) and the heads (cin 512)."""
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    from pantomatrix_b200.emage_audio import engine
    engine.set_precision("fp16x3")
    model = build_lstm_product(kind)
    audio = torch.from_numpy(synth_audio(4, 160000, 99)).cuda()
    out = model(audio, torch.zeros(4, 1, dtype=torch.long, device="cuda"))
    torch.cuda.synchronize()
    assert bool(torch.isfinite(out["motion"]).all())
    cins = {s[6] for s in shadow.sigs["tapgemm_tc"]}
    print(f"[{kind}] tap-GEMM input widths {sorted(cins)}")
    assert cins >= ({32, 403, 512} if kind == "camn" else {32}), sorted(cins)
    shadow.report(f"{kind} fp16x3", ("tapgemm_tc",))

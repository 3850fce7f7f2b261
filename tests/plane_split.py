"""CPU restatement of the split-plane rule every plane-writing kernel follows (pm_common.cuh pm_store_planes_t /
pm_store_planes4_t, the pair stores of wav_stem and attention_tc, pm_split_bf16), worked on fp32 bit patterns in
numpy.  The tests hold each producer's planes to it bit for bit.

The rule, for one fp32 value x and `nsplit` planes (each plane is stored as its uint16 bit pattern):

* bf16, any nsplit: peel the running remainder, v = x; plane p = RNE_bf16(v); v -= plane p (fp32 arithmetic).
* fp16 activations (act=True): v = 64 x (exact: a power of two).
  - nsplit 2: head = (bits(v) + 0x1000) & 0xFFFFE000 with uint32 wrap (v rounded half away from zero to 11
    significant bits, exponent carry included); plane 0 = RNE_fp16(head), plane 1 = RNE_fp16(v - head).  The head is
    exact in fp16 wherever |v| >= 2^-14 and no overflow occurs, so plane 1 is the exact remainder there.
  - nsplit 1 and 3: RNE peel, as for bf16.
* Weights (act=False, ops.PackedW): RNE peel in either format, no x64 (PackedW applies its own power-of-two scale
  before the split).

Non-finite inputs are specified by class, not by payload: a NaN input gives planes whose sum is NaN, +-inf planes
whose sum is not finite.  (The two-plane fp16 head of the canonical NaN 0x7FFFFFFF wraps to -0; plane 1 = v - head
carries the NaN.)  fp32 subnormal inputs are kept (the kernels are built without flush-to-zero)."""
import numpy as np

BF16, FP16 = "bf16", "fp16"
F16_ACT_SCALE = np.float32(64.0)


def _f32(x) -> np.ndarray:
    return np.ascontiguousarray(np.asarray(x, dtype=np.float32))


def rne_bf16(v: np.ndarray) -> np.ndarray:
    """fp32 -> bf16 bits, round to nearest even (overflow to inf, subnormals kept); NaN -> a quiet NaN of its sign."""
    b = _f32(v).view(np.uint32)
    r = ((b + np.uint32(0x7FFF) + ((b >> np.uint32(16)) & np.uint32(1))) >> np.uint32(16)).astype(np.uint16)
    nan = np.isnan(_f32(v))
    return np.where(nan, ((b >> np.uint32(16)) | np.uint32(0x0040)).astype(np.uint16), r)


def rne_fp16(v: np.ndarray) -> np.ndarray:
    """fp32 -> fp16 bits, round to nearest even (numpy's conversion: overflow to inf, gradual underflow)."""
    with np.errstate(over="ignore", invalid="ignore"):
        return _f32(v).astype(np.float16).view(np.uint16)


def bits_to_f32(bits: np.ndarray, fmt: str) -> np.ndarray:
    """uint16 plane bits -> their (exact) fp32 values."""
    bits = np.asarray(bits, dtype=np.uint16)
    if fmt == BF16:
        return (bits.astype(np.uint32) << np.uint32(16)).view(np.float32)
    return bits.view(np.float16).astype(np.float32)


def f16_head(v: np.ndarray) -> np.ndarray:
    """pm_f16_head: v rounded half away from zero to 11 significant bits on the bit pattern (uint32 wrap)."""
    b = _f32(v).view(np.uint32)
    return ((b + np.uint32(0x1000)) & np.uint32(0xFFFFE000)).astype(np.uint32).view(np.float32)


def split(x, nsplit: int, fmt: str, act: bool = True) -> np.ndarray:
    """The planes of fp32 x as uint16 bits, shape (nsplit, *x.shape)."""
    assert 1 <= nsplit <= 3 and fmt in (BF16, FP16)
    v = _f32(x).copy()
    rne = rne_bf16 if fmt == BF16 else rne_fp16
    out = np.empty((nsplit,) + v.shape, dtype=np.uint16)
    with np.errstate(over="ignore", invalid="ignore"):
        if fmt == FP16 and act:
            v = v * F16_ACT_SCALE
            if nsplit == 2:
                head = f16_head(v)
                out[0] = rne_fp16(head)
                out[1] = rne_fp16(v - head)
                return out
        for p in range(nsplit):
            out[p] = rne(v)
            v = v - bits_to_f32(out[p], fmt)
    return out


def plane_sum(bits: np.ndarray, fmt: str, act: bool = True) -> np.ndarray:
    """float64 value the planes stand for (their exact sum, / 64 for fp16 activation planes)."""
    s = bits_to_f32(bits, fmt).astype(np.float64).sum(0)
    return s / 64.0 if (fmt == FP16 and act) else s


def mismatches(got: np.ndarray, x, fmt: str, act: bool = True) -> np.ndarray:
    """Boolean mask over the elements of x where the planes `got` (uint16 bits, (nsplit, *x.shape)) break the rule:
    at a finite x every plane must carry the restated bits (any NaN for a NaN); at a NaN x the plane sum must be NaN,
    at an infinite x it must not be finite."""
    x = _f32(x)
    got = np.asarray(got, dtype=np.uint16)
    want = split(x, got.shape[0], fmt, act)
    gv, wv = bits_to_f32(got, fmt), bits_to_f32(want, fmt)
    same = (got == want) | (np.isnan(gv) & np.isnan(wv))
    bad = ~same.all(0)
    with np.errstate(invalid="ignore", over="ignore"):
        s = plane_sum(got, fmt, act)
    nan_in, inf_in = np.isnan(x), np.isinf(x)
    bad = np.where(nan_in, ~np.isnan(s), bad)
    bad = np.where(inf_in, np.isfinite(s), bad)
    return bad


def edge_values() -> np.ndarray:
    """fp32 values where a split goes wrong first: ties of bf16 rounding and of the fp16 head, mantissa carries, the
    fp16 subnormal thresholds after the x64 pre-scale (2^-9 for a second plane, 2^-20 for the first), the fp16 overflow
    edge (65504 / 64 = 1023.5), fp32 subnormals, +-0, +-inf and NaN - each with both signs."""
    vals = []
    for e in (-126, -125, -60, -30, -22, -21, -20, -19, -10, -9, -8, -3, -1, 0, 1, 5, 9, 10, 20, 60, 126):
        for low in (0x0000, 0x0FFF, 0x1000, 0x1001, 0x1FFF, 0x3000, 0x7FFF, 0x8000, 0x8001, 0xFFFF, 0x17FFF, 0x18000):
            for kept in (0x000000, 0x010000, 0x7E0000, 0x7F0000):     # even / odd kept bits, a carry into the exponent
                m = (kept | low) & 0x7FFFFF
                vals.append(np.uint32(((e + 127) << 23) | m).view(np.float32))
    for t in (2.0 ** -9, 2.0 ** -20, 2.0 ** -14 / 64, 2.0 ** -24 / 64):
        b = int(np.float32(t).view(np.uint32))
        vals += [np.uint32(b + d).view(np.float32) for d in (-3, -2, -1, 0, 1, 2, 3)]
        vals += [np.float32(t * f) for f in (0.49, 0.5, 0.51, 0.75, 1.5, 1.99)]
    vals += list(np.linspace(1023.49, 1023.76, 28, dtype=np.float32))
    vals += [np.float32(1023.5), np.float32(1023.515625), np.float32(65504.0 / 64), np.float32(65520.0 / 64)]
    vals += [np.uint32(b).view(np.float32) for b in (0x00000001, 0x00000002, 0x00001000, 0x003FFFFF, 0x00400000,
                                                    0x007FFFFF, 0x00800000, 0x7F7FFFFF, 0x3F7FFFFF, 0x3F801000)]
    vals += [np.float32(1.0), np.float32(1.0 / 3.0), np.float32(np.pi), np.float32(0.0)]
    v = np.array(vals, dtype=np.float32)
    v = np.concatenate([v, -v])
    return np.concatenate([v, np.array([np.inf, -np.inf, np.nan], dtype=np.float32),
                           np.uint32([0x7FFFFFFF, 0xFFFFFFFF, 0x7FC00000]).view(np.float32)])

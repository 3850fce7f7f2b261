"""CPU restatement of the H.264 rule of pantomatrix_b200.video (DESIGN.md section 12), shared by the CPU and GPU tests
and tools/bench_video.py, on top of oracle/h264_oracle.py (O: CAVLC, transform constants, colour, parameter sets):
  - frame t is IDR when t mod gop == 0, else a P frame against frame t - 1's reconstruction; one slice per row;
  - P_Skip when every level of the zero-motion inter candidate (f = 2^qbits / 6, all 16 positions) is zero;
  - search > 0: the whole-pixel vector within +-search of lowest J = SAD_Y + LAMBDA[qp] (b(mvx) + b(mvy)), refined at
    +-2 then +-1 quarter-pels; 8.4.2.2's luma and chroma prediction;
  - Intra16x16: DC, or Horizontal when its SAD J16 is strictly lower; DC chroma;
  - intra4x4: I_NxN, each 4x4 block by the 8.3.1.2 mode of lowest SAD + lambda (1 or 4 mode bits), when J4 + c lambda
    < J16;
  - P slices: P_L0_16x16 (mvd = mv - mvp, mvp the left macroblock's vector when it is P_L0_16x16, else (0, 0)) when
    its luma SAD is <= the intra cost, intra mb_type + 5; I_PCM past 3200 bits or on a level escape.
A column of macroblocks needs only the columns to its left, so the intra candidates are computed for one column of
every row at once, and the inter candidate for the whole frame."""
from __future__ import annotations

import math
from collections import namedtuple

import numpy as np

from oracle import h264_oracle as O

SKIP, INTER, I4 = "SKIP", "P", "I4"
C_I4 = 6                                      # the I_NxN choice's constant c, in units of lambda(qp)
MB_BITS_LIMIT_P = O.MB_BITS_LIMIT + 1         # a coded macroblock and its ue(mb_skip_run): every skipped macroblock
SLICE_HEADER_BITS_GOP = 70                    # the longest slice header of either kind (IDR at qp 0, last row)
LAMBDA = [0, 0, 0, 0, 0, 0, 0, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 2, 2, 2, 2, 3, 3, 3, 4, 4, 5, 5, 6, 7, 7, 8, 9, 10, 12, 13,
          15, 17, 19, 21, 23, 26, 30, 33, 37, 42, 47, 53, 59, 66, 74, 83]
# Table 9-4, ChromaArrayType 1: coded_block_pattern of each codeNum, Inter and Intra_4x4 columns; the CODE lists invert
INTER_CBP = [0, 16, 1, 2, 4, 8, 32, 3, 5, 10, 12, 15, 47, 7, 11, 13, 14, 6, 9, 31, 35, 37, 42, 44, 33, 34, 36, 40,
             39, 43, 45, 46, 17, 18, 20, 24, 19, 21, 26, 28, 23, 27, 29, 30, 22, 25, 38, 41]
INTRA_CBP = [47, 31, 15, 0, 23, 27, 29, 30, 7, 11, 13, 14, 39, 43, 45, 46, 16, 3, 5, 10, 12, 19, 21, 26, 28, 35, 37,
             42, 44, 1, 2, 4, 8, 17, 18, 20, 24, 6, 9, 22, 25, 32, 33, 34, 36, 40, 38, 41]
INTER_CODE = [INTER_CBP.index(c) for c in range(48)]
INTRA_CODE = [INTRA_CBP.index(c) for c in range(48)]
LUMA_BLK = [(2 * (b // 8) + (b % 4) // 2, 2 * ((b // 4) % 2) + b % 2) for b in range(16)]   # luma4x4BlkIdx -> by, bx
BLK_OF = {rc: b for b, rc in enumerate(LUMA_BLK)}

# One coded frame.  types: 'DC', 'H' (Intra16x16), 'I4', 'PCM', 'P' or 'SKIP' per macroblock; modes (H/16, W/16, 4, 4)
# the Intra 4x4 modes by block row and column, -1 outside I_NxN macroblocks; mv (H/16, W/16, 2) the quarter-pel (x, y)
# vectors, zero where not P_L0_16x16, None for IDR frames.
Frame = namedtuple("Frame", "data recon types modes mv")


def lam(qp):
    """lambda(qp) from its formula, in float64."""
    return math.floor(math.sqrt(0.85 * 2.0 ** ((qp - 12) / 3)) + 0.5)


def max_bytes(h, w, gop=1):
    """Per-frame bound.  gop 1: oracle.h264_oracle.max_bytes.  gop > 1: each slice has at most
    P = ceil((70 + 3201 (w / 16) + 8) / 8) RBSP bytes: the longest slice header, at most 3201 bits per macroblock (a
    coded macroblock_layer() of at most 3200 bits after its ue(mb_skip_run) of 1 bit, or a skip run of r >= 1
    macroblocks in at most 2 log2(r + 1) + 1 <= 3 r bits, I_PCM 9 + 7 + 3072), the stop bit and alignment; then P / 2
    emulation prevention bytes and the 4-byte length prefix."""
    if gop == 1:
        return O.max_bytes(h, w)
    p = (SLICE_HEADER_BITS_GOP + MB_BITS_LIMIT_P * (w // 16) + 8 + 7) // 8
    return (h // 16) * (4 + p + p // 2)


def sps(h, w, gop=1):
    """oracle.h264_oracle.sps with max_num_ref_frames = 1 when gop > 1: the ue(0) at bit 37 becomes ue(1)."""
    if gop == 1:
        return O.sps(h, w)
    b = O.Bits()
    b.put(0x67, 8), b.put(66, 8), b.put(0xC0, 8), b.put(51, 8)
    b.ue(0), b.ue(0), b.ue(2), b.ue(1)                  # sps id, log2_max_frame_num - 4, poc type 2, one reference
    b.put(0, 1)
    b.ue(w // 16 - 1), b.ue(h // 16 - 1)
    b.put(1, 1), b.put(1, 1), b.put(0, 1), b.put(1, 1), b.put(0, 1), b.put(0, 1), b.put(1, 1), b.put(5, 3)
    b.put(0, 1), b.put(1, 1), b.put(6, 8), b.put(6, 8), b.put(6, 8)
    for _ in range(6):
        b.put(0, 1)
    b.trailing()
    return O.emulation_prevent(b.tobytes())


def p_slice_header(first_mb, frame_num, qp):
    b = O.Bits()
    b.put(0x41, 8)                        # nal_ref_idc 2, nal_unit_type 1 (non-IDR)
    b.ue(first_mb)
    b.ue(5)                               # slice_type: P, every slice of the picture
    b.ue(0)                               # pic_parameter_set_id
    b.put(frame_num, 4)
    b.put(0, 1)                           # num_ref_idx_active_override_flag
    b.put(0, 1)                           # ref_pic_list_modification_flag_l0
    b.put(0, 1)                           # adaptive_ref_pic_marking_mode_flag
    b.se(qp - 26)                         # slice_qp_delta
    b.ue(1)                               # disable_deblocking_filter_idc
    return b


# ---- transform, quantisation and reconstruction, over any leading axes ----

def _mbs(plane, n):
    """(H, W) -> (H / n, W / n, n, n): the n x n macroblocks of a plane."""
    h, w = plane.shape
    return plane.reshape(h // n, n, w // n, n).swapaxes(1, 2)


def _plane(mbs):
    """_mbs' inverse."""
    mbh, mbw, n, _ = mbs.shape
    return mbs.swapaxes(1, 2).reshape(mbh * n, mbw * n)


def _split(x):
    """(..., n, n) -> (..., n / 4, n / 4, 4, 4): the 4x4 blocks of x by block row and column."""
    *lead, n, _ = x.shape
    return x.reshape(*lead, n // 4, 4, n // 4, 4).swapaxes(-3, -2)


def _join(b):
    """_split's inverse."""
    *lead, k, _, _, _ = b.shape
    return b.swapaxes(-3, -2).reshape(*lead, 4 * k, 4 * k)


def _fdct(blk):
    """The 4x4 forward core transform of every block of (..., 4, 4)."""
    return np.einsum("ij,...jk,lk->...il", O.CF, blk, O.CF)


def _idct(d):
    """8.5.12.2 of every block of (..., 4, 4): rows first, then columns, then (x + 32) >> 6."""
    def one(x):
        e0, e1 = x[..., 0] + x[..., 2], x[..., 0] - x[..., 2]
        e2, e3 = (x[..., 1] >> 1) - x[..., 3], x[..., 1] + (x[..., 3] >> 1)
        return np.stack([e0 + e3, e1 + e2, e1 - e2, e0 - e3], -1)
    return (one(one(d).swapaxes(-1, -2)).swapaxes(-1, -2) + 32) >> 6


def _quant(w, qp, div):
    """Levels of the coefficients w (..., 4, 4) with f = 2^qbits / div: 3 for intra, 6 for inter."""
    qbits = 15 + qp // 6
    return np.sign(w) * ((np.abs(w) * np.array(O.MF[qp % 6])[O.CLASS] + (1 << qbits) // div) >> qbits)


def _quant_dc(d, qp, div):
    qbits = 15 + qp // 6
    return np.sign(d) * ((np.abs(d) * O.MF[qp % 6][0] + 2 * ((1 << qbits) // div)) >> (qbits + 1))


def _scale(c, qp):
    """8.5.12.1 for all 16 positions of every block of (..., 4, 4)."""
    ls = 16 * np.array(O.V[qp % 6])[O.CLASS]
    if qp >= 24:
        return (c * ls) << (qp // 6 - 4)
    return (c * ls + (1 << (3 - qp // 6))) >> (4 - qp // 6)


def _scan(x, first=0):
    """(..., 4, 4) raster -> (..., 16 - first) in zig-zag order from scan position first."""
    return x.reshape(*x.shape[:-2], 16)[..., O.ZIGZAG[first:]]


def _luma(src, pred, qp, div):
    """Levels (..., 4, 4, 4, 4) of all 16 positions of each 4x4 block of src - pred (..., 16, 16), and the
    reconstruction."""
    q = _quant(_fdct(_split(src - pred)), qp, div)
    return q, np.clip(pred + _join(_idct(_scale(q, qp))), 0, 255)


def _chroma(src, pred, qp, div):
    """Chroma of (..., 2, 8, 8) samples against pred: AC levels (..., 2, 2, 2, 4, 4) with position 0 zero, DC levels
    (..., 2, 2, 2) by 8.5.11's 2x2 transform, and the reconstruction."""
    qpc = O.QPC[qp]
    w = _fdct(_split(src - pred))
    ac = _quant(w, qpc, div)
    ac[..., 0, 0] = 0
    dc = _quant_dc(O.H2 @ w[..., 0, 0] @ O.H2, qpc, div)
    c = _scale(ac, qpc)
    c[..., 0, 0] = ((O.H2 @ dc @ O.H2 * 16 * O.V[qpc % 6][0]) << (qpc // 6)) >> 5
    return ac, dc, np.clip(pred + _join(_idct(c)), 0, 255)


# ---- motion ----

def se_len(v):
    """Bits of se(v), elementwise."""
    k = np.where(np.asarray(v) > 0, 2 * np.asarray(v) - 1, -2 * np.asarray(v)).astype(np.int64)
    return 2 * np.floor(np.log2(k + 1)).astype(np.int64) + 1


def _at(a, dy, dx):
    """a[Y + dy, X + dx] (wrapping; only read far from the padded border)."""
    return np.roll(a, (-dy, -dx), (0, 1))


def luma_phases(y, m):
    """P[fy, fx] (4, 4, H + 2m, W + 2m): the 8.4.2.2.1 prediction at quarter-pel phase (fx, fy) right of and below each
    sample of y padded by m with its edge samples (reading the padding is reading clipped coordinates).  Exact at
    least 3 samples from the padded border."""
    g = np.pad(y, m, mode="edge").astype(np.int64)
    tap = lambda a, ax: sum(c * np.roll(a, -o, ax) for o, c in zip(range(-2, 4), (1, -5, 20, 20, -5, 1)))
    b1, h1 = tap(g, 1), tap(g, 0)
    clip = lambda v: np.clip(v, 0, 255)
    b, h, j = clip((b1 + 16) >> 5), clip((h1 + 16) >> 5), clip((tap(b1, 0) + 512) >> 10)
    m_, s = _at(h, 0, 1), _at(b, 1, 0)                  # the vertical half right of h, the horizontal half below b
    avg = lambda u, v: (u + v + 1) >> 1
    p = np.empty((4, 4) + g.shape, np.int64)
    p[0] = [g, avg(g, b), b, avg(_at(g, 0, 1), b)]                          # G a b c
    p[1] = [avg(g, h), avg(b, h), avg(b, j), avg(b, m_)]                    # d e f g
    p[2] = [h, avg(h, j), j, avg(j, m_)]                                    # h i j k
    p[3] = [avg(_at(g, 1, 0), h), avg(h, s), avg(j, s), avg(m_, s)]         # n p q r
    return p


def _mb_grid(mbh, mbw, n):
    """Row and column offsets (mbh, mbw, n, n) of every n x n block of the macroblocks."""
    my, mx = np.meshgrid(np.arange(mbh), np.arange(mbw), indexing="ij")
    return n * my[..., None, None] + np.arange(n)[:, None], n * mx[..., None, None] + np.arange(n)[None, :]


def luma_pred(phases, m, mv):
    """The luma prediction (mbh, mbw, 16, 16) of every macroblock at its quarter-pel vector mv (mbh, mbw, 2) (x, y)."""
    r, c = _mb_grid(*mv.shape[:2], 16)
    vx, vy = mv[..., 0][..., None, None], mv[..., 1][..., None, None]
    return phases[vy & 3, vx & 3, m + r + (vy >> 2), m + c + (vx >> 2)]


def chroma_pred(plane, mv):
    """8.4.2.2.2: the (mbh, mbw, 8, 8) chroma prediction of one plane, the luma vector in eighth chroma samples."""
    hc, wc = plane.shape
    r, c = _mb_grid(*mv.shape[:2], 8)
    vx, vy = mv[..., 0][..., None, None], mv[..., 1][..., None, None]
    x, y, fx, fy = c + (vx >> 3), r + (vy >> 3), vx & 7, vy & 7
    at = lambda dy, dx: plane[np.clip(y + dy, 0, hc - 1), np.clip(x + dx, 0, wc - 1)]
    return ((8 - fx) * (8 - fy) * at(0, 0) + fx * (8 - fy) * at(0, 1) + (8 - fx) * fy * at(1, 0) + fx * fy * at(1, 1)
            + 32) >> 6


def motion_search(cur_y, ref_y, qp, rng):
    """The searched quarter-pel vector (mbh, mbw, 2) (x, y) of every macroblock of cur_y against ref_y, rng >= 1."""
    h, w = cur_y.shape
    mbh, mbw = h // 16, w // 16
    lmb = LAMBDA[qp]
    m = rng + 8
    pad = np.pad(ref_y, m, mode="edge")
    my, mx = np.meshgrid(np.arange(mbh), np.arange(mbw), indexing="ij")
    best_j = np.full((mbh, mbw), np.iinfo(np.int64).max)
    best = np.zeros((mbh, mbw, 2), np.int64)
    # the tie rule as the visiting order: a later candidate replaces only with a strictly lower J
    order = sorted(((dx, dy) for dy in range(-rng, rng + 1) for dx in range(-rng, rng + 1)),
                   key=lambda v: (abs(v[0]) + abs(v[1]), v[1], v[0]))
    for dx, dy in order:
        shifted = pad[m + dy:m + dy + h, m + dx:m + dx + w]
        sad = np.abs(cur_y - shifted).reshape(mbh, 16, mbw, 16).sum((1, 3))
        j = sad + lmb * int(se_len(4 * dx) + se_len(4 * dy))
        inside = (16 * mx + dx >= 0) & (16 * mx + dx + 16 <= w) & (16 * my + dy >= 0) & (16 * my + dy + 16 <= h)
        better = inside & (j < best_j)
        best_j = np.where(better, j, best_j)
        best[better] = (4 * dx, 4 * dy)
    phases = luma_phases(ref_y, m)
    src = _mbs(cur_y, 16)
    for step in (2, 1):
        centre = best.copy()
        for oy in (-step, 0, step):
            for ox in (-step, 0, step):
                if ox == oy == 0:
                    continue
                cand = centre + (ox, oy)
                j = np.abs(src - luma_pred(phases, m, cand)).sum((2, 3)) + lmb * (se_len(cand[..., 0])
                                                                                   + se_len(cand[..., 1]))
                better = j < best_j
                best_j = np.where(better, j, best_j)
                best[better] = cand[better]
    return best


# ---- intra candidates of one macroblock column ----

def _intra16(ys, ly, qp):
    """The Intra16x16 candidate of n macroblocks: ys (n, 16, 16) samples, ly (n, 16) the left macroblocks'
    reconstructed right columns or None.  Returns whether Horizontal (n,), J16 (n,), DC levels (n, 4, 4), AC levels
    (n, 4, 4, 4, 4) with position 0 zero, and the reconstruction."""
    if ly is None:
        pred = np.full_like(ys, 128)
        use_h = np.zeros(len(ys), bool)
    else:
        ph, pdc = ly[:, :, None], ((ly.sum(1) + 8) >> 4)[:, None, None]
        use_h = np.abs(ys - ph).sum((1, 2)) < np.abs(ys - pdc).sum((1, 2))
        pred = np.where(use_h[:, None, None], ph, pdc)
    w = _fdct(_split(ys - pred))
    ac = _quant(w, qp, 3)
    ac[..., 0, 0] = 0
    d = O.H4 @ w[..., 0, 0] @ O.H4
    dc = np.sign(d) * _quant_dc(np.abs(d) >> 1, qp, 3)
    f, ls0 = O.H4 @ dc @ O.H4, 16 * O.V[qp % 6][0]
    c = _scale(ac, qp)
    c[..., 0, 0] = (f * ls0) << (qp // 6 - 6) if qp >= 36 else (f * ls0 + (1 << (5 - qp // 6))) >> (6 - qp // 6)
    return use_h, np.abs(ys - pred).sum((1, 2)), dc, ac, np.clip(pred + _join(_idct(c)), 0, 255)


def _ar_available(by, bx):
    """6.4.11.4 inside one macroblock: the block above-right of (by, bx) is coded before it (and lies in this
    macroblock, as the macroblocks above and to the right are not available)."""
    return by > 0 and bx < 3 and BLK_OF[(by - 1, bx + 1)] < BLK_OF[(by, bx)]


def predict(mode, top, left, tl):
    """8.3.1.2: the (n, 4, 4) [y, x] prediction of mode 0, 1, 3..8 from p[x, -1] = top[:, x] (x 0..7), p[-1, y] =
    left[:, y] and p[-1, -1] = tl."""
    def p(x, y):
        if y == -1:
            return tl if x == -1 else top[:, x]
        return left[:, y]
    out = np.empty(((top if top is not None else left).shape[0], 4, 4), np.int64)
    t3 = lambda a, b, c: (a + 2 * b + c + 2) >> 2
    a2 = lambda a, b: (a + b + 1) >> 1
    for y in range(4):
        for x in range(4):
            if mode == 0:
                v = p(x, -1)
            elif mode == 1:
                v = p(-1, y)
            elif mode == 3:
                v = (p(6, -1) + 3 * p(7, -1) + 2) >> 2 if x == y == 3 else t3(p(x + y, -1), p(x + y + 1, -1),
                                                                               p(x + y + 2, -1))
            elif mode == 4:
                if x > y:
                    v = t3(p(x - y - 2, -1), p(x - y - 1, -1), p(x - y, -1))
                elif x < y:
                    v = t3(p(-1, y - x - 2), p(-1, y - x - 1), p(-1, y - x))
                else:
                    v = t3(p(0, -1), p(-1, -1), p(-1, 0))
            elif mode == 5:
                z = 2 * x - y
                if z >= 0 and z % 2 == 0:
                    v = a2(p(x - (y >> 1) - 1, -1), p(x - (y >> 1), -1))
                elif z >= 0:
                    v = t3(p(x - (y >> 1) - 2, -1), p(x - (y >> 1) - 1, -1), p(x - (y >> 1), -1))
                elif z == -1:
                    v = t3(p(-1, 0), p(-1, -1), p(0, -1))
                else:
                    v = t3(p(-1, y - 1), p(-1, y - 2), p(-1, y - 3))
            elif mode == 6:
                z = 2 * y - x
                if z >= 0 and z % 2 == 0:
                    v = a2(p(-1, y - (x >> 1) - 1), p(-1, y - (x >> 1)))
                elif z >= 0:
                    v = t3(p(-1, y - (x >> 1) - 2), p(-1, y - (x >> 1) - 1), p(-1, y - (x >> 1)))
                elif z == -1:
                    v = t3(p(-1, 0), p(-1, -1), p(0, -1))
                else:
                    v = t3(p(x - 1, -1), p(x - 2, -1), p(x - 3, -1))
            elif mode == 7:
                if y % 2 == 0:
                    v = a2(p(x + (y >> 1), -1), p(x + (y >> 1) + 1, -1))
                else:
                    v = t3(p(x + (y >> 1), -1), p(x + (y >> 1) + 1, -1), p(x + (y >> 1) + 2, -1))
            else:
                z = x + 2 * y
                if z in (0, 2, 4):
                    v = a2(p(-1, y + (x >> 1)), p(-1, y + (x >> 1) + 1))
                elif z in (1, 3):
                    v = t3(p(-1, y + (x >> 1)), p(-1, y + (x >> 1) + 1), p(-1, y + (x >> 1) + 2))
                elif z == 5:
                    v = (p(-1, 2) + 3 * p(-1, 3) + 2) >> 2
                else:
                    v = p(-1, 3)
            out[:, y, x] = v
    return out


def i4_candidate(src, ly, lmode, qp):
    """The I_NxN candidate of n macroblocks: src (n, 16, 16) luma, ly (n, 16) the left macroblocks' reconstructed
    right columns or None, lmode (n, 4) the modes of their right blocks (2 where not I_NxN).  Returns J4 (n,), recon
    (n, 16, 16), modes and predicted modes (n, 4, 4), levels (n, 4, 4, 4, 4) by block row and column."""
    n = src.shape[0]
    lmb = LAMBDA[qp]
    rec = np.zeros((n, 16, 16), np.int64)
    modes, predm = np.zeros((n, 4, 4), np.int64), np.zeros((n, 4, 4), np.int64)
    lev = np.zeros((n, 4, 4, 4, 4), np.int64)
    j4 = np.zeros(n, np.int64)
    for by, bx in LUMA_BLK:
        ys, xs = slice(4 * by, 4 * by + 4), slice(4 * bx, 4 * bx + 4)
        la, ua = bx > 0 or ly is not None, by > 0
        left = rec[:, ys, 4 * bx - 1] if bx > 0 else (ly[:, 4 * by:4 * by + 4] if la else None)
        top = tl = None
        if ua:
            top = np.empty((n, 8), np.int64)
            top[:, :4] = rec[:, 4 * by - 1, xs]
            top[:, 4:] = (rec[:, 4 * by - 1, 4 * bx + 4:4 * bx + 8] if _ar_available(by, bx)
                          else top[:, 3:4])
            if la:
                tl = rec[:, 4 * by - 1, 4 * bx - 1] if bx > 0 else ly[:, 4 * by - 1]
        # 8.3.1.1: dcPredModePredictedFlag when the block above or to the left is not available; a neighbour outside
        # I_NxN counts as mode 2
        if not (la and ua):
            pm = np.full(n, 2, np.int64)
        else:
            pm = np.minimum(modes[:, by, bx - 1] if bx > 0 else lmode[:, by], modes[:, by - 1, bx])
        cost = np.full((9, n), np.iinfo(np.int64).max)
        preds = {}
        for m in range(9):
            if m == 2:
                if la and ua:
                    dc = (top[:, :4].sum(1) + left.sum(1) + 4) >> 3
                elif la:
                    dc = (left.sum(1) + 2) >> 2
                elif ua:
                    dc = (top[:, :4].sum(1) + 2) >> 2
                else:
                    dc = np.full(n, 128, np.int64)
                preds[m] = np.broadcast_to(dc[:, None, None], (n, 4, 4))
            elif (m in (0, 3, 7) and ua) or (m in (1, 8) and la) or (m in (4, 5, 6) and la and ua):
                preds[m] = predict(m, top, left, tl)
            else:
                continue
            cost[m] = np.abs(src[:, ys, xs] - preds[m]).sum((1, 2)) + lmb * np.where(pm == m, 1, 4)
        best = np.argmin(cost, 0)                          # the first minimum: ties go to the lower mode
        j4 += cost[best, np.arange(n)]
        pred = np.stack([preds.get(m, np.zeros((n, 4, 4), np.int64)) for m in range(9)])[best, np.arange(n)]
        q = _quant(_fdct(src[:, ys, xs] - pred), qp, 3)
        rec[:, ys, xs] = np.clip(pred + _idct(_scale(q, qp)), 0, 255)
        modes[:, by, bx], predm[:, by, bx], lev[:, by, bx] = best, pm, q
    return j4, rec, modes, predm, lev


# ---- macroblock_layer() ----

def _nc(grid, left, by, bx):
    """nC (9.2.1) of block (by, bx) from the TotalCoeff grid of its macroblock and of the left macroblock (None when
    there is none): a P_Skip neighbour holds 0, an I_PCM one 16."""
    a = grid[by, bx - 1] if bx > 0 else (None if left is None else left[by, -1])
    t = grid[by - 1, bx] if by > 0 else None
    if a is not None and t is not None:
        return (int(a) + int(t) + 1) >> 1
    return int(a) if a is not None else (int(t) if t is not None else 0)


def _cbp_chroma(cac, cdc):
    return 2 if cac.any() else (1 if cdc.any() else 0)


def _cbp_luma(lev):
    """One bit per 8x8 block holding a non-zero level; lev (4, 4, ...) by block row and column."""
    return sum(1 << b8 for b8 in range(4) if lev[2 * (b8 // 2):2 * (b8 // 2) + 2, 2 * (b8 % 2):2 * (b8 % 2) + 2].any())


def _residual(b, luma, cbp_l, cac, cdc, nz, left):
    """residual() into b: the luma blocks (luma (4, 4, k): levels in scan order) of each coded 8x8 block, then chroma DC
    and AC.  nz = (luma (4, 4), chroma (2, 2, 2)) TotalCoeff grids of this macroblock, filled here; left: the left
    macroblock's, or None.  Raises O.LevelEscape."""
    for by, bx in LUMA_BLK:
        if cbp_l >> ((by // 2) * 2 + bx // 2) & 1:
            nz[0][by, bx] = O.residual_block(b, luma[by, bx].tolist(), _nc(nz[0], left and left[0], by, bx),
                                             luma.shape[-1])
    cbp_c = _cbp_chroma(cac, cdc)
    if cbp_c:
        for k in range(2):
            O.residual_block(b, cdc[k].reshape(4).tolist(), -1, 4)
    if cbp_c == 2:
        for k in range(2):
            for by, bx in ((0, 0), (0, 1), (1, 0), (1, 1)):
                nz[1][k, by, bx] = O.residual_block(b, _scan(cac[k, by, bx], 1).tolist(),
                                                    _nc(nz[1][k], left and left[1][k], by, bx), 15)


def encode_inter_mb(ly, cac, cdc, nz, left, mvd):
    """One P_L0_16x16 macroblock_layer(): ly (4, 4, 4, 4) luma levels by block row and column, cac (2, 2, 2, 4, 4) and
    cdc (2, 2, 2) chroma levels, mvd its mvd_l0 (x, y); nz, left as _residual's."""
    luma = _scan(ly)
    cbp = _cbp_luma(luma) | _cbp_chroma(cac, cdc) << 4
    b = O.Bits()
    b.ue(0)                                               # mb_type P_L0_16x16
    b.se(int(mvd[0])), b.se(int(mvd[1]))
    b.ue(INTER_CODE[cbp])
    if cbp:
        b.se(0)                                           # mb_qp_delta
    _residual(b, luma, cbp & 15, cac, cdc, nz, left)
    return b


def _intra16_mb(use_h, dc, ac, cac, cdc, nz, left, mb_type):
    """One Intra16x16 macroblock_layer() with DC chroma; mb_type 1 in I slices, 6 in P slices."""
    cbp_l, cbp_c = 15 if ac.any() else 0, _cbp_chroma(cac, cdc)
    b = O.Bits()
    b.ue(mb_type + (1 if use_h else 2) + 4 * cbp_c + 12 * (cbp_l == 15))
    b.ue(0)                                               # intra_chroma_pred_mode: DC
    b.se(0)                                               # mb_qp_delta
    O.residual_block(b, _scan(dc).tolist(), _nc(nz[0], left and left[0], 0, 0), 16)
    _residual(b, _scan(ac, 1), cbp_l, cac, cdc, nz, left)
    return b


def _intra4_mb(modes, predm, lev, cac, cdc, nz, left, mb_type):
    """One I_NxN macroblock_layer() with DC chroma; mb_type 0 in I slices, 5 in P slices."""
    luma = _scan(lev)
    cbp = _cbp_luma(luma) | _cbp_chroma(cac, cdc) << 4
    b = O.Bits()
    b.ue(mb_type)
    for by, bx in LUMA_BLK:
        m, pm = int(modes[by, bx]), int(predm[by, bx])
        if m == pm:
            b.put(1, 1)                                   # prev_intra4x4_pred_mode_flag
        else:
            b.put(0, 1)
            b.put(m if m < pm else m - 1, 3)              # rem_intra4x4_pred_mode
    b.ue(0)                                               # intra_chroma_pred_mode: DC
    b.ue(INTRA_CODE[cbp])
    if cbp:
        b.se(0)                                           # mb_qp_delta
    _residual(b, luma, cbp & 15, cac, cdc, nz, left)
    return b


def _pcm(b, y, c, mb_type):
    """I_PCM: mb_type (25 in I slices, 30 in P slices), pcm_alignment_zero_bits, the 384 samples."""
    b.ue(mb_type)
    b.put(0, (-b.n) % 8)
    b.put(int.from_bytes(np.concatenate([y.reshape(-1), c.reshape(-1)]).astype(np.uint8).tobytes(), "big"), 8 * 384)


# ---- frames ----

def encode_frame(frame, ref, qp, t, gop, search=0, intra4x4=False, c=C_I4):
    """Frame t of its clip, (H, W, 3) uint8: IDR when ref is None, else a P frame against ref (Y, Cb, Cr)."""
    frame = np.asarray(frame)
    h, w, _ = frame.shape
    O.check_shape(h, w)
    mbh, mbw = h // 16, w // 16
    cur = O.colour(frame)
    ys, cs = _mbs(cur[0], 16), np.stack([_mbs(cur[1], 8), _mbs(cur[2], 8)], 2)    # (mbh, mbw, 16, 16), (.., 2, 8, 8)
    pf = ref is not None
    intra_type = 5 if pf else 0                           # mb_type of I_NxN; Intra16x16 and I_PCM follow it
    rec_y, rec_c = np.zeros_like(ys), np.zeros_like(cs)
    types = np.empty((mbh, mbw), object)
    modes = np.full((mbh, mbw, 4, 4), -1, np.int64)
    mv = np.zeros((mbh, mbw, 2), np.int64)
    nz = (np.zeros((mbh, mbw, 4, 4), np.int64), np.zeros((mbh, mbw, 2, 2, 2), np.int64))
    if pf:
        col_y, col_c = _mbs(ref[0], 16), np.stack([_mbs(ref[1], 8), _mbs(ref[2], 8)], 2)
        zero_motion = _luma(ys, col_y, qp, 6), _chroma(cs, col_c, qp, 6)
        if search:
            vec = motion_search(cur[0], ref[0], qp, search)
            m = search + 8
            py = luma_pred(luma_phases(ref[0], m), m, vec)
            pc = np.stack([chroma_pred(ref[1], vec), chroma_pred(ref[2], vec)], 2)
            inter = _luma(ys, py, qp, 6), _chroma(cs, pc, qp, 6)
        else:                                             # the co-located reference: no search, no interpolation
            vec, py, inter = np.zeros_like(mv), col_y, zero_motion
        (zl, _), (zac, zdc, _) = zero_motion
        skip = ~(zl.any((2, 3, 4, 5)) | zac.any((2, 3, 4, 5, 6)) | zdc.any((2, 3, 4)))
        (ly, ry), (cac, cdc, rc) = inter
        sad = np.abs(ys - py).sum((2, 3))
    slices = [p_slice_header(my * mbw, (t % gop) % 16, qp) if pf else O.slice_header(my * mbw, (t // gop) % 2, qp)
              for my in range(mbh)]
    runs = [0] * mbh
    for mx in range(mbw):
        lcol = rec_y[:, mx - 1, :, 15] if mx else None
        # the intra chroma: DC of each half of the left macroblocks' reconstructed right columns
        cpred = (np.full_like(cs[:, mx], 128) if not mx else
                 np.repeat((rec_c[:, mx - 1, :, :, 7].reshape(mbh, 2, 2, 4).sum(-1) + 2) >> 2, 4, -1)[..., None])
        icac, icdc, irc = _chroma(cs[:, mx], cpred, qp, 3)
        use_h, j16, dc16, ac16, r16 = _intra16(ys[:, mx], lcol, qp)
        if intra4x4:
            lmode = np.where(modes[:, mx - 1, :, 3] < 0, 2, modes[:, mx - 1, :, 3]) if mx else None
            j4, r4, m4, pm4, lev4 = i4_candidate(ys[:, mx], lcol, lmode, qp)
        for my in range(mbh):
            at, b = (my, mx), slices[my]
            left = (nz[0][my, mx - 1], nz[1][my, mx - 1]) if mx else None
            mb_nz = (nz[0][at], nz[1][at])
            if pf and skip[at]:
                runs[my] += 1
                types[at], rec_y[at], rec_c[at] = SKIP, col_y[at], col_c[at]
                continue
            j_intra = j16[my]
            use_i4 = intra4x4 and j4[my] + c * LAMBDA[qp] < j_intra
            if use_i4:
                j_intra = j4[my] + c * LAMBDA[qp]
            try:
                if pf and sad[at] <= j_intra:
                    mvp = mv[my, mx - 1] if mx else 0
                    mb = encode_inter_mb(ly[at], cac[at], cdc[at], mb_nz, left, vec[at] - mvp)
                    kind, r, mv[at] = INTER, (ry[at], rc[at]), vec[at]
                elif use_i4:
                    mb = _intra4_mb(m4[my], pm4[my], lev4[my], icac[my], icdc[my], mb_nz, left, intra_type)
                    kind, r, modes[at] = I4, (r4[my], irc[my]), m4[my]
                else:
                    mb = _intra16_mb(use_h[my], dc16[my], ac16[my], icac[my], icdc[my], mb_nz, left, intra_type + 1)
                    kind, r = ("H" if use_h[my] else "DC"), (r16[my], irc[my])
            except O.LevelEscape:
                mb = None
            if pf:
                b.ue(runs[my])
                runs[my] = 0
            if mb is None or mb.n > O.MB_BITS_LIMIT:
                _pcm(b, ys[at], cs[at], intra_type + 25)
                kind, r, modes[at], mv[at] = O.PCM, (ys[at], cs[at]), -1, 0
                mb_nz[0][:], mb_nz[1][:] = 16, 16
            else:
                b.extend(mb)
            types[at], (rec_y[at], rec_c[at]) = kind, r
    out = bytearray()
    for b, run in zip(slices, runs):
        if run:
            b.ue(run)
        b.trailing()
        nal = O.emulation_prevent(b.tobytes())
        out += len(nal).to_bytes(4, "big") + nal
    recon = (_plane(rec_y), _plane(rec_c[:, :, 0]), _plane(rec_c[:, :, 1]))
    return Frame(bytes(out), recon, types, modes, mv if pf else None)


def encode_clip(frames, qp=20, gop=1, search=0, intra4x4=False, c=C_I4):
    """The Frames of one clip (a list of (H, W, 3) uint8 frames) with keyframe interval gop, search range search and
    Intra 4x4 on or off.  c is the I_NxN choice's constant; without intra4x4 the candidate is not computed."""
    out = []
    for t, f in enumerate(frames):
        out.append(encode_frame(f, out[-1].recon if t % gop else None, qp, t, gop, search, intra4x4, c))
        h, w = out[-1].recon[0].shape
        assert len(out[-1].data) <= max_bytes(h, w, gop)
    return out

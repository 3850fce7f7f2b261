"""CPU restatement of the H.264 encoding rule of pantomatrix_b200.video (DESIGN.md section 12) (TEST / MEASUREMENT
INFRASTRUCTURE; never imported by the product).

Each (H, W, 3) uint8 RGB frame (H, W multiples of 16) becomes one IDR access unit of a Constrained Baseline stream:
  - colour: BT.601 limited range in integers, Y per pixel, Cb / Cr from the sums of each 2x2 block;
  - one I slice per macroblock row, deblocking off, every macroblock Intra16x16 (DC or Horizontal luma, DC chroma) or
    I_PCM when its Intra16x16 layer would pass 3200 bits or need a level_prefix above 15;
  - each slice one NAL unit with emulation prevention, prefixed by its 4-byte big-endian length.
The parameter sets, the slice header, the transform, quantisation, reconstruction and the CAVLC code tables (ITU-T
H.264 tables 9-5, 9-7, 9-8, 9-9 and 9-10) are written out here from the standard.  encode() also returns the
reconstruction and the macroblock types, which a decoder's output must equal.
"""
from __future__ import annotations

import numpy as np

MAX_FS, MAX_DIM_MBS = 36864, 543          # level 5.1 MaxFS, and sqrt(8 MaxFS) in macroblocks
MB_BITS_LIMIT = 3200                      # 128 + RawMbBits (A.3.1)
PCM = "PCM"

# ---- CAVLC tables: codes as (length, value) ----
# coeff_token, table 9-5, indexed [nC class][4 * TotalCoeff + TrailingOnes], classes 0 <= nC < 2, 2 <= nC < 4,
# 4 <= nC < 8; 8 <= nC is the 6-bit fixed-length code and nC = -1 (chroma DC) has its own table
_CT_LEN = [
    [1, 0, 0, 0, 6, 2, 0, 0, 8, 6, 3, 0, 9, 8, 7, 5, 10, 9, 8, 6, 11, 10, 9, 7, 13, 11, 10, 8, 13, 13, 11, 9,
     13, 13, 13, 10, 14, 14, 13, 11, 14, 14, 14, 13, 15, 15, 14, 14, 15, 15, 15, 14, 16, 15, 15, 15, 16, 16, 16, 15,
     16, 16, 16, 16, 16, 16, 16, 16],
    [2, 0, 0, 0, 6, 2, 0, 0, 6, 5, 3, 0, 7, 6, 6, 4, 8, 6, 6, 4, 8, 7, 7, 5, 9, 8, 8, 6, 11, 9, 9, 6,
     11, 11, 11, 7, 12, 11, 11, 9, 12, 12, 12, 11, 12, 12, 12, 11, 13, 13, 13, 12, 13, 13, 13, 13, 13, 14, 13, 13,
     14, 14, 14, 13, 14, 14, 14, 14],
    [4, 0, 0, 0, 6, 4, 0, 0, 6, 5, 4, 0, 6, 5, 5, 4, 7, 5, 5, 4, 7, 5, 5, 4, 7, 6, 6, 4, 7, 6, 6, 4,
     8, 7, 7, 5, 8, 8, 7, 6, 9, 8, 8, 7, 9, 9, 8, 8, 9, 9, 9, 8, 10, 9, 9, 9, 10, 10, 10, 10,
     10, 10, 10, 10, 10, 10, 10, 10],
]
_CT_VAL = [
    [1, 0, 0, 0, 5, 1, 0, 0, 7, 4, 1, 0, 7, 6, 5, 3, 7, 6, 5, 3, 7, 6, 5, 4, 15, 6, 5, 4, 11, 14, 5, 4,
     8, 10, 13, 4, 15, 14, 9, 4, 11, 10, 13, 12, 15, 14, 9, 12, 11, 10, 13, 8, 15, 1, 9, 12, 11, 14, 13, 8,
     7, 10, 9, 12, 4, 6, 5, 8],
    [3, 0, 0, 0, 11, 2, 0, 0, 7, 7, 3, 0, 7, 10, 9, 5, 7, 6, 5, 4, 4, 6, 5, 6, 7, 6, 5, 8, 15, 6, 5, 4,
     11, 14, 13, 4, 15, 10, 9, 4, 11, 14, 13, 12, 8, 10, 9, 8, 15, 14, 13, 12, 11, 10, 9, 12, 7, 11, 6, 8,
     9, 8, 10, 1, 7, 6, 5, 4],
    [15, 0, 0, 0, 15, 14, 0, 0, 11, 15, 13, 0, 8, 12, 14, 12, 15, 10, 11, 11, 11, 8, 9, 10, 9, 14, 13, 9,
     8, 10, 9, 8, 15, 14, 13, 13, 11, 14, 10, 12, 15, 10, 13, 12, 11, 14, 9, 12, 8, 10, 13, 8, 13, 7, 9, 12,
     9, 12, 11, 10, 5, 8, 7, 6, 1, 4, 3, 2],
]
_CDC_CT_LEN = [2, 0, 0, 0, 6, 1, 0, 0, 6, 6, 3, 0, 6, 7, 7, 6, 6, 8, 8, 7]
_CDC_CT_VAL = [1, 0, 0, 0, 7, 1, 0, 0, 4, 6, 1, 0, 3, 3, 2, 5, 2, 3, 2, 0]
# total_zeros, tables 9-7 and 9-8, indexed [TotalCoeff - 1][total_zeros]
_TZ_LEN = [[1, 3, 3, 4, 4, 5, 5, 6, 6, 7, 7, 8, 8, 9, 9, 9], [3, 3, 3, 3, 3, 4, 4, 4, 4, 5, 5, 6, 6, 6, 6],
           [4, 3, 3, 3, 4, 4, 3, 3, 4, 5, 5, 6, 5, 6], [5, 3, 4, 4, 3, 3, 3, 4, 3, 4, 5, 5, 5],
           [4, 4, 4, 3, 3, 3, 3, 3, 4, 5, 4, 5], [6, 5, 3, 3, 3, 3, 3, 3, 4, 3, 6], [6, 5, 3, 3, 3, 2, 3, 4, 3, 6],
           [6, 4, 5, 3, 2, 2, 3, 3, 6], [6, 6, 4, 2, 2, 3, 2, 5], [5, 5, 3, 2, 2, 2, 4], [4, 4, 3, 3, 1, 3],
           [4, 4, 2, 1, 3], [3, 3, 1, 2], [2, 2, 1], [1, 1]]
_TZ_VAL = [[1, 3, 2, 3, 2, 3, 2, 3, 2, 3, 2, 3, 2, 3, 2, 1], [7, 6, 5, 4, 3, 5, 4, 3, 2, 3, 2, 3, 2, 1, 0],
           [5, 7, 6, 5, 4, 3, 4, 3, 2, 3, 2, 1, 1, 0], [3, 7, 5, 4, 6, 5, 4, 3, 3, 2, 2, 1, 0],
           [5, 4, 3, 7, 6, 5, 4, 3, 2, 1, 1, 0], [1, 1, 7, 6, 5, 4, 3, 2, 1, 1, 0], [1, 1, 5, 4, 3, 3, 2, 1, 1, 0],
           [1, 1, 1, 3, 3, 2, 2, 1, 0], [1, 0, 1, 3, 2, 1, 1, 1], [1, 0, 1, 3, 2, 1, 1], [0, 1, 1, 2, 1, 3],
           [0, 1, 1, 1, 1], [0, 1, 1, 1], [0, 1, 1], [0, 1]]
# total_zeros for chroma DC (table 9-9a), [TotalCoeff - 1][total_zeros]
_CDC_TZ_LEN = [[1, 2, 3, 3], [1, 2, 2], [1, 1]]
_CDC_TZ_VAL = [[1, 1, 1, 0], [1, 1, 0], [1, 0]]
# run_before (table 9-10), [min(zerosLeft, 7) - 1][run_before]
_RB_LEN = [[1, 1], [1, 2, 2], [2, 2, 2, 2], [2, 2, 2, 3, 3], [2, 2, 3, 3, 3, 3], [2, 3, 3, 3, 3, 3, 3],
           [3, 3, 3, 3, 3, 3, 3, 4, 5, 6, 7, 8, 9, 10, 11]]
_RB_VAL = [[1, 0], [1, 1, 0], [3, 2, 1, 0], [3, 2, 1, 1, 0], [3, 2, 3, 2, 1, 0], [3, 0, 1, 3, 2, 5, 4],
           [7, 6, 5, 4, 3, 2, 1, 1, 1, 1, 1, 1, 1, 1, 1]]

# ---- transform and quantisation ----
ZIGZAG = [0, 1, 4, 8, 5, 2, 3, 6, 9, 12, 13, 10, 7, 11, 14, 15]   # scan index -> raster index (4 * row + column)
MF = [[13107, 5243, 8066], [11916, 4660, 7490], [10082, 4194, 6554], [9362, 3647, 5825], [8192, 3355, 5243],
      [7282, 2893, 4559]]
V = [[10, 16, 13], [11, 18, 14], [13, 20, 16], [14, 23, 18], [16, 25, 20], [18, 29, 23]]
QPC = list(range(30)) + [29, 30, 31, 32, 32, 33, 34, 34, 35, 35, 36, 36, 37, 37, 37, 38, 38, 38, 39, 39, 39, 39]
CF = np.array([[1, 1, 1, 1], [2, 1, -1, -2], [1, -1, -1, 1], [1, -2, 2, -1]], np.int64)
H4 = np.array([[1, 1, 1, 1], [1, 1, -1, -1], [1, -1, -1, 1], [1, -1, 1, -1]], np.int64)
H2 = np.array([[1, 1], [1, -1]], np.int64)


def pos_class(r, c):
    """0 for (even, even), 1 for (odd, odd), 2 otherwise."""
    return 0 if r % 2 == 0 and c % 2 == 0 else (1 if r % 2 == 1 and c % 2 == 1 else 2)


CLASS = np.array([[pos_class(r, c) for c in range(4)] for r in range(4)])


def max_bytes(h, w):
    """Per-frame bound: each of the h / 16 slices has at most P = ceil((62 + 3200 (w / 16) + 8) / 8) bytes of RBSP
    (slice header with the NAL header byte, the macroblocks, the stop bit and alignment), at most P // 2 emulation
    prevention bytes, and the 4-byte length prefix."""
    p = (62 + MB_BITS_LIMIT * (w // 16) + 8 + 7) // 8
    return (h // 16) * (4 + p + p // 2)


class Bits:
    def __init__(self):
        self.v, self.n = 0, 0

    def put(self, v, n):
        assert 0 <= v < (1 << n) or n == 0
        self.v = (self.v << n) | v
        self.n += n

    def ue(self, k):
        m = (k + 1).bit_length() - 1
        self.put(k + 1, 2 * m + 1)

    def se(self, k):
        self.ue(2 * k - 1 if k > 0 else -2 * k)

    def extend(self, other):
        self.put(other.v, other.n)

    def trailing(self):
        self.put(1, 1)
        self.put(0, (-self.n) % 8)

    def tobytes(self):
        assert self.n % 8 == 0
        return self.v.to_bytes(self.n // 8, "big")


def emulation_prevent(rbsp):
    out, zeros = bytearray(), 0
    for b in rbsp:
        if zeros >= 2 and b <= 3:
            out.append(3)
            zeros = 0
        out.append(b)
        zeros = zeros + 1 if b == 0 else 0
    return bytes(out)


def colour(frame):
    """Y (H, W), Cb and Cr (H / 2, W / 2) of an (H, W, 3) uint8 RGB frame, as int64."""
    f = np.asarray(frame, np.int64)
    r, g, b = f[..., 0], f[..., 1], f[..., 2]
    y = ((66 * r + 129 * g + 25 * b + 128) >> 8) + 16
    s = lambda x: x[0::2, 0::2] + x[0::2, 1::2] + x[1::2, 0::2] + x[1::2, 1::2]
    rs, gs, bs = s(r), s(g), s(b)
    cb = ((-38 * rs - 74 * gs + 112 * bs + 512) >> 10) + 128
    cr = ((112 * rs - 94 * gs - 18 * bs + 512) >> 10) + 128
    return y, cb, cr


def sps(h, w):
    b = Bits()
    b.put(0x67, 8)
    b.put(66, 8)
    b.put(0xC0, 8)                        # constraint_set0_flag = constraint_set1_flag = 1
    b.put(51, 8)
    b.ue(0)                               # seq_parameter_set_id
    b.ue(0)                               # log2_max_frame_num_minus4
    b.ue(2)                               # pic_order_cnt_type
    b.ue(0)                               # max_num_ref_frames
    b.put(0, 1)                           # gaps_in_frame_num_value_allowed_flag
    b.ue(w // 16 - 1)
    b.ue(h // 16 - 1)
    b.put(1, 1)                           # frame_mbs_only_flag
    b.put(1, 1)                           # direct_8x8_inference_flag
    b.put(0, 1)                           # frame_cropping_flag
    b.put(1, 1)                           # vui_parameters_present_flag
    b.put(0, 1)                           # aspect_ratio_info_present_flag
    b.put(0, 1)                           # overscan_info_present_flag
    b.put(1, 1)                           # video_signal_type_present_flag
    b.put(5, 3)                           # video_format: unspecified
    b.put(0, 1)                           # video_full_range_flag
    b.put(1, 1)                           # colour_description_present_flag
    b.put(6, 8), b.put(6, 8), b.put(6, 8)   # SMPTE 170M primaries, transfer, matrix
    b.put(0, 1)                           # chroma_loc_info_present_flag
    b.put(0, 1)                           # timing_info_present_flag
    b.put(0, 1), b.put(0, 1)              # nal / vcl hrd
    b.put(0, 1)                           # pic_struct_present_flag
    b.put(0, 1)                           # bitstream_restriction_flag
    b.trailing()
    return emulation_prevent(b.tobytes())


def pps():
    b = Bits()
    b.put(0x68, 8)
    b.ue(0), b.ue(0)                      # pic / seq parameter set ids
    b.put(0, 1), b.put(0, 1)              # entropy_coding_mode_flag, bottom_field_pic_order_in_frame_present_flag
    b.ue(0)                               # num_slice_groups_minus1
    b.ue(0), b.ue(0)                      # num_ref_idx_l0 / l1_default_active_minus1
    b.put(0, 1), b.put(0, 2)              # weighted_pred_flag, weighted_bipred_idc
    b.se(0), b.se(0), b.se(0)             # pic_init_qp_minus26, pic_init_qs_minus26, chroma_qp_index_offset
    b.put(1, 1)                           # deblocking_filter_control_present_flag
    b.put(0, 1), b.put(0, 1)              # constrained_intra_pred_flag, redundant_pic_cnt_present_flag
    b.trailing()
    return emulation_prevent(b.tobytes())


class LevelEscape(Exception):
    """A level needs a level_prefix above 15."""


def residual_block(b, coeffs, nc, max_num):
    """CAVLC residual_block() of coeffs (scan order, len max_num) with context nC into b; returns TotalCoeff."""
    nz = [i for i, c in enumerate(coeffs) if c]
    total = len(nz)
    levels = [coeffs[i] for i in reversed(nz)]              # highest frequency first
    t1 = 0
    while t1 < min(3, total) and abs(levels[t1]) == 1:
        t1 += 1
    if nc == -1:
        b.put(_CDC_CT_VAL[4 * total + t1], _CDC_CT_LEN[4 * total + t1])
    elif nc >= 8:
        b.put(((total - 1) << 2 | t1) if total else 3, 6)
    else:
        k = 0 if nc < 2 else (1 if nc < 4 else 2)
        b.put(_CT_VAL[k][4 * total + t1], _CT_LEN[k][4 * total + t1])
    if total == 0:
        return 0
    for i in range(t1):
        b.put(1 if levels[i] < 0 else 0, 1)
    suffix = 1 if total > 10 and t1 < 3 else 0
    for i in range(t1, total):
        lv = levels[i]
        code = 2 * lv - 2 if lv > 0 else -2 * lv - 1
        if i == t1 and t1 < 3:
            code -= 2
        if suffix == 0:
            if code < 14:
                prefix, sfx, size = code, 0, 0
            elif code < 30:
                prefix, sfx, size = 14, code - 14, 4
            else:
                prefix, sfx, size = 15, code - 30, 12
        elif code < (15 << suffix):
            prefix, sfx, size = code >> suffix, code & ((1 << suffix) - 1), suffix
        else:
            prefix, sfx, size = 15, code - (15 << suffix), 12
        if sfx >= 4096:
            raise LevelEscape
        b.put(1, prefix + 1)
        b.put(sfx, size)
        if suffix == 0:
            suffix = 1
        if abs(lv) > (3 << (suffix - 1)) and suffix < 6:
            suffix += 1
    if total < max_num:
        tz = nz[-1] + 1 - total
        if nc == -1:
            b.put(_CDC_TZ_VAL[total - 1][tz], _CDC_TZ_LEN[total - 1][tz])
        else:
            b.put(_TZ_VAL[total - 1][tz], _TZ_LEN[total - 1][tz])
        left = tz
        for i in range(total - 1):
            if left <= 0:
                break
            run = nz[total - 1 - i] - nz[total - 2 - i] - 1
            t = min(left, 7) - 1
            b.put(_RB_VAL[t][run], _RB_LEN[t][run])
            left -= run
    return total


def quant(w, qp, cls):
    qbits, f = 15 + qp // 6, (1 << (15 + qp // 6)) // 3
    return np.sign(w) * ((np.abs(w) * np.array(MF[qp % 6])[cls] + f) >> qbits)


def quant_dc(d, qp):
    qbits, f = 15 + qp // 6, (1 << (15 + qp // 6)) // 3
    return np.sign(d) * ((np.abs(d) * MF[qp % 6][0] + 2 * f) >> (qbits + 1))


def idct(d):
    """8.5.12.2: rows (horizontal) first, then columns, then (x + 32) >> 6."""
    d = np.array(d, np.int64)
    def one(x):   # along the last axis
        e0, e1 = x[..., 0] + x[..., 2], x[..., 0] - x[..., 2]
        e2, e3 = (x[..., 1] >> 1) - x[..., 3], x[..., 1] + (x[..., 3] >> 1)
        return np.stack([e0 + e3, e1 + e2, e1 - e2, e0 - e3], -1)
    g = one(one(d).T).T
    return (g + 32) >> 6


def scale_ac(c, qp):
    """8.5.12.1 for the AC positions of a 4x4 block (c raster, position 0 left as is)."""
    ls = 16 * np.array(V[qp % 6])[CLASS]
    if qp >= 24:
        d = (c * ls) << (qp // 6 - 4)
    else:
        d = (c * ls + (1 << (3 - qp // 6))) >> (4 - qp // 6)
    d = d.copy()
    d[0, 0] = c[0, 0]
    return d


def encode_mb(ys, cbs, crs, left, qp, mbx):
    """One macroblock: ys (16, 16), cbs / crs (8, 8) source samples; left: the left macroblock's reconstructed right
    column and its right blocks' TotalCoeff, or None.  Returns (Bits, recon (y, cb, cr), new left, mb type)."""
    qpc = QPC[qp]
    # luma prediction
    if left is None:
        dc, use_h = 128, False
    else:
        dc = (int(left["y"].sum()) + 8) >> 4
        pred_h = np.repeat(left["y"][:, None], 16, 1)
        use_h = int(np.abs(ys - pred_h).sum()) < int(np.abs(ys - dc).sum())
    pred = pred_h if use_h else np.full((16, 16), dc, np.int64)
    # luma transform: W per 4x4 block (by, bx)
    res = ys - pred
    W = np.zeros((4, 4, 4, 4), np.int64)
    for by in range(4):
        for bx in range(4):
            W[by, bx] = CF @ res[4 * by:4 * by + 4, 4 * bx:4 * bx + 4] @ CF.T
    ac = quant(W, qp, CLASS)
    ac[:, :, 0, 0] = 0
    D = H4 @ W[:, :, 0, 0] @ H4
    dcl = np.sign(D) * quant_dc(np.abs(D) >> 1, qp)
    # chroma prediction and transform
    cpred, cac, cdcl = [], [], []
    for k, src in enumerate((cbs, crs)):
        p = np.empty((8, 8), np.int64)
        for hy in range(2):
            p[4 * hy:4 * hy + 4] = 128 if left is None else (int(left["c"][k][4 * hy:4 * hy + 4].sum()) + 2) >> 2
        cpred.append(p)
        r = src - p
        Wc = np.zeros((2, 2, 4, 4), np.int64)
        for by in range(2):
            for bx in range(2):
                Wc[by, bx] = CF @ r[4 * by:4 * by + 4, 4 * bx:4 * bx + 4] @ CF.T
        a = quant(Wc, qpc, CLASS)
        a[:, :, 0, 0] = 0
        cac.append(a)
        cdcl.append(quant_dc(H2 @ Wc[:, :, 0, 0] @ H2, qpc))
    cbp_l = 15 if ac.any() else 0
    cbp_c = 2 if (cac[0].any() or cac[1].any()) else (1 if (cdcl[0].any() or cdcl[1].any()) else 0)
    # reconstruction (8.5.10, 8.5.11, 8.5.12)
    f = H4 @ dcl @ H4
    ls0 = 16 * V[qp % 6][0]
    dcy = (f * ls0) << (qp // 6 - 6) if qp >= 36 else (f * ls0 + (1 << (5 - qp // 6))) >> (6 - qp // 6)
    ry = np.empty((16, 16), np.int64)
    for by in range(4):
        for bx in range(4):
            c = ac[by, bx].copy()
            c[0, 0] = dcy[by, bx]
            ry[4 * by:4 * by + 4, 4 * bx:4 * bx + 4] = idct(scale_ac(c, qp))
    ry = np.clip(pred + ry, 0, 255)
    rc = []
    for k in range(2):
        fc = H2 @ cdcl[k] @ H2
        dcc = ((fc * 16 * V[qpc % 6][0]) << (qpc // 6)) >> 5
        r = np.empty((8, 8), np.int64)
        for by in range(2):
            for bx in range(2):
                c = cac[k][by, bx].copy()
                c[0, 0] = dcc[by, bx]
                r[4 * by:4 * by + 4, 4 * bx:4 * bx + 4] = idct(scale_ac(c, qpc))
        rc.append(np.clip(cpred[k] + r, 0, 255))
    # macroblock_layer()
    b = Bits()
    b.ue(1 + (1 if use_h else 2) + 4 * cbp_c + 12 * (cbp_l == 15))
    b.ue(0)                                               # intra_chroma_pred_mode: DC
    b.se(0)                                               # mb_qp_delta
    tc = np.zeros((4, 4), np.int64)                       # TotalCoeff of each luma 4x4 block (AC)
    ctc = np.zeros((2, 2, 2), np.int64)

    def nc_of(grid, lgrid, by, bx):
        a = grid[by, bx - 1] if bx > 0 else (lgrid[by] if left is not None else None)
        t = grid[by - 1, bx] if by > 0 else None
        if a is not None and t is not None:
            return (int(a) + int(t) + 1) >> 1
        return int(a) if a is not None else (int(t) if t is not None else 0)

    try:
        residual_block(b, [int(dcl.reshape(16)[z]) for z in ZIGZAG], nc_of(tc, left["nz"] if left else None, 0, 0), 16)
        if cbp_l:
            for blk in range(16):                         # luma4x4BlkIdx order
                by = 2 * (blk // 8) + (blk % 4) // 2
                bx = 2 * ((blk // 4) % 2) + blk % 2
                sc = [int(ac[by, bx].reshape(16)[z]) for z in ZIGZAG[1:]]
                tc[by, bx] = residual_block(b, sc, nc_of(tc, left["nz"] if left else None, by, bx), 15)
        if cbp_c:
            for k in range(2):
                residual_block(b, [int(x) for x in cdcl[k].reshape(4)], -1, 4)
        if cbp_c == 2:
            for k in range(2):
                for blk in range(4):
                    by, bx = blk // 2, blk % 2
                    sc = [int(cac[k][by, bx].reshape(16)[z]) for z in ZIGZAG[1:]]
                    ctc[k, by, bx] = residual_block(b, sc, nc_of(ctc[k], left["cnz"][k] if left else None, by, bx),
                                                    15)
        escape = False
    except LevelEscape:
        escape = True
    if escape or b.n > MB_BITS_LIMIT:
        return None, (ys, cbs, crs), {"y": ys[:, 15], "c": (cbs[:, 7], crs[:, 7]), "nz": np.full(4, 16),
                                      "cnz": (np.full(2, 16), np.full(2, 16))}, PCM
    return b, (ry, rc[0], rc[1]), {"y": ry[:, 15], "c": (rc[0][:, 7], rc[1][:, 7]), "nz": tc[:, 3],
                                   "cnz": (ctc[0][:, 1], ctc[1][:, 1])}, ("H" if use_h else "DC")


def slice_header(first_mb, idr_pic_id, qp):
    b = Bits()
    b.put(0x65, 8)                        # nal_ref_idc 3, nal_unit_type 5 (IDR)
    b.ue(first_mb)
    b.ue(7)                               # slice_type: I, every slice of the picture
    b.ue(0)                               # pic_parameter_set_id
    b.put(0, 4)                           # frame_num
    b.ue(idr_pic_id)
    b.put(0, 1), b.put(0, 1)              # no_output_of_prior_pics_flag, long_term_reference_flag
    b.se(qp - 26)                         # slice_qp_delta
    b.ue(1)                               # disable_deblocking_filter_idc
    return b


def check_shape(h, w):
    if h % 16 or w % 16 or h < 16 or w < 16:
        raise ValueError(f"H and W must be positive multiples of 16, got {h} x {w}")
    if (h // 16) * (w // 16) > MAX_FS or h // 16 > MAX_DIM_MBS or w // 16 > MAX_DIM_MBS:
        raise ValueError(f"a {h} x {w} frame passes level 5.1's frame size")


def encode(frame, qp=20, index=0):
    """The sample (length-prefixed slices) of one (H, W, 3) uint8 frame at position `index` of its clip.  Returns
    (bytes, recon (Y, Cb, Cr) int64, mb types (H / 16, W / 16) of 'DC', 'H' or 'PCM')."""
    frame = np.asarray(frame)
    h, w, _ = frame.shape
    check_shape(h, w)
    y, cb, cr = colour(frame)
    ry, rcb, rcr = np.empty_like(y), np.empty_like(cb), np.empty_like(cr)
    types = np.empty((h // 16, w // 16), object)
    out = bytearray()
    for my in range(h // 16):
        b = slice_header(my * (w // 16), index % 2, qp)
        left = None
        for mx in range(w // 16):
            sy, sx = slice(16 * my, 16 * my + 16), slice(16 * mx, 16 * mx + 16)
            cy, cx = slice(8 * my, 8 * my + 8), slice(8 * mx, 8 * mx + 8)
            bits, rec, left, t = encode_mb(y[sy, sx], cb[cy, cx], cr[cy, cx], left, qp, mx)
            if bits is None:
                b.ue(25)
                b.put(0, (-b.n) % 8)
                for plane in rec:
                    for v in plane.reshape(-1):
                        b.put(int(v), 8)
            else:
                b.extend(bits)
            ry[sy, sx], rcb[cy, cx], rcr[cy, cx] = rec
            types[my, mx] = t
        b.trailing()
        nal = emulation_prevent(b.tobytes())
        out += len(nal).to_bytes(4, "big") + nal
    assert len(out) <= max_bytes(h, w)
    return bytes(out), (ry, rcb, rcr), types

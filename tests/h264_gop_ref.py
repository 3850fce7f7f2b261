"""CPU restatement of the H.264 GOP rule of pantomatrix_b200.video (DESIGN.md section 12): an IDR frame every `gop`
frames, P frames between them, shared by the CPU and GPU tests.  The intra rule (IDR frames, Intra16x16 and I_PCM
macroblocks, CAVLC, framing) is oracle/h264_oracle.py's, called as it is; this module adds what P frames need:
  - the P slice header (nal_ref_idc 2, nal_unit_type 1, slice_type 5, frame_num = (t mod gop) mod 16);
  - the zero-motion inter candidate: the full 4x4 transform of source - reference, quantised with f = 2^qbits / 6,
    computed for a whole frame at once, and the P_Skip test on it;
  - the decision (P_Skip, else inter when its luma SAD <= the Intra16x16 candidate's, else Intra16x16 with
    mb_type + 5), I_PCM as mb_type 30, mb_skip_run, the Table 9-4 Inter cbp mapping and the inter reconstruction.
encode_clip(frames, qp, 1) is oracle.h264_oracle.encode per frame."""
from __future__ import annotations

import numpy as np

from oracle import h264_oracle as O

SKIP, INTER = "SKIP", "P"
MB_BITS_LIMIT_P = O.MB_BITS_LIMIT + 1         # a coded macroblock and its ue(mb_skip_run): every skipped macroblock
SLICE_HEADER_BITS_GOP = 70                    # the longest slice header of either kind (IDR at qp 0, last row)
# Table 9-4, ChromaArrayType 1: coded_block_pattern of each codeNum for Inter macroblocks; INTER_CODE is its inverse
INTER_CBP = [0, 16, 1, 2, 4, 8, 32, 3, 5, 10, 12, 15, 47, 7, 11, 13, 14, 6, 9, 31, 35, 37, 42, 44, 33, 34, 36, 40,
             39, 43, 45, 46, 17, 18, 20, 24, 19, 21, 26, 28, 23, 27, 29, 30, 22, 25, 38, 41]
INTER_CODE = [INTER_CBP.index(c) for c in range(48)]
LUMA_BLK = [(2 * (b // 8) + (b % 4) // 2, 2 * ((b // 4) % 2) + b % 2) for b in range(16)]   # luma4x4BlkIdx -> by, bx


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


def _blocks(p, n):
    """(H, W) -> (H / n, W / n, n, n)."""
    h, w = p.shape
    return p.reshape(h // n, n, w // n, n).swapaxes(1, 2)


def _fdct(blk):
    """The 4x4 forward core transform of every block of (..., 4, 4)."""
    return np.einsum("ij,...jk,lk->...il", O.CF, blk, O.CF)


def _quant_inter(w, q):
    qbits = 15 + q // 6
    f = (1 << qbits) // 6
    return np.sign(w) * ((np.abs(w) * np.array(O.MF[q % 6])[O.CLASS] + f) >> qbits)


def inter_levels(cur, ref, qp):
    """The zero-motion inter candidate of a whole frame: cur, ref = (Y, Cb, Cr) int64 planes.  Returns luma levels
    (H/16, W/16, 4, 4, 4, 4) by (block row, block column, raster), chroma AC levels (2, H/16, W/16, 2, 2, 4, 4) with
    position 0 zero, chroma DC levels (2, H/16, W/16, 2, 2), and the P_Skip mask (H/16, W/16)."""
    qpc = O.QPC[qp]
    y = _fdct(_blocks(cur[0] - ref[0], 4))
    mbh, mbw = y.shape[0] // 4, y.shape[1] // 4
    ly = _quant_inter(y, qp).reshape(mbh, 4, mbw, 4, 4, 4).swapaxes(1, 2)
    cac, cdc = [], []
    for k in (1, 2):
        c = _fdct(_blocks(cur[k] - ref[k], 4)).reshape(mbh, 2, mbw, 2, 4, 4).swapaxes(1, 2)
        a = _quant_inter(c, qpc)
        a[..., 0, 0] = 0
        cac.append(a)
        d = np.einsum("ij,...jk,kl->...il", O.H2, c[..., 0, 0], O.H2)
        qbits = 15 + qpc // 6
        f = (1 << qbits) // 6
        cdc.append(np.sign(d) * ((np.abs(d) * O.MF[qpc % 6][0] + 2 * f) >> (qbits + 1)))
    cac, cdc = np.stack(cac), np.stack(cdc)
    skip = ~(ly.any((2, 3, 4, 5)) | cac.any((0, 3, 4, 5, 6)) | cdc.any((0, 3, 4)))
    return ly, cac, cdc, skip


def _scale_all(c, qp):
    """8.5.12.1 for all 16 positions of a 4x4 block of an inter macroblock (raster)."""
    ls = 16 * np.array(O.V[qp % 6])[O.CLASS]
    if qp >= 24:
        return (c * ls) << (qp // 6 - 4)
    return (c * ls + (1 << (3 - qp // 6))) >> (4 - qp // 6)


def encode_inter_mb(ly, cac, cdc, ref, left, qp):
    """One P_L0_16x16 macroblock with mvd (0, 0): ly (4, 4, 4, 4), cac (2, 2, 2, 4, 4), cdc (2, 2, 2) its levels,
    ref (y (16, 16), cb, cr (8, 8)) its prediction, left as in oracle.h264_oracle.encode_mb.  Returns (Bits of its
    macroblock_layer() or None for a level escape, recon, new left)."""
    qpc = O.QPC[qp]
    cbp_l = sum(1 << b8 for b8 in range(4) if ly[2 * (b8 // 2):2 * (b8 // 2) + 2, 2 * (b8 % 2):2 * (b8 % 2) + 2].any())
    cbp_c = 2 if cac.any() else (1 if cdc.any() else 0)
    ry = np.empty((16, 16), np.int64)
    for by in range(4):
        for bx in range(4):
            ry[4 * by:4 * by + 4, 4 * bx:4 * bx + 4] = O.idct(_scale_all(ly[by, bx], qp))
    ry = np.clip(ref[0] + ry, 0, 255)
    rc = []
    for k in range(2):
        fc = O.H2 @ cdc[k] @ O.H2
        dcc = ((fc * 16 * O.V[qpc % 6][0]) << (qpc // 6)) >> 5
        r = np.empty((8, 8), np.int64)
        for by in range(2):
            for bx in range(2):
                c = cac[k][by, bx].copy()
                c[0, 0] = dcc[by, bx]
                r[4 * by:4 * by + 4, 4 * bx:4 * bx + 4] = O.idct(O.scale_ac(c, qpc))
        rc.append(np.clip(ref[1 + k] + r, 0, 255))
    b = O.Bits()
    b.ue(0)                                               # mb_type P_L0_16x16
    b.se(0), b.se(0)                                      # mvd_l0 (0, 0): the predictor is (0, 0)
    b.ue(INTER_CODE[cbp_l | cbp_c << 4])
    tc = np.zeros((4, 4), np.int64)
    ctc = np.zeros((2, 2, 2), np.int64)

    def nc_of(grid, lgrid, by, bx):
        a = grid[by, bx - 1] if bx > 0 else (lgrid[by] if left is not None else None)
        t = grid[by - 1, bx] if by > 0 else None
        if a is not None and t is not None:
            return (int(a) + int(t) + 1) >> 1
        return int(a) if a is not None else (int(t) if t is not None else 0)

    try:
        if cbp_l or cbp_c:
            b.se(0)                                       # mb_qp_delta
        for blk in range(16):
            by, bx = LUMA_BLK[blk]
            if cbp_l >> ((by // 2) * 2 + bx // 2) & 1:
                sc = [int(ly[by, bx].reshape(16)[z]) for z in O.ZIGZAG]
                tc[by, bx] = O.residual_block(b, sc, nc_of(tc, left["nz"] if left else None, by, bx), 16)
        if cbp_c:
            for k in range(2):
                O.residual_block(b, [int(x) for x in cdc[k].reshape(4)], -1, 4)
        if cbp_c == 2:
            for k in range(2):
                for blk in range(4):
                    by, bx = blk // 2, blk % 2
                    sc = [int(cac[k][by, bx].reshape(16)[z]) for z in O.ZIGZAG[1:]]
                    ctc[k, by, bx] = O.residual_block(b, sc, nc_of(ctc[k], left["cnz"][k] if left else None, by, bx),
                                                      15)
    except O.LevelEscape:
        b = None
    return b, (ry, rc[0], rc[1]), {"y": ry[:, 15], "c": (rc[0][:, 7], rc[1][:, 7]), "nz": tc[:, 3],
                                   "cnz": (ctc[0][:, 1], ctc[1][:, 1])}


def _intra_sad(ys, left):
    """The SAD of today's Intra16x16 luma choice: DC, or Horizontal when its SAD is strictly lower."""
    if left is None:
        return int(np.abs(ys - 128).sum())
    dc = (int(left["y"].sum()) + 8) >> 4
    return min(int(np.abs(ys - dc).sum()), int(np.abs(ys - left["y"][:, None]).sum()))


def _ue_len(k):
    return 2 * (k + 1).bit_length() - 1


def encode_p(frame, ref, qp, frame_num):
    """The sample of one P frame against ref (Y, Cb, Cr).  Returns (bytes, recon, mb types)."""
    frame = np.asarray(frame)
    h, w, _ = frame.shape
    cur = O.colour(frame)
    ly, cac, cdc, skip = inter_levels(cur, ref, qp)
    rec = tuple(p.copy() for p in ref)
    types = np.empty((h // 16, w // 16), object)
    out = bytearray()
    for my in range(h // 16):
        b = p_slice_header(my * (w // 16), frame_num, qp)
        left, run = None, 0
        for mx in range(w // 16):
            sy, sx = slice(16 * my, 16 * my + 16), slice(16 * mx, 16 * mx + 16)
            cy, cx = slice(8 * my, 8 * my + 8), slice(8 * mx, 8 * mx + 8)
            src = (cur[0][sy, sx], cur[1][cy, cx], cur[2][cy, cx])
            pred = (ref[0][sy, sx], ref[1][cy, cx], ref[2][cy, cx])
            if skip[my, mx]:
                run += 1
                types[my, mx] = SKIP
                left = {"y": pred[0][:, 15], "c": (pred[1][:, 7], pred[2][:, 7]), "nz": np.zeros(4, np.int64),
                        "cnz": (np.zeros(2, np.int64), np.zeros(2, np.int64))}
                continue
            if int(np.abs(src[0] - pred[0]).sum()) <= _intra_sad(src[0], left):
                bits, r, new_left = encode_inter_mb(ly[my, mx], cac[:, my, mx], cdc[:, my, mx], pred, left, qp)
                t = INTER
            else:
                bits, r, new_left, t = O.encode_mb(src[0], src[1], src[2], left, qp, mx)
                if bits is not None:                      # mb_type ue(m) -> ue(m + 5)
                    lead = bits.n - bits.v.bit_length()  # the leading zeros of ue(m)
                    m = (bits.v >> (bits.n - 2 * lead - 1)) - 1
                    rest = bits.n - 2 * lead - 1
                    nb = O.Bits()
                    nb.ue(m + 5)
                    nb.put(bits.v & ((1 << rest) - 1), rest)
                    bits = nb
            b.ue(run)
            run = 0
            if bits is None or bits.n > O.MB_BITS_LIMIT:
                b.ue(30)                                  # I_PCM in a P slice, then pcm_alignment_zero_bits
                b.put(0, (-b.n) % 8)
                for plane in src:
                    for v in plane.reshape(-1):
                        b.put(int(v), 8)
                r, t = src, O.PCM
                new_left = {"y": src[0][:, 15], "c": (src[1][:, 7], src[2][:, 7]), "nz": np.full(4, 16),
                            "cnz": (np.full(2, 16), np.full(2, 16))}
            else:
                b.extend(bits)
            rec[0][sy, sx], rec[1][cy, cx], rec[2][cy, cx] = r
            types[my, mx], left = t, new_left
        if run:
            b.ue(run)
        b.trailing()
        nal = O.emulation_prevent(b.tobytes())
        out += len(nal).to_bytes(4, "big") + nal
    return bytes(out), rec, types


def encode_clip(frames, qp=20, gop=1):
    """The samples of one clip (a list of (H, W, 3) uint8 frames): frame t is IDR when t mod gop == 0 (idr_pic_id =
    (t div gop) mod 2, oracle.h264_oracle.encode), else a P frame against frame t - 1's reconstruction.  Returns a list
    of (bytes, recon (Y, Cb, Cr) int64, mb types of 'DC', 'H', 'PCM', 'P' or 'SKIP') per frame."""
    out = []
    for t, f in enumerate(frames):
        if t % gop == 0:
            out.append(O.encode(f, qp, t // gop))
        else:
            out.append(encode_p(f, out[-1][1], qp, (t % gop) % 16))
        h, w = out[-1][1][0].shape
        assert len(out[-1][0]) <= max_bytes(h, w, gop)
    return out

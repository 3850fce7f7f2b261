"""CPU restatement of the H.264 Intra 4x4 rule of pantomatrix_b200.video (encode(..., intra4x4=True), DESIGN.md
section 12), shared by the CPU and GPU tests.  Everything but Intra 4x4 is tests/h264_me_ref.py's and
tests/h264_gop_ref.py's rule, called as it is (and through them oracle/h264_oracle.py's); this module adds:
  - the I_NxN candidate of every macroblock: its 16 blocks in luma4x4BlkIdx order, each predicted by the 8.3.1.2
    mode of the lowest J = SAD + lambda(qp) (1 when the mode is predIntra4x4PredMode, else 4) among the modes its
    available samples define (ties to the lower mode), its residual transformed, quantised with f = 2^qbits / 3 at
    all 16 positions and reconstructed before the next block is predicted; computed for the macroblocks of one column
    of every row at once, since each row is its own slice;
  - the choice: I_NxN when J4 + C_I4 lambda < J16 (J4 the sum of the blocks' J, J16 the Intra16x16 candidate's SAD);
    in P slices the inter candidate when its luma SAD is <= min(J16, J4 + C_I4 lambda);
  - the I_NxN macroblock_layer(): mb_type 0 (I slice) or 5 (P slice), the 16 mode flags, intra_chroma_pred_mode 0,
    coded_block_pattern by Table 9-4's Intra column, mb_qp_delta when it is non-zero, residual_block(..., 16) for each
    block of a coded 8x8 block, then the chroma as an Intra16x16 macroblock codes it; I_PCM past 3200 bits or on a
    level escape.
encode_clip(frames, qp, gop, rng) returns per frame (bytes, recon (Y, Cb, Cr), mb types, Intra 4x4 modes
(H / 16, W / 16, 4, 4) by block row and column, -1 outside I_NxN macroblocks, vectors or None)."""
from __future__ import annotations

import numpy as np

import h264_gop_ref as G
import h264_me_ref as M
from oracle import h264_oracle as O

I4 = "I4"
C_I4 = 6                                      # the macroblock choice's constant c, in units of lambda(qp)
# Table 9-4 (ChromaArrayType 1): coded_block_pattern of each codeNum for Intra_4x4 macroblocks; INTRA_CODE inverts it
INTRA_CBP = [47, 31, 15, 0, 23, 27, 29, 30, 7, 11, 13, 14, 39, 43, 45, 46, 16, 3, 5, 10, 12, 19, 21, 26, 28, 35, 37,
             42, 44, 1, 2, 4, 8, 17, 18, 20, 24, 6, 9, 22, 25, 32, 33, 34, 36, 40, 38, 41]
INTRA_CODE = [INTRA_CBP.index(c) for c in range(48)]
BLK_OF = {rc: b for b, rc in enumerate(G.LUMA_BLK)}          # (by, bx) -> luma4x4BlkIdx


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


def _idct(d):
    """oracle.h264_oracle.idct of every block of (..., 4, 4)."""
    def one(x):
        e0, e1 = x[..., 0] + x[..., 2], x[..., 0] - x[..., 2]
        e2, e3 = (x[..., 1] >> 1) - x[..., 3], x[..., 1] + (x[..., 3] >> 1)
        return np.stack([e0 + e3, e1 + e2, e1 - e2, e0 - e3], -1)
    return (one(one(d).swapaxes(-1, -2)).swapaxes(-1, -2) + 32) >> 6


def i4_candidate(src, ly, lmode, have_left, qp):
    """The I_NxN candidate of n macroblocks of one column: src (n, 16, 16) luma, ly (n, 16) the left macroblock's
    reconstructed right column (unused without have_left), lmode (n, 4) the modes of the left macroblock's right
    blocks (2 where it is not I_NxN).  Returns J4 (n,), recon (n, 16, 16), modes and predicted modes (n, 4, 4), levels
    (n, 4, 4, 16) in scan order by block row and column, TotalCoeff (n, 4, 4)."""
    n = src.shape[0]
    lmb = M.LAMBDA[qp]
    rec = np.zeros((n, 16, 16), np.int64)
    modes, predm = np.zeros((n, 4, 4), np.int64), np.zeros((n, 4, 4), np.int64)
    lev, tc = np.zeros((n, 4, 4, 16), np.int64), np.zeros((n, 4, 4), np.int64)
    j4 = np.zeros(n, np.int64)
    for by, bx in G.LUMA_BLK:
        ys, xs = slice(4 * by, 4 * by + 4), slice(4 * bx, 4 * bx + 4)
        la, ua = bx > 0 or have_left, by > 0
        left = rec[:, ys, 4 * bx - 1] if bx > 0 else (ly[:, 4 * by:4 * by + 4] if have_left else None)
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
            ma = modes[:, by, bx - 1] if bx > 0 else lmode[:, by]
            pm = np.minimum(ma, modes[:, by - 1, bx])
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
        w = G._fdct(src[:, ys, xs] - pred)
        q = O.quant(w, qp, O.CLASS)
        rec[:, ys, xs] = np.clip(pred + _idct(G._scale_all(q, qp)), 0, 255)
        modes[:, by, bx], predm[:, by, bx] = best, pm
        lev[:, by, bx] = q.reshape(n, 16)[:, O.ZIGZAG]
        tc[:, by, bx] = (q != 0).sum((1, 2))
    return j4, rec, modes, predm, lev, tc


def _chroma(cbs, crs, left, qp):
    """The chroma of an intra macroblock as oracle.h264_oracle.encode_mb codes it: DC prediction from the left
    macroblock's reconstructed right columns.  Returns AC levels (2, 2, 2, 4, 4), DC levels (2, 2, 2), recon."""
    qpc = O.QPC[qp]
    cac, cdc, rc = [], [], []
    for k, src in enumerate((cbs, crs)):
        p = np.empty((8, 8), np.int64)
        for hy in range(2):
            p[4 * hy:4 * hy + 4] = 128 if left is None else (int(left["c"][k][4 * hy:4 * hy + 4].sum()) + 2) >> 2
        w = G._fdct(G._blocks(src - p, 4))
        a = O.quant(w, qpc, O.CLASS)
        a[..., 0, 0] = 0
        d = O.quant_dc(O.H2 @ w[..., 0, 0] @ O.H2, qpc)
        fc = O.H2 @ d @ O.H2
        c = a.copy()
        c[..., 0, 0] = ((fc * 16 * O.V[qpc % 6][0]) << (qpc // 6)) >> 5
        r = np.empty((8, 8), np.int64)
        for by in range(2):
            for bx in range(2):
                r[4 * by:4 * by + 4, 4 * bx:4 * bx + 4] = O.idct(O.scale_ac(c[by, bx], qpc))
        cac.append(a), cdc.append(d), rc.append(np.clip(p + r, 0, 255))
    return np.stack(cac), np.stack(cdc), rc


def encode_i4_mb(modes, predm, lev, tc, ry, cbs, crs, left, qp, pslice):
    """One I_NxN macroblock from i4_candidate's outputs for it.  Returns (Bits of its macroblock_layer() or None for a
    level escape, recon, new left as oracle.h264_oracle.encode_mb's)."""
    cac, cdc, rc = _chroma(cbs, crs, left, qp)
    cbp_l = sum(1 << b8 for b8 in range(4) if tc[2 * (b8 // 2):2 * (b8 // 2) + 2, 2 * (b8 % 2):2 * (b8 % 2) + 2].any())
    cbp_c = 2 if cac.any() else (1 if cdc.any() else 0)
    b = O.Bits()
    b.ue(5 if pslice else 0)                              # mb_type I_NxN
    for by, bx in G.LUMA_BLK:
        m, pm = int(modes[by, bx]), int(predm[by, bx])
        if m == pm:
            b.put(1, 1)                                   # prev_intra4x4_pred_mode_flag
        else:
            b.put(0, 1)
            b.put(m if m < pm else m - 1, 3)              # rem_intra4x4_pred_mode
    b.ue(0)                                               # intra_chroma_pred_mode: DC
    b.ue(INTRA_CODE[cbp_l | cbp_c << 4])
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
            by, bx = G.LUMA_BLK[blk]
            if cbp_l >> ((by // 2) * 2 + bx // 2) & 1:
                O.residual_block(b, [int(v) for v in lev[by, bx]], nc_of(tc, left["nz"] if left else None, by, bx), 16)
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


def encode_frame(frame, ref, qp, t, gop, rng, c=C_I4):
    """The sample of frame t of its clip: IDR when ref is None, else a P frame against ref (Y, Cb, Cr) with search
    range rng.  Returns (bytes, recon, mb types, Intra 4x4 modes, vectors or None)."""
    frame = np.asarray(frame)
    h, w, _ = frame.shape
    mbh, mbw = h // 16, w // 16
    cur = O.colour(frame)
    lmb = M.LAMBDA[qp]
    pf = ref is not None
    if pf:
        mv = M.search(cur[0], ref[0], qp, rng)
        m = rng + 8
        pred = (M._frame(M.luma_pred(M.luma_phases(ref[0], m), m, mv)) if rng else ref[0],
                M._frame(M.chroma_pred(ref[1], mv)), M._frame(M.chroma_pred(ref[2], mv)))
        skip = G.inter_levels(cur, ref, qp)[3]
        ly, cac, cdc, _ = G.inter_levels(cur, pred, qp)
        coded_mv = np.zeros((mbh, mbw, 2), np.int64)
    rec = tuple(np.zeros_like(p) for p in cur)
    types = np.empty((mbh, mbw), object)
    all_modes = np.full((mbh, mbw, 4, 4), -1, np.int64)
    bits = [G.p_slice_header(my * mbw, (t % gop) % 16, qp) if pf else O.slice_header(my * mbw, (t // gop) % 2, qp)
            for my in range(mbh)]
    lefts, runs = [None] * mbh, [0] * mbh
    mvps = np.zeros((mbh, 2), np.int64)
    lmode = np.full((mbh, 4), 2, np.int64)
    ysrc = cur[0].reshape(mbh, 16, mbw, 16)
    for mx in range(mbw):
        lcol = np.stack([l["y"] if l is not None else np.zeros(16, np.int64) for l in lefts])
        j4, r4, modes, predm, lev, tc = i4_candidate(ysrc[:, :, mx], lcol, lmode, mx > 0, qp)
        for my in range(mbh):
            b, left = bits[my], lefts[my]
            sy, sx = slice(16 * my, 16 * my + 16), slice(16 * mx, 16 * mx + 16)
            cy, cx = slice(8 * my, 8 * my + 8), slice(8 * mx, 8 * mx + 8)
            src = (cur[0][sy, sx], cur[1][cy, cx], cur[2][cy, cx])
            if pf and skip[my, mx]:
                runs[my] += 1
                types[my, mx] = G.SKIP
                col = (ref[0][sy, sx], ref[1][cy, cx], ref[2][cy, cx])
                rec[0][sy, sx], rec[1][cy, cx], rec[2][cy, cx] = col
                lefts[my] = {"y": col[0][:, 15], "c": (col[1][:, 7], col[2][:, 7]), "nz": np.zeros(4, np.int64),
                             "cnz": (np.zeros(2, np.int64), np.zeros(2, np.int64))}
                mvps[my] = 0
                lmode[my] = 2
                continue
            j_intra = G._intra_sad(src[0], left)
            i4 = j4[my] + c * lmb < j_intra
            if i4:
                j_intra = int(j4[my] + c * lmb)
            inter = False
            if pf:
                p = (pred[0][sy, sx], pred[1][cy, cx], pred[2][cy, cx])
                inter = int(np.abs(src[0] - p[0]).sum()) <= j_intra
            if inter:
                mb, r, new_left = G.encode_inter_mb(ly[my, mx], cac[:, my, mx], cdc[:, my, mx], p, left, qp)
                if mb is not None:
                    mb = M._with_mvd(mb, mv[my, mx] - mvps[my])
                kind = G.INTER
            elif i4:
                mb, r, new_left = encode_i4_mb(modes[my], predm[my], lev[my], tc[my], r4[my], src[1], src[2], left,
                                               qp, pf)
                kind = I4
            else:
                mb, r, new_left, kind = O.encode_mb(src[0], src[1], src[2], left, qp, mx)
                if mb is not None and pf:
                    mb = M._intra_p(mb)
            if pf:
                b.ue(runs[my])
                runs[my] = 0
            if mb is None or mb.n > O.MB_BITS_LIMIT:
                b.ue(30 if pf else 25)                    # I_PCM, then pcm_alignment_zero_bits
                b.put(0, (-b.n) % 8)
                for plane in src:
                    for v in plane.reshape(-1):
                        b.put(int(v), 8)
                r, kind = src, O.PCM
                new_left = {"y": src[0][:, 15], "c": (src[1][:, 7], src[2][:, 7]), "nz": np.full(4, 16),
                            "cnz": (np.full(2, 16), np.full(2, 16))}
            else:
                b.extend(mb)
            if pf:
                mvps[my] = mv[my, mx] if kind == G.INTER else 0
                if kind == G.INTER:
                    coded_mv[my, mx] = mv[my, mx]
            lmode[my] = modes[my, :, 3] if kind == I4 else 2
            if kind == I4:
                all_modes[my, mx] = modes[my]
            rec[0][sy, sx], rec[1][cy, cx], rec[2][cy, cx] = r
            types[my, mx], lefts[my] = kind, new_left
    out = bytearray()
    for my in range(mbh):
        b = bits[my]
        if runs[my]:
            b.ue(runs[my])
        b.trailing()
        nal = O.emulation_prevent(b.tobytes())
        out += len(nal).to_bytes(4, "big") + nal
    return bytes(out), rec, types, all_modes, coded_mv if pf else None


def encode_clip(frames, qp=20, gop=1, rng=0, c=C_I4):
    """The samples of one clip with Intra 4x4 on: keyframe interval gop and search range rng as
    h264_me_ref.encode_clip.  Returns a list of (bytes, recon (Y, Cb, Cr), mb types ('DC', 'H', 'I4', 'PCM', 'P',
    'SKIP'), Intra 4x4 modes (H / 16, W / 16, 4, 4), vectors or None) per frame."""
    out = []
    for t, f in enumerate(frames):
        ref = None if t % gop == 0 else out[-1][1]
        out.append(encode_frame(f, ref, qp, t, gop, rng, c))
        h, w = out[-1][1][0].shape
        assert len(out[-1][0]) <= G.max_bytes(h, w, gop)
    return out

"""CPU restatement of the H.264 motion search rule of pantomatrix_b200.video (encode(..., gop > 1, search > 0),
DESIGN.md section 12), shared by the CPU and GPU tests.  Everything but the motion is tests/h264_gop_ref.py's rule,
called as it is (and through it oracle/h264_oracle.py's); this module adds:
  - lambda(qp) = floor(sqrt(0.85 2^((qp - 12) / 3)) + 0.5), as the 52 integers LAMBDA;
  - the integer search: J = SAD_Y + lambda (b(mvx) + b(mvy)) of every whole-pixel vector within +-search whose block
    lies inside the frame, one shifted-frame SAD per candidate for a whole frame at once; lowest J, then the smaller
    |mvx| + |mvy|, then mvy, then mvx;
  - the sub-pel refinement: the 8 neighbours at +-2 quarter-pels of the integer winner, then at +-1 of the half-pel
    winner, in raster order, each replacing the centre only when its J is strictly lower; the luma prediction of
    8.4.2.2.1 computed for the whole padded frame once per quarter-pel phase, the chroma of 8.4.2.2.2 per macroblock;
  - the decision: P_Skip by the zero-motion candidate as before, else the inter candidate at the searched vector,
    P_L0_16x16 with mvd = mv - mvp (mvp: the left macroblock's vector when it is P_L0_16x16, else (0, 0)) when its luma
    SAD is <= the Intra16x16 candidate's.
encode_clip(frames, qp, gop, 0) is h264_gop_ref.encode_clip(frames, qp, gop) byte for byte."""
from __future__ import annotations

import math

import numpy as np

import h264_gop_ref as G
from oracle import h264_oracle as O

LAMBDA = [0, 0, 0, 0, 0, 0, 0, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 2, 2, 2, 2, 3, 3, 3, 4, 4, 5, 5, 6, 7, 7, 8, 9, 10, 12, 13,
          15, 17, 19, 21, 23, 26, 30, 33, 37, 42, 47, 53, 59, 66, 74, 83]


def lam(qp):
    """lambda(qp) from its formula, in float64."""
    return math.floor(math.sqrt(0.85 * 2.0 ** ((qp - 12) / 3)) + 0.5)


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
    r = n * my[..., None, None] + np.arange(n)[:, None]
    c = n * mx[..., None, None] + np.arange(n)[None, :]
    return r, c


def luma_pred(phases, m, mv):
    """The luma prediction (mbh, mbw, 16, 16) of every macroblock at its quarter-pel vector mv (mbh, mbw, 2) (x, y)."""
    mbh, mbw = mv.shape[:2]
    r, c = _mb_grid(mbh, mbw, 16)
    vx, vy = mv[..., 0][..., None, None], mv[..., 1][..., None, None]
    return phases[vy & 3, vx & 3, m + r + (vy >> 2), m + c + (vx >> 2)]


def chroma_pred(plane, mv):
    """8.4.2.2.2: the (mbh, mbw, 8, 8) chroma prediction of one plane, the luma vector in eighth chroma samples."""
    mbh, mbw = mv.shape[:2]
    hc, wc = plane.shape
    r, c = _mb_grid(mbh, mbw, 8)
    vx, vy = mv[..., 0][..., None, None], mv[..., 1][..., None, None]
    x, y, fx, fy = c + (vx >> 3), r + (vy >> 3), vx & 7, vy & 7
    at = lambda dy, dx: plane[np.clip(y + dy, 0, hc - 1), np.clip(x + dx, 0, wc - 1)]
    return ((8 - fx) * (8 - fy) * at(0, 0) + fx * (8 - fy) * at(0, 1) + (8 - fx) * fy * at(1, 0) + fx * fy * at(1, 1)
            + 32) >> 6


def _frame(blocks):
    """(mbh, mbw, n, n) -> (mbh n, mbw n)."""
    mbh, mbw, n, _ = blocks.shape
    return blocks.swapaxes(1, 2).reshape(mbh * n, mbw * n)


def search(cur_y, ref_y, qp, rng):
    """The searched quarter-pel vector (mbh, mbw, 2) (x, y) of every macroblock of cur_y against ref_y."""
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
    if rng == 0:
        return best
    phases = luma_phases(ref_y, m)
    src = cur_y.reshape(mbh, 16, mbw, 16).swapaxes(1, 2)
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


def _intra_p(bits):
    """An Intra16x16 macroblock_layer() of an I slice with mb_type ue(m) recoded as ue(m + 5) for a P slice."""
    lead = bits.n - bits.v.bit_length()
    m = (bits.v >> (bits.n - 2 * lead - 1)) - 1
    rest = bits.n - 2 * lead - 1
    nb = O.Bits()
    nb.ue(m + 5)
    nb.put(bits.v & ((1 << rest) - 1), rest)
    return nb


def _with_mvd(bits, mvd):
    """h264_gop_ref.encode_inter_mb's layer (ue(0) se(0) se(0) ...) with mvd_l0 = mvd."""
    nb = O.Bits()
    nb.ue(0)
    nb.se(int(mvd[0])), nb.se(int(mvd[1]))
    nb.put(bits.v & ((1 << (bits.n - 3)) - 1), bits.n - 3)
    return nb


def encode_p(frame, ref, qp, frame_num, rng):
    """The sample of one P frame against ref (Y, Cb, Cr) with search range rng.  Returns (bytes, recon, mb types,
    vectors (H / 16, W / 16, 2) quarter-pel (x, y), zero where not P_L0_16x16)."""
    frame = np.asarray(frame)
    h, w, _ = frame.shape
    cur = O.colour(frame)
    mv = search(cur[0], ref[0], qp, rng)
    m = rng + 8
    pred = (_frame(luma_pred(luma_phases(ref[0], m), m, mv)) if rng else ref[0],
            _frame(chroma_pred(ref[1], mv)), _frame(chroma_pred(ref[2], mv)))
    skip = G.inter_levels(cur, ref, qp)[3]
    ly, cac, cdc, _ = G.inter_levels(cur, pred, qp)
    rec = tuple(p.copy() for p in ref)
    types = np.empty((h // 16, w // 16), object)
    coded_mv = np.zeros((h // 16, w // 16, 2), np.int64)
    out = bytearray()
    for my in range(h // 16):
        b = G.p_slice_header(my * (w // 16), frame_num, qp)
        left, run, mvp = None, 0, np.zeros(2, np.int64)
        for mx in range(w // 16):
            sy, sx = slice(16 * my, 16 * my + 16), slice(16 * mx, 16 * mx + 16)
            cy, cx = slice(8 * my, 8 * my + 8), slice(8 * mx, 8 * mx + 8)
            src = (cur[0][sy, sx], cur[1][cy, cx], cur[2][cy, cx])
            if skip[my, mx]:
                run += 1
                types[my, mx] = G.SKIP
                col = (ref[0][sy, sx], ref[1][cy, cx], ref[2][cy, cx])
                left = {"y": col[0][:, 15], "c": (col[1][:, 7], col[2][:, 7]), "nz": np.zeros(4, np.int64),
                        "cnz": (np.zeros(2, np.int64), np.zeros(2, np.int64))}
                mvp = np.zeros(2, np.int64)
                continue
            p = (pred[0][sy, sx], pred[1][cy, cx], pred[2][cy, cx])
            inter = int(np.abs(src[0] - p[0]).sum()) <= G._intra_sad(src[0], left)
            if inter:
                bits, r, new_left = G.encode_inter_mb(ly[my, mx], cac[:, my, mx], cdc[:, my, mx], p, left, qp)
                if bits is not None:
                    bits = _with_mvd(bits, mv[my, mx] - mvp)
                t = G.INTER
            else:
                bits, r, new_left, t = O.encode_mb(src[0], src[1], src[2], left, qp, mx)
                if bits is not None:
                    bits = _intra_p(bits)
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
            mvp = mv[my, mx].copy() if t == G.INTER else np.zeros(2, np.int64)
            if t == G.INTER:
                coded_mv[my, mx] = mv[my, mx]
            rec[0][sy, sx], rec[1][cy, cx], rec[2][cy, cx] = r
            types[my, mx], left = t, new_left
        if run:
            b.ue(run)
        b.trailing()
        nal = O.emulation_prevent(b.tobytes())
        out += len(nal).to_bytes(4, "big") + nal
    return bytes(out), rec, types, coded_mv


def encode_clip(frames, qp=20, gop=2, rng=0):
    """The samples of one clip with keyframe interval gop and search range rng: as h264_gop_ref.encode_clip, P frames
    by encode_p.  Returns a list of (bytes, recon (Y, Cb, Cr), mb types, vectors or None for IDR frames) per frame."""
    out = []
    for t, f in enumerate(frames):
        if t % gop == 0:
            out.append(O.encode(f, qp, t // gop) + (None,))
        else:
            out.append(encode_p(f, out[-1][1], qp, (t % gop) % 16, rng))
        h, w = out[-1][1][0].shape
        assert len(out[-1][0]) <= G.max_bytes(h, w, gop)
    return out

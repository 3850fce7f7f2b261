"""The pose and body-model kernels on the GPU, every output element against its float64 bound (tests/pose_bounds.py),
at the shapes and inputs where they go wrong: rotations near pi, at 0 and across the 1e-6 branch, degenerate and
scaled rot6d, row counts around each grid-stride cap, saturated softmax logits, column-sliced and strided views,
chain / star / SMPL-X / random kinematic trees and vertices with 1 to 55 skinning weights.  Each sweep prints the
largest share of its bound used; the rotation sweeps also print how many sign decisions float64 settles."""

import numpy as np
import pytest
import torch

import pose_bounds as pb
from body_cases import random_tree
from pantomatrix_b200 import _lib
from pantomatrix_b200.body_model import ALL_JOINTS, MOTION_REP_JOINTS, SmplxBodyModel
from synthetic_models import SMPLX_FULL_VERTS, SMPLX_PARENTS, smplx_arrays
from test_pose_bounds import rot6d_cases, softmax_cases

pytestmark = pytest.mark.gpu
DEV = "cuda"
CHUNK = 1 << 16                        # rot6d rows per float64 reference call


@pytest.fixture(scope="module")
def ops():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    from pantomatrix_b200 import ops as o
    assert _lib.load().pm_device_cc() == 90, "sm_90a kernels need a Hopper (H100) device"
    return o


def _rot_rows(n, seed):
    """n fp32 rot6d rows on the GPU: the edge cases of rot6d_cases, cycled in a seeded order."""
    base = rot6d_cases(seed=seed)
    idx = torch.randperm(n, generator=torch.Generator().manual_seed(seed)) % len(base)
    return base[idx].to(DEV)


def _check_aa(got, d6, tag):
    """got (m, 3) vs rot6d_to_aa(d6 (m, 6)), chunked; returns (worst fraction, decided, total)."""
    worst, dec = 0.0, 0
    for s in range(0, len(d6), CHUNK):
        want, bound, decided = pb.rot6d_to_aa(d6[s:s + CHUNK])
        g = got[s:s + CHUNK]
        frac = pb.bound_fraction(g, pb.pick_signs(g, want, decided), bound)
        assert frac <= 1.0, (tag, s, frac)
        worst, dec = max(worst, frac), dec + int(decided.sum())
    return worst, dec, 3 * len(d6)


# ------------------------------------------------------------------------------------------------------------------
# rot6d_to_aa (CaMN / DisCo heads)
# ------------------------------------------------------------------------------------------------------------------


def _slot_map(n_sel, seed):
    """A gapped slot map: n_sel of the 55 joints, in a shuffled order, the rest -1."""
    g = torch.Generator().manual_seed(seed)
    joints = torch.randperm(55, generator=g)[:n_sel]
    slot = torch.full((55,), -1, dtype=torch.int32)
    slot[joints] = torch.randperm(n_sel, generator=g).int()
    return slot


@pytest.mark.parametrize("n_sel,rows", [(1, 11021), (13, 11022), (55, 11021), (55, 11022), (13, 1)])
def test_rot6d_to_aa_every_element(ops, n_sel, rows):
    slot = _slot_map(n_sel, n_sel + rows)
    d6 = _rot_rows(rows * n_sel, seed=rows)
    got = ops.rot6d_to_aa(d6.reshape(rows, n_sel * 6), slot.to(DEV), n_sel).reshape(rows, 55, 3)
    sel = slot >= 0
    if (~sel).any():
        assert got[:, (~sel).to(DEV)].abs().max() == 0
    joints = torch.nonzero(sel).flatten()[torch.argsort(slot[sel])].to(DEV)   # the selected joints in slot order
    worst, dec, tot = _check_aa(got[:, joints].reshape(-1, 3), d6, (n_sel, rows))
    print(f"rot6d_to_aa n_sel {n_sel} rows {rows}: worst {worst:.3g} of the bound, signs decided {dec}/{tot}")


def test_rot6d_to_aa_refuses_a_bad_slot_table(ops):
    d6 = torch.zeros(4, 13 * 6, device=DEV)
    with pytest.raises(_lib.PmError):
        ops.rot6d_to_aa(d6, torch.zeros(55, dtype=torch.int64, device=DEV), 13)
    with pytest.raises(_lib.PmError):
        ops.rot6d_to_aa(d6, torch.zeros(54, dtype=torch.int32, device=DEV), 13)


# ------------------------------------------------------------------------------------------------------------------
# pose_compose (EMAGE decode)
# ------------------------------------------------------------------------------------------------------------------

DIMS = dict(face=106, upper=78, hands=180, lower=61)


def _parts(bs, t, seed):
    """Decoder outputs whose rot6d slots carry the edge-case rows (each slot its own rows) and random tails."""
    g = torch.Generator().manual_seed(seed)
    out = {}
    for i, (k, dim) in enumerate(DIMS.items()):
        x = torch.randn(bs * t, dim, generator=g).to(DEV)
        n6 = {"face": 1, "upper": 13, "hands": 30, "lower": 9}[k]
        x[:, :6 * n6] = _rot_rows(bs * t * n6, seed=seed + i).reshape(bs * t, 6 * n6)
        out[k] = x.reshape(bs, t, dim)
    return out


def _check_pose_compose(ops, parts, bs, t, tag):
    expr, aa, m4 = ops.pose_compose(parts["face"], parts["upper"], parts["hands"], parts["lower"], bs, t, DEV)
    worst, dec, tot = 0.0, 0, 0
    if any(v is not None for v in parts.values()):
        step = max(1, CHUNK // (55 * t))                              # clips per reference call
        for b in range(0, bs, step):
            sl = {k: None if v is None else v[b:b + step] for k, v in parts.items()}
            want, bound, decided = pb.pose_compose(sl["face"], sl["upper"], sl["hands"], sl["lower"])
            g = aa[b:b + step]
            frac = pb.bound_fraction(g, pb.pick_signs(g, want, decided), bound)
            assert frac <= 1.0, (tag, b, frac)
            worst, dec, tot = max(worst, frac), dec + int(decided.sum()), tot + decided.numel()
    else:
        assert aa.abs().max() == 0
    (w4, b4), want_expr = pb.pose_compose_rest(parts["face"], parts["lower"], aa)
    frac4 = pb.bound_fraction(m4, w4, b4)
    assert frac4 <= 1.0, (tag, frac4)
    assert torch.equal(expr, want_expr) and torch.equal(m4[..., 330:].double(), w4[..., 330:])
    return worst, frac4, dec, tot


@pytest.mark.parametrize("bs,t", [(1, 1), (1, 147), (1, 9472), (1, 9473), (32, 300)])
def test_pose_compose_every_element(ops, bs, t):
    """bt = bs t around the grid cap: 148 * 16 blocks of 256 threads cover 9472 rows of 64 threads each."""
    worst, frac4, dec, tot = _check_pose_compose(ops, _parts(bs, t, seed=bs * t), bs, t, (bs, t))
    print(f"pose_compose bt {bs * t}: axis-angle worst {worst:.3g}, motion4inf worst {frac4:.3g}, signs decided "
          f"{dec}/{tot}")


def test_pose_compose_each_part_present_or_absent(ops):
    bs, t = 3, 49
    full = _parts(bs, t, seed=5)
    worst = 0.0
    for mask in range(16):
        parts = {k: (v if (mask >> i) & 1 else None) for i, (k, v) in enumerate(full.items())}
        w, f4, _, _ = _check_pose_compose(ops, parts, bs, t, mask)
        worst = max(worst, w, f4)
    print(f"pose_compose, all 16 part subsets: worst {worst:.3g}")


# ------------------------------------------------------------------------------------------------------------------
# softmax2_mix (DisCo content mix)
# ------------------------------------------------------------------------------------------------------------------


@pytest.mark.parametrize("ch", [37, 300])
def test_softmax2_mix_every_element_into_a_column_slice(ops, ch):
    sel, c1, c2 = (x.to(DEV) for x in softmax_cases(ch))
    rows = len(sel)
    t = 7
    sel, c1, c2 = (x.repeat(t, 1).reshape(t, rows, -1).transpose(0, 1).contiguous() for x in (sel, c1, c2))
    wide = torch.full((rows, t, ch + 19), 12345.0, device=DEV)
    out = wide[:, :, 5:5 + ch]
    ops.softmax2_mix(sel, c1, c2, out=out)
    want, bound = pb.softmax2_mix(sel, c1, c2)
    frac = pb.bound_fraction(out, want, bound)
    assert frac <= 1.0, frac
    assert (wide[..., :5] == 12345.0).all() and (wide[..., 5 + ch:] == 12345.0).all()
    assert torch.equal(ops.softmax2_mix(sel, c1, c2), out)
    gap = sel[..., 0] - sel[..., 1]                                  # expf(-gap) underflows: the other operand exactly
    assert torch.equal(out[gap >= 104], c1[gap >= 104]) and torch.equal(out[gap <= -104], c2[gap <= -104])
    print(f"softmax2_mix ch {ch}: worst {frac:.3g} of the bound")


def test_softmax2_mix_refuses_an_out_with_a_longer_clip_stride(ops):
    """A (B, T, ch) out cut as [:, :T] from a (B, T', ch) buffer has clips T' rows apart: the kernel addresses rows by
    one stride, so such an out would be written at the wrong rows.  ops refuses it (and accepts its dense twin)."""
    sel, c1, c2 = torch.randn(2, 5, 2, device=DEV), torch.randn(2, 5, 16, device=DEV), torch.randn(2, 5, 16, device=DEV)
    longer = torch.zeros(2, 8, 16, device=DEV)
    with pytest.raises(_lib.PmError):
        ops.softmax2_mix(sel, c1, c2, out=longer[:, :5])
    assert longer.abs().max() == 0
    with pytest.raises(_lib.PmError):
        ops.softmax2_mix(sel, c1, c2, out=torch.zeros(2, 16, 5, device=DEV).transpose(1, 2))
    ok = torch.zeros(2, 5, 20, device=DEV)[:, :, 2:18]
    assert torch.equal(ops.softmax2_mix(sel, c1, c2, out=ok), ops.softmax2_mix(sel, c1, c2))


# ------------------------------------------------------------------------------------------------------------------
# motion_rep
# ------------------------------------------------------------------------------------------------------------------


def _poses_view(x, strided):
    if not strided:
        return x
    b, t, _ = x.shape
    wide = torch.zeros(b, 2 * t, 171, device=DEV)
    v = wide[:, ::2, 3:168]
    v.copy_(x)
    return v


@pytest.mark.parametrize("batch,t", [(1, 2), (4, 3), (2, 300), (107, 103), (3674, 3), (5511, 2)])
def test_motion_rep_every_element(ops, batch, t):
    """rows = batch t of 11021 and 11022 straddle the grid cap (148 * 16 * 256 threads over 55 joints per row)."""
    g = torch.Generator().manual_seed(batch * t)
    aa = _rot_rows(batch * t * 55, seed=t)                          # axis-angle rows: reuse the rotations' values
    poses = (aa[:, :3] * 2.0).reshape(batch, t, 165)
    joints = torch.randn(batch, t, 55, 3, generator=g).to(DEV)
    dt, two_dt = np.float32(1 / 30), np.float32(2 / 30)
    worst = 0.0
    for strided in (False, True):
        p = _poses_view(poses, strided)
        out = ops.motion_rep(p, joints, dt, two_dt, torch.empty(batch, t, 825, device=DEV))
        for b in range(0, batch, max(1, 20000 // t)):
            sl = slice(b, b + max(1, 20000 // t))
            want, bound = pb.motion_rep(p[sl], joints[sl], dt, two_dt)
            frac = pb.bound_fraction(out[sl], want, bound)
            assert frac <= 1.0, (strided, b, frac)
            worst = max(worst, frac)
        # position, velocity and angular velocity are one subtraction and one division: torch fp32 gives the same bits
        v = out.view(batch, t, 55, 15)
        tt = torch.arange(t, device=DEV)
        hi, lo = (tt + 1).clamp_max(t - 1), (tt - 1).clamp_min(0)
        den = torch.where((tt == 0) | (tt == t - 1), torch.tensor(dt, device=DEV), torch.tensor(two_dt, device=DEV))
        den = den[None, :, None, None]
        P = p.reshape(batch, t, 55, 3)
        assert torch.equal(v[..., 0:3], joints)
        assert torch.equal(v[..., 3:6], (joints[:, hi] - joints[:, lo]) / den)
        assert torch.equal(v[..., 12:15], (P[:, hi] - P[:, lo]) / den)
    print(f"motion_rep batch {batch} t {t}: worst {worst:.3g} of the bound")


def test_motion_rep_refuses_unsupported_layouts(ops):
    poses, joints = torch.zeros(2, 5, 165, device=DEV), torch.zeros(2, 5, 55, 3, device=DEV)
    with pytest.raises(_lib.PmError):                                # poses with a strided last dimension
        ops.motion_rep(torch.zeros(2, 5, 330, device=DEV)[..., ::2], joints, 0.1, 0.2, torch.empty(2, 5, 825, device=DEV))
    with pytest.raises(_lib.PmError):                                # out of another shape
        ops.motion_rep(poses, joints, 0.1, 0.2, torch.empty(2, 4, 825, device=DEV))
    with pytest.raises(_lib.PmError):                                # joints of fewer frames
        ops.motion_rep(poses, joints[:, :4].contiguous(), 0.1, 0.2, torch.empty(2, 5, 825, device=DEV))


# ------------------------------------------------------------------------------------------------------------------
# SMPL-X forward kinematics
# ------------------------------------------------------------------------------------------------------------------

CHAIN = tuple(range(-1, 54))                                         # 55 levels
STAR = (-1,) + (0,) * 54


def _fk_inputs(rng, B, T, strided):
    """poses with components up to +-2 pi and exactly zero joints / frames; betas, expression, transl; strided=True
    gives views with clip and frame strides."""
    def put(x, c):
        x = torch.from_numpy(np.asarray(x, np.float32)).to(DEV).reshape(B, T, c)
        if not strided:
            return x
        v = torch.zeros(B, 2 * T, c + 13, device=DEV)[:, ::2, 5:5 + c]
        v.copy_(x)
        return v
    p = rng.uniform(-2 * np.pi, 2 * np.pi, (B * T, 55, 3)) * rng.uniform(0, 1, (B * T, 55, 1))
    p[:, 7] = 0.0
    p[::4] = 0.0
    betas = torch.from_numpy(rng.normal(0, 1, (B, 300)).astype(np.float32)).to(DEV)
    if strided:
        betas = torch.zeros(B, 320, device=DEV)[:, 10:310].copy_(betas)
    return (put(p.reshape(B * T, 165), 165), betas, put(rng.normal(0, 1, (B * T, 100)), 100),
            put(rng.normal(0, 1, (B * T, 3)), 3))


def _fk_check(ops, bm, poses, betas, expr, transl, mask, tag):
    B, T = poses.shape[:2]
    rows = B * T
    joints = torch.empty(rows, 55, 3, device=DEV)
    rel = torch.empty(rows, 55, 12, device=DEV)
    feat = torch.full((rows, 893), 777.0, device=DEV)
    ops.smplx_fk(poses, betas, expr, None, mask, bm._tables, joints, rel, feat)
    assert (feat[:, 886:] == 777.0).all()
    worst = {}
    got = pb.fk_outputs(joints, rel, feat)
    clips = max(1, 4096 // T)                                      # clips per reference call
    for b0 in range(0, B, clips):
        cb = slice(b0, b0 + clips)
        sl = slice(b0 * T, (b0 + clips) * T)
        ref = pb.smplx_fk(poses[cb], None if betas is None else betas[cb], None if expr is None else expr[cb],
                          mask, bm._tables, joints[sl], rel[sl])
        for k, (want, bound) in ref.items():
            frac = pb.bound_fraction(got[k][sl], want, bound)
            assert frac <= 1.0, (tag, k, b0, frac)
            worst[k] = max(worst.get(k, 0.0), frac)
    only = torch.empty_like(joints)
    ops.smplx_fk(poses, betas, expr, None, mask, bm._tables, only)  # the joints-only launch: the same bits
    assert torch.equal(only, joints)
    if transl is not None:
        jt = torch.empty_like(joints)
        rel_t = torch.empty_like(rel)
        ops.smplx_fk(poses, betas, expr, transl, mask, bm._tables, jt, rel_t)
        want, bound = pb.transl_add(joints, transl)
        frac = pb.bound_fraction(jt, want, bound)
        assert frac <= 1.0 and torch.equal(rel_t, rel), (tag, frac)
        worst["transl"] = frac
    return worst


def _merge(worst, new):
    return {k: max(worst.get(k, 0.0), new.get(k, 0.0)) for k in set(worst) | set(new)}


def _fmt(worst):
    """The worst share of the bound per output: G's rotation and translation, rel's translation column, the GEMM
    operand row and the final transl addition."""
    return ", ".join(f"{k} {worst[k]:.3g}" for k in sorted(worst))


TREES = {"smplx": SMPLX_PARENTS, "chain": CHAIN, "star": STAR,
         "random": random_tree(np.random.default_rng(17)), "random2": random_tree(np.random.default_rng(18))}


@pytest.mark.parametrize("tree", list(TREES))
def test_fk_every_element_per_level(ops, tree):
    """Each level teacher-forced from the kernel's own parent transforms; rows % 16 of 0, 1 and 15 (partial last CTA);
    every betas / expression / transl None combination on the SMPL-X tree, two on the others; both joint masks; dense
    and strided views."""
    rng = np.random.default_rng(len(tree) + sum(map(ord, tree)))
    bm = SmplxBodyModel(smplx_arrays(64, 3, TREES[tree]), DEV)
    combos = [(b, e, t) for b in (0, 1) for e in (0, 1) for t in (0, 1)] if tree == "smplx" else [(1, 1, 1), (0, 0, 0)]
    worst = {}
    for (B, T) in ((2, 8), (1, 17), (3, 5), (1, 33)):
        for strided in (False, True):
            poses, betas, expr, transl = _fk_inputs(rng, B, T, strided)
            for (ub, ue, ut) in combos:
                for mask in (ALL_JOINTS, MOTION_REP_JOINTS):
                    args = (betas if ub else None, expr if ue else None, transl if ut else None)
                    worst = _merge(worst, _fk_check(ops, bm, poses, *args, mask, (tree, B, T, strided, ub, ue, ut, mask)))
    print(f"smplx_fk {tree} tree, worst share of the bound: {_fmt(worst)}")


def test_fk_every_element_at_the_product_size(ops):
    rng = np.random.default_rng(21)
    bm = SmplxBodyModel(smplx_arrays(64), DEV)
    poses, betas, expr, transl = _fk_inputs(rng, 32, 300, True)
    worst = _fk_check(ops, bm, poses, betas, expr, transl, ALL_JOINTS, "32x300")
    print(f"smplx_fk 32 x 300 frames, worst share of the bound: {_fmt(worst)}")


# ------------------------------------------------------------------------------------------------------------------
# SMPL-X skinning
# ------------------------------------------------------------------------------------------------------------------


def _csr(n_verts, seed):
    """Vertex v has 1 + v % 55 weights on distinct joints, every 7th of them exactly 0."""
    rng = np.random.default_rng(seed)
    ptr, col, val = [0], [], []
    for v in range(n_verts):
        k = 1 + v % 55
        col += rng.permutation(55)[:k].tolist()
        w = rng.dirichlet(np.ones(k))
        w[::7] = 0.0 if k > 1 else w[::7]
        val += w.tolist()
        ptr.append(ptr[-1] + k)
    i32 = lambda x: torch.tensor(x, dtype=torch.int32, device=DEV)
    return i32(ptr), i32(col), torch.tensor(val, dtype=torch.float32, device=DEV)


@pytest.mark.parametrize("n_verts,B,T", [(1, 2, 3), (255, 3, 7), (257, 1, 33), (SMPLX_FULL_VERTS, 2, 5),
                                         (SMPLX_FULL_VERTS, 32, 300)])
def test_skin_every_element(ops, n_verts, B, T):
    g = torch.Generator().manual_seed(n_verts + B * T)
    rows = B * T
    csr = _csr(n_verts, n_verts)
    rel = torch.randn(rows, 55, 12, generator=g).to(DEV)
    ld = 3 * n_verts + 5
    buf = torch.randn(rows, ld, generator=g).to(DEV)
    transl = torch.zeros(B, 2 * T, 7, device=DEV)[:, ::2, 2:5].copy_(torch.randn(B, T, 3, generator=g).to(DEV))
    worst = 0.0
    for tr in (transl, None):
        v_posed = buf.clone()
        ops.smplx_skin(buf, n_verts, csr, rel, tr, T)
        assert torch.equal(buf[:, 3 * n_verts:], v_posed[:, 3 * n_verts:])
        step = max(1, (1 << 26) // (n_verts * 12 * 8))
        for s in range(0, rows, step):
            sl = slice(s, s + step)
            want, bound = pb.smplx_skin(v_posed[sl], n_verts, csr, rel[sl],
                                        None if tr is None else tr.reshape(rows, 3)[sl], T)
            frac = pb.bound_fraction(buf[sl, :3 * n_verts], want, bound)
            assert frac <= 1.0, (n_verts, rows, tr is None, s, frac)
            worst = max(worst, frac)
        buf = v_posed
    print(f"smplx_skin {n_verts} vertices x {rows} rows: worst {worst:.3g} of the bound")

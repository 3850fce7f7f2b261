"""The per-element checks of tests/pose_bounds.py can fail: each is fed a CPU fp32 restatement of its kernel (torch fp32
in the kernel's operation order: torch's CPU elementwise ops round once each, like -fmad=false), which it must accept,
and small copies of plausible kernel bugs applied to that restatement, each of which it must reject.  No GPU needed."""
import math

import numpy as np
import pytest
import torch

import pose_bounds as pb
from body_cases import small_arrays
from pantomatrix_b200.body_model import ALL_JOINTS, MOTION_REP_JOINTS, SmplxBodyModel

# pose_compose_kernel's joint tables (pm_pose.cu kJointPart / kJointSlot), restated for the fp32 restatement; the
# reference takes the joint map from the reference's joint lists instead (pose_bounds.joint_sources)
PART = [1, 1, 1, 0, 1, 1, 0, 1, 1, 0, 1, 1, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 3, 4, 4] + [2] * 30
SLOT = [0, 1, 2, 0, 3, 4, 1, 5, 6, 2, 7, 8, 3, 4, 5, 6, 7, 8, 9, 10, 11, 12, 0, 0, 0] + list(range(30))


def _gen(seed):
    return torch.Generator().manual_seed(seed)


def _rotations(angles, axes):
    """float64 (n, 3, 3) rotation matrices of the given angles about the given (unnormalised) axes (Rodrigues)."""
    k = axes / axes.norm(dim=-1, keepdim=True)
    K = torch.zeros(len(k), 3, 3, dtype=torch.float64)
    K[:, 0, 1], K[:, 0, 2], K[:, 1, 2] = -k[:, 2], k[:, 1], -k[:, 0]
    K = K - K.transpose(1, 2)
    a = angles[:, None, None]
    return torch.eye(3, dtype=torch.float64) + torch.sin(a) * K + (1 - torch.cos(a)) * K @ K


def rot6d_cases(n=512, seed=0):
    """fp32 (m, 6) rot6d rows: random; exact rotations over [0, pi]; within 1e-4 of pi and exactly pi about coordinate
    and oblique axes; angles straddling the 1e-6 branch and 0; zero vectors and collinear column pairs; all scaled by
    2^+-20 as well."""
    g = _gen(seed)
    rows = [torch.randn(n, 6, generator=g, dtype=torch.float64)]
    axes = torch.randn(n, 3, generator=g, dtype=torch.float64)
    coord = torch.eye(3, dtype=torch.float64).repeat(4, 1)
    oblique = torch.tensor([[1.0, 1.0, 0.0], [1.0, -1.0, 1.0], [0.0, 2.0, -1.0], [3.0, 1.0, 2.0]], dtype=torch.float64)
    six = lambda m: m[:, :2, :].reshape(-1, 6)
    rows.append(six(_rotations(torch.linspace(0, math.pi, n, dtype=torch.float64), axes)))
    for ax in (coord, oblique, axes[:64]):
        for a in (math.pi, math.pi - 1e-4, math.pi - 3e-5, math.pi - 1e-6):
            rows.append(six(_rotations(torch.full((len(ax),), a, dtype=torch.float64), ax)))
    small = torch.tensor([0.0, 1e-8, 4.9e-7, 5e-7, 5.1e-7, 9.9e-7, 1e-6, 1.01e-6, 2e-6, 1e-5, 1e-3], dtype=torch.float64)
    rows.append(six(_rotations(small.repeat(8), axes[:8].repeat_interleave(len(small), 0))))
    d = torch.randn(8, 3, generator=g, dtype=torch.float64)
    special = torch.cat([torch.zeros(2, 6, dtype=torch.float64), torch.cat([d, 2 * d], 1), torch.cat([d, -d], 1),
                         torch.cat([d, torch.zeros_like(d)], 1), torch.cat([torch.zeros_like(d), d], 1)])
    rows.append(special)
    base = torch.cat(rows).float()
    return torch.cat([base, base * 2.0 ** 20, base * 2.0 ** -20])


# ------------------------------------------------------------------------------------------------------------------
# rot6d -> axis-angle
# ------------------------------------------------------------------------------------------------------------------


def _rot6d_to_aa32(d, bug=None):
    """fp32 restatement of the device function rot6d_to_aa (pm_pose.cu), one rounding per op in source order.
    bug: 'atan2_args' (atan2f(w, n)), 'sqrtf' (sqrtf instead of sqrt_pos), 'sign_pair'
    (x's sign from y's off-diagonal pair), 'no_projection' (Gram-Schmidt without removing b1 from the second column)."""
    f = lambda c: d[..., c]
    n1 = (f(0) * f(0) + f(1) * f(1) + f(2) * f(2)).sqrt().clamp_min(pb.EPS_NORM)
    b1x, b1y, b1z = f(0) / n1, f(1) / n1, f(2) / n1
    dot = b1x * f(3) + b1y * f(4) + b1z * f(5)
    if bug == "no_projection":
        dot = torch.zeros_like(dot)
    b2x, b2y, b2z = f(3) - dot * b1x, f(4) - dot * b1y, f(5) - dot * b1z
    n2 = (b2x * b2x + b2y * b2y + b2z * b2z).sqrt().clamp_min(pb.EPS_NORM)
    b2x, b2y, b2z = b2x / n2, b2y / n2, b2z / n2
    b3x = b1y * b2z - b1z * b2y
    b3y = b1z * b2x - b1x * b2z
    b3z = b1x * b2y - b1y * b2x
    m00, m11, m22 = b1x, b2y, b3z
    sq = (lambda a: a.sqrt()) if bug == "sqrtf" else (lambda a: torch.where(a > 0, a.clamp_min(0).sqrt(), 0.0))
    w = 0.5 * sq(1 + m00 + m11 + m22)
    x = 0.5 * sq(1 + m00 - m11 - m22)
    y = 0.5 * sq(1 - m00 + m11 - m22)
    z = 0.5 * sq(1 - m00 - m11 + m22)
    sign_like = lambda a, b: torch.where((a < 0) != (b < 0), -a, a)
    x = sign_like(x, (b1z - b3x) if bug == "sign_pair" else (b3y - b2z))
    y = sign_like(y, b1z - b3x)
    z = sign_like(z, b2x - b1y)
    n = (x * x + y * y + z * z).sqrt()
    half = torch.atan2(w, n) if bug == "atan2_args" else torch.atan2(n, w)
    ang = 2 * half
    s = torch.where(ang.abs() < pb.EPS_BRANCH, 0.5 - (ang * ang) / 48, torch.sin(half) / ang)
    return torch.stack([x / s, y / s, z / s], -1)


def _check_aa(got, want, bound, decided):
    return pb.within(got, pb.pick_signs(got, want, decided), bound)


def test_rot6d_to_aa_bound_accepts_fp32():
    d = rot6d_cases()
    want, bound, decided = pb.rot6d_to_aa(d)
    assert _check_aa(_rot6d_to_aa32(d), want, bound, decided)
    assert not decided.all() and decided.float().mean() > 0.5     # the near-pi rows leave some signs to the kernel


def _small_angle_rows():
    """Exact fp32 rotations at angles 1e-3 .. 0.1 rad (the regime where a 0.2 degree gate sees nothing)."""
    g = _gen(5)
    ang = 10.0 ** torch.linspace(-3, -1, 256, dtype=torch.float64)
    m = _rotations(ang, torch.randn(256, 3, generator=g, dtype=torch.float64) + 0.5)
    return m[:, :2, :].reshape(-1, 6).float()


def _near_pi_rows():
    ax = torch.tensor([[1.0, 0.0, 0.0], [0.0, 1.0, 0.0], [1.0, 1.0, 0.0], [1.0, -1.0, 1.0], [2.0, 0.5, -1.0]],
                      dtype=torch.float64).repeat(20, 1)
    a = math.pi - torch.linspace(0, 1e-4, len(ax), dtype=torch.float64)
    m = _rotations(a, ax)
    return m[:, :2, :].reshape(-1, 6).float()


# half = acosf(w) is not among these: the four sqrt_pos arguments sum to exactly 4, so n^2 + w^2 = 1 up to rounding and
# acos(w) = atan2(n, w) up to a few U / sin(half) in half, which moves s = sin(half) / (2 half) by about U / 6 - the
# same function to within the kernel's own rounding, which no valid bound can tell apart.
@pytest.mark.parametrize("bug,rows", [
    ("atan2_args", _small_angle_rows),     # atan2f(w, n): half ~ pi / 2 at small angles, aa 57 % too long
    ("sqrtf", _near_pi_rows),              # sqrtf of 1 + trace < 0 near pi: NaN
    ("sign_pair", lambda: rot6d_cases(256, seed=3)[:512]),
    ("no_projection", lambda: torch.randn(256, 6, generator=_gen(4))),
])
def test_rot6d_to_aa_bound_rejects(bug, rows):
    d = rows()
    want, bound, decided = pb.rot6d_to_aa(d)
    assert _check_aa(_rot6d_to_aa32(d), want, bound, decided)
    assert not _check_aa(_rot6d_to_aa32(d, bug), want, bound, decided)


def test_rot6d_to_aa_bound_is_not_vacuous():
    """Near-orthonormal rot6d (every entry within 1e-3) at angles in [0.1, 3.0] rad.  Where every axis component is at
    least 0.3 in magnitude the bound is below 2^-15 max(|aa|, 1).  It grows where a component approaches 0: that
    component is x = sqrt_pos(a) / 2 with a = 4 x^2 computed from 1 +- m00 +- m11 +- m22 with an absolute error of some
    10 U, so x carries a relative error of about 10 U / (8 x^2) - the formula's own conditioning, which the kernel
    follows on purpose - and the bound stays below 2^-9 over the whole class."""
    g = _gen(6)
    n = 4096
    axes = torch.randn(n, 3, generator=g, dtype=torch.float64)
    axes /= axes.norm(dim=-1, keepdim=True)
    ang = 0.1 + 2.9 * torch.rand(n, generator=g, dtype=torch.float64)
    m = _rotations(ang, axes)[:, :2, :].reshape(n, 6)
    d = (m + 1e-3 * (2 * torch.rand(n, 6, generator=g, dtype=torch.float64) - 1)).float()
    want, bound, _ = pb.rot6d_to_aa(d)
    rel = (bound / want.norm(dim=-1, keepdim=True).clamp_min(1.0)).amax(-1)
    assert float(rel.max()) < 2.0 ** -9
    good = axes.abs().amin(-1) >= 0.3
    assert good.sum() > 500 and float(rel[good].max()) < 2.0 ** -15
    assert float(rel.median()) < 2.0 ** -17


# ------------------------------------------------------------------------------------------------------------------
# pose_compose: the joint map, motion4inf
# ------------------------------------------------------------------------------------------------------------------


def _aa_to_rot6d32(aa):
    """fp32 restatement of the device function aa_to_rot6d (pm_pose.cu)."""
    a0, a1, a2 = aa[..., 0], aa[..., 1], aa[..., 2]
    ang = (a0 * a0 + a1 * a1 + a2 * a2).sqrt()
    half = 0.5 * ang
    s = torch.where(ang.abs() < pb.EPS_BRANCH, 0.5 - (ang * ang) / 48, torch.sin(half) / ang)
    r, i, j, k = torch.cos(half), a0 * s, a1 * s, a2 * s
    two_s = 2.0 / (r * r + i * i + j * j + k * k)
    return torch.stack([1 - two_s * (j * j + k * k), two_s * (i * j - k * r), two_s * (i * k + j * r),
                        two_s * (i * j + k * r), 1 - two_s * (i * i + k * k), two_s * (j * k - i * r)], -1)


def _pose_compose32(face, upper, hands, lower, slot=SLOT):
    """fp32 restatement of pose_compose_kernel's axis_angle and motion4inf with its joint tables."""
    srcs = {0: (upper, 78), 1: (lower, 61), 2: (hands, 180), 3: (face, 106)}
    bs, t = upper.shape[:2]
    aa = torch.zeros(bs, t, 55, 3)
    for j in range(55):
        src = srcs.get(PART[j], (None, 0))[0]
        if src is not None:
            aa[:, :, j] = _rot6d_to_aa32(src[:, :, 6 * slot[j]:6 * slot[j] + 6])
    m4 = torch.cat([_aa_to_rot6d32(aa).reshape(bs, t, 330), lower[:, :, 54:]], -1)
    return aa.reshape(bs, t, 165), m4


def test_pose_compose_bound_accepts_fp32_and_rejects_swapped_slots():
    g = _gen(7)
    bs, t = 2, 9
    parts = [torch.randn(bs, t, n, generator=g) for n in (106, 78, 180, 61)]     # distinct inputs per slot
    want, bound, decided = pb.pose_compose(*parts)
    aa, m4 = _pose_compose32(*parts)
    assert _check_aa(aa, want, bound, decided)
    (w4, b4), expr = pb.pose_compose_rest(parts[0], parts[3], aa)
    assert pb.within(m4, w4, b4) and torch.equal(expr, parts[0][:, :, 6:])
    swapped = list(SLOT)
    swapped[28], swapped[29] = swapped[29], swapped[28]                           # two hand joints' slots
    aa_bad, _ = _pose_compose32(*parts, slot=swapped)
    assert not _check_aa(aa_bad, want, bound, decided)


def test_aa_to_rot6d_bound_accepts_fp32():
    g = _gen(8)
    aa = torch.cat([torch.randn(2000, 3, generator=g) * 2, torch.zeros(4, 3), torch.full((4, 3), 1e-7),
                    torch.tensor([[2 * math.pi, 0, 0], [0, 0, -math.pi], [4.9e-7, 0, 0], [5.1e-7, 0, 0]])])
    want, bound = pb.aa_to_rot6d(aa)
    got = _aa_to_rot6d32(aa)
    assert pb.within(got, want, bound)
    scale = aa.double().norm(dim=-1, keepdim=True).clamp_min(1.0)
    assert float((bound / scale).max()) < 64 * pb.U                 # a few dozen roundings per radian


# ------------------------------------------------------------------------------------------------------------------
# softmax2_mix
# ------------------------------------------------------------------------------------------------------------------


def _softmax2_mix32(sel, c1, c2, bug=None):
    """fp32 restatement of softmax2_mix_kernel.  bug: 'no_max' (expf of the raw logits), 'one_minus' (w1 = 1 - w0)."""
    a, b = sel[..., 0:1], sel[..., 1:2]
    m = torch.zeros_like(a) if bug == "no_max" else torch.maximum(a, b)
    ea, eb = torch.exp(a - m), torch.exp(b - m)
    s = ea + eb
    w0 = ea / s
    w1 = 1 - w0 if bug == "one_minus" else eb / s
    return w0 * c1 + w1 * c2


def softmax_cases(ch=37, seed=9):
    """Logit gaps 0, +-1e-7, +-1, +-20, +-88, +-104, +-1e4 around several bases, and equal large logits; the channel
    values of the small weight's operand 1e6 times the other's, so a small weight that goes missing shows."""
    g = _gen(seed)
    gaps = torch.tensor([0.0, 1e-7, -1e-7, 1.0, -1.0, 20.0, -20.0, 88.0, -88.0, 104.0, -104.0, 1e4, -1e4])
    base = torch.tensor([0.0, 3.0, -50.0, 90.0, 1e3])
    a = base[:, None].expand(-1, len(gaps)).reshape(-1)
    sel = torch.stack([a, a - gaps.repeat(len(base))], -1)
    sel = torch.cat([sel, torch.tensor([[1e4, 1e4], [-1e4, -1e4], [88.5, 88.5]])])
    c1 = torch.randn(len(sel), ch, generator=g)
    c2 = torch.randn(len(sel), ch, generator=g)
    small = (sel[:, 1] < sel[:, 0])[:, None]                        # w1 is the small weight: scale c2 up, else c1
    return sel, torch.where(small, c1, c1 * 1e6), torch.where(small, c2 * 1e6, c2)


def test_softmax2_mix_bound_accepts_fp32_and_rejects_bugs():
    sel, c1, c2 = softmax_cases()
    want, bound = pb.softmax2_mix(sel, c1, c2)
    assert pb.within(_softmax2_mix32(sel, c1, c2), want, bound)
    big = sel.amax(-1) > 88                                          # expf overflows without the max
    assert big.any() and not pb.within(_softmax2_mix32(sel[big], c1[big], c2[big], "no_max"),
                                       want[big], bound[big])
    assert not pb.within(_softmax2_mix32(sel, c1, c2, "one_minus"), want, bound)


# ------------------------------------------------------------------------------------------------------------------
# motion_rep
# ------------------------------------------------------------------------------------------------------------------


def _motion_rep32(poses, joints, dt, two_dt, bug=None):
    """fp32 restatement of motion_rep_kernel.  bug: 'two_dt_end' (two_dt at the clip ends too), 'last_from_tt' (the
    last frame's velocity reads both ends from frame tt)."""
    batch, t = poses.shape[:2]
    P, J = poses.reshape(batch, t, 55, 3), joints.reshape(batch, t, 55, 3)
    tt = torch.arange(t)
    hi, lo = (tt + 1).clamp_max(t - 1), (tt - 1).clamp_min(0)
    if bug == "last_from_tt":
        lo = torch.where(tt == t - 1, tt, lo)
    den = torch.full((t,), float(two_dt))
    if bug != "two_dt_end":
        den[(tt == 0) | (tt == t - 1)] = float(dt)
    den = den[None, :, None, None]
    out = torch.cat([J, (J[:, hi] - J[:, lo]) / den, _aa_to_rot6d32(P), (P[:, hi] - P[:, lo]) / den], -1)
    return out.reshape(batch, t, 825)


@pytest.mark.parametrize("t", [2, 3, 17])
def test_motion_rep_bound_accepts_fp32_and_rejects_bugs(t):
    g = _gen(10 + t)
    poses = torch.randn(3, t, 165, generator=g)
    joints = torch.randn(3, t, 55, 3, generator=g)
    dt, two_dt = np.float32(1 / 30), np.float32(2 / 30)
    want, bound = pb.motion_rep(poses, joints, dt, two_dt)
    assert pb.within(_motion_rep32(poses, joints, dt, two_dt), want, bound)
    if t > 2:                                                      # t = 2: every frame is a clip end
        assert not pb.within(_motion_rep32(poses, joints, dt, two_dt, "two_dt_end"), want, bound)
    assert not pb.within(_motion_rep32(poses, joints, dt, two_dt, "last_from_tt"), want, bound)


# ------------------------------------------------------------------------------------------------------------------
# SMPL-X forward kinematics and skinning
# ------------------------------------------------------------------------------------------------------------------


@pytest.fixture(scope="module")
def body():
    return SmplxBodyModel(small_arrays(), "cpu")


def _fk32(poses, betas, expr, mask, tables, bug=None):
    """fp32 restatement of smplx_fk_kernel (transl=None): (joints (rows, 55, 3), rel (rows, 55, 12), feat (rows, 886)).
    bug: 'no_eps' (Rodrigues angle |r| without + 1e-8), 'drop_expr99' (the rest-joint GEMV skips expression
    coefficient 99), 'absolute_offset' (FK translates by J_j instead of J_j - J_parent)."""
    jt, jd, pmean, parents, order, start = tables
    batch, t = poses.shape[:2]
    rows = batch * t
    keep = torch.tensor([(mask >> j) & 1 for j in range(55)], dtype=torch.bool)
    p = torch.where(keep[:, None], poses.reshape(rows, 55, 3), 0.0) + pmean.reshape(55, 3)
    e = p if bug == "no_eps" else p + pb.EPS_RODRIGUES
    ang = (e[..., 0] * e[..., 0] + e[..., 1] * e[..., 1] + e[..., 2] * e[..., 2]).sqrt()
    kx, ky, kz = p[..., 0] / ang, p[..., 1] / ang, p[..., 2] / ang
    s, c = torch.sin(ang), torch.cos(ang)
    omc = 1 - c
    R = torch.stack([1 + omc * (-kz * kz - ky * ky), -s * kz + omc * (kx * ky), s * ky + omc * (kx * kz),
                     s * kz + omc * (kx * ky), 1 + omc * (-kz * kz - kx * kx), -s * kx + omc * (ky * kz),
                     -s * ky + omc * (kx * kz), s * kx + omc * (ky * kz), 1 + omc * (-ky * ky - kx * kx)], -1)
    coef = torch.zeros(rows, 400)
    if betas is not None:
        coef[:, :300] = betas[:, None].expand(batch, t, 300).reshape(rows, 300)
    if expr is not None:
        coef[:, 300:] = expr.reshape(rows, 100)
    k0, k1 = (0 if betas is not None else 300), (400 if expr is not None else 300)
    w = jd.clone()
    if bug == "drop_expr99":
        w[399] = 0
    J = (jt + coef[:, k0:k1] @ w[k0:k1]).reshape(rows, 55, 3)
    G = torch.zeros(rows, 55, 3, 4)
    R3 = R.reshape(rows, 55, 3, 3)
    for l in range(len(start) - 1):
        for j in order[int(start[l]):int(start[l + 1])].tolist():
            pj = int(parents[j])
            if pj < 0:
                G[:, j, :, :3], G[:, j, :, 3] = R3[:, j], J[:, j]
                continue
            tv = J[:, j] if bug == "absolute_offset" else J[:, j] - J[:, pj]
            gp = G[:, pj]
            G[:, j, :, :3] = gp[..., 0:1] * R3[:, j, 0:1] + gp[..., 1:2] * R3[:, j, 1:2] + gp[..., 2:3] * R3[:, j, 2:3]
            G[:, j, :, 3] = gp[..., 0] * tv[:, 0:1] + gp[..., 1] * tv[:, 1:2] + gp[..., 2] * tv[:, 2:3] + gp[..., 3]
    rel = G.clone()
    rel[..., 3] = G[..., 3] - (G[..., 0] * J[..., 0:1] + G[..., 1] * J[..., 1:2] + G[..., 2] * J[..., 2:3])
    fe = R.clone()
    fe[..., 0::4] = R[..., 0::4] - 1
    return G[..., 3], rel.reshape(rows, 55, 12), torch.cat([coef, fe[:, 1:].reshape(rows, 486)], 1)


def _fk_ok(outs, ref):
    got = pb.fk_outputs(*outs)
    return all(pb.within(got[k], *ref[k]) for k in ref)


def _fk_inputs(seed, batch=2, t=5):
    g = _gen(seed)
    poses = torch.randn(batch, t, 165, generator=g) * 0.8
    poses[:, :, 6:9] = 0.0                                         # an exactly zero pose
    return (poses, torch.randn(batch, 300, generator=g), torch.randn(batch, t, 100, generator=g),
            torch.randn(batch, t, 3, generator=g))


@pytest.mark.parametrize("use_b,use_e,mask", [(1, 1, ALL_JOINTS), (0, 0, MOTION_REP_JOINTS), (0, 1, ALL_JOINTS)])
def test_fk_bound_accepts_fp32(body, use_b, use_e, mask):
    poses, betas, expr, _ = _fk_inputs(11)
    args = (poses, betas if use_b else None, expr if use_e else None)
    outs = _fk32(*args, mask, body._tables)
    assert _fk_ok(outs, pb.smplx_fk(*args, mask, body._tables, outs[0], outs[1]))


@pytest.mark.parametrize("bug", ["no_eps", "drop_expr99", "absolute_offset"])
def test_fk_bound_rejects(body, bug):
    poses, betas, expr, _ = _fk_inputs(12)
    mask = MOTION_REP_JOINTS if bug == "no_eps" else ALL_JOINTS    # masked joints and joint 3 get a zero pose
    good = _fk32(poses, betas, expr, mask, body._tables)
    bad = _fk32(poses, betas, expr, mask, body._tables, bug)
    # the teacher-forced reference is formed from the outputs it checks, as on the GPU
    assert _fk_ok(good, pb.smplx_fk(poses, betas, expr, mask, body._tables, good[0], good[1]))
    assert not _fk_ok(bad, pb.smplx_fk(poses, betas, expr, mask, body._tables, bad[0], bad[1]))


def test_fk_transl_add_bound(body):
    poses, betas, expr, transl = _fk_inputs(13)
    joints, _, _ = _fk32(poses, betas, expr, ALL_JOINTS, body._tables)
    want, bound = pb.transl_add(joints, transl)
    assert pb.within(joints + transl.reshape(-1, 1, 3), want, bound)
    clip0 = transl[:1].expand_as(transl).reshape(-1, 1, 3)
    assert not pb.within(joints + clip0, want, bound)


def _skin32(v_posed, n_verts, csr, rel, transl, t, bug=None):
    """fp32 restatement of smplx_skin_kernel.  bug: 'drop_last' (each vertex's last CSR entry skipped),
    'transl_clip0' (every frame adds clip 0's transl)."""
    row_ptr, col, val = csr
    rows = v_posed.shape[0]
    A = rel.reshape(rows, 55, 12)
    T = torch.zeros(rows, n_verts, 12)
    for v in range(n_verts):
        e1 = int(row_ptr[v + 1]) - (1 if bug == "drop_last" else 0)
        for e in range(int(row_ptr[v]), e1):
            T[:, v] = T[:, v] + val[e] * A[:, int(col[e])]
    x = v_posed[:, :3 * n_verts].reshape(rows, n_verts, 3)
    d = torch.zeros(rows, 1, 3)
    if transl is not None:
        tr = transl[:1].expand_as(transl) if bug == "transl_clip0" else transl
        d = tr.reshape(rows, 1, 3)
    out = torch.stack([T[..., 4 * c] * x[..., 0] + T[..., 4 * c + 1] * x[..., 1] + T[..., 4 * c + 2] * x[..., 2]
                       + T[..., 4 * c + 3] + d[..., c] for c in range(3)], -1)
    return out.reshape(rows, 3 * n_verts)


@pytest.mark.parametrize("bug", ["drop_last", "transl_clip0"])
def test_skin_bound_accepts_fp32_and_rejects_bugs(body, bug):
    poses, betas, expr, transl = _fk_inputs(14)
    batch, t = poses.shape[:2]
    _, rel, _ = _fk32(poses, betas, expr, ALL_JOINTS, body._tables)
    nv = 64
    csr = tuple(x.clone() for x in body.skin_csr)
    csr = (csr[0][:nv + 1], csr[1], csr[2])
    v_posed = torch.randn(batch * t, 3 * nv, generator=_gen(15))
    want, bound = pb.smplx_skin(v_posed, nv, csr, rel, transl, t)
    assert pb.within(_skin32(v_posed, nv, csr, rel, transl, t), want, bound)
    assert not pb.within(_skin32(v_posed, nv, csr, rel, transl, t, bug), want, bound)

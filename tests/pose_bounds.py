"""float64 references with per-element error bounds for the pose and body-model kernels: the rotation conversions,
the DisCo mix and the motion representation (pm_pose.cu) and SMPL-X forward kinematics and skinning (pm_body.cu).

Each function takes the fp32 operands the kernel received (on any device) and returns float64 (want, bound):
|got - want| <= bound must hold for every output element.  The bounds are carried through the kernel's source
operation by operation (a running error analysis): every fp32 quantity q of the kernel is a `_V` holding the float64
value v of the same formula in exact arithmetic and e >= |q - v|.  The rules, for computed operands within e_a, e_b
of a, b:

* a + b, a - b: e_a + e_b, then the rounding of the result, U (|v| + e).
* a * b: |a| e_b + |b| e_a + e_a e_b, then U (|v| + e) + 2^-150 (a product may underflow).
* a / b: (e_a + |v| e_b) / (|b| - e_b) (infinite where the interval of b holds 0), then the rounding.
* sqrtf / sqrt_pos of an argument a +- e_a: the interval [sqrt(max(a - e_a, 0)), sqrt(max(a + e_a, 0))] - never
  linearised, so an argument within its bound of 0 (the near-pi quaternion components) gets its true sqrt(e_a) -
  then one rounding (sqrtf is correctly rounded).
* fmaxf(a, c), negation, * 0.5f and * 2.f: exact.
* expf, sinf, cosf, sincosf: 2 ulp (<= 4 U relative + 2 * 2^-149 absolute), atan2f 3 ulp, after the function's
  Lipschitz bound times e (CUDA math guide; the library is built without fast-math, so these are the libdevice
  functions, and sqrtf and '/' are correctly rounded).

Compile flags.  pm_pose.cu is built with -fmad=false (pantomatrix_b200/build.py EXTRA): one rounding per operation
in source order, exactly the rules above.  pm_body.cu allows contraction: a * b + c may be one fma, which drops the
product's rounding and keeps the sum's, so the separate-form bound counted here covers both forms.

Notation and the shared helpers (U, gamma, SECOND, within, bound_fraction) are those of tests/simt_bounds.py."""
import math

import numpy as np
import torch

from simt_bounds import SECOND, U, bound_fraction, gamma, within  # noqa: F401  (re-exported for the tests)

TINY = 2.0 ** -150                    # absolute part of a rounding that underflows (half the least subnormal)
SUB = 2.0 ** -149                     # one ulp of the subnormal range
F32 = lambda x: float(np.float32(x))  # the fp32 value of a source-code literal such as 1e-12f
EPS_NORM, EPS_BRANCH, EPS_RODRIGUES = F32(1e-12), F32(1e-6), F32(1e-8)


class _V:
    """An fp32 quantity of the kernel: float64 value v of its formula in exact arithmetic, and e >= |computed - v|."""
    __slots__ = ("v", "e")

    def __init__(self, v, e=None):
        self.v = v
        self.e = torch.zeros_like(v) if e is None else e

    def __add__(self, o):
        return _round(self.v + o.v, self.e + o.e, 0.0)

    def __sub__(self, o):
        return _round(self.v - o.v, self.e + o.e, 0.0)

    def __mul__(self, o):
        return _round(self.v * o.v, self.v.abs() * o.e + o.v.abs() * self.e + self.e * o.e, TINY)

    def __truediv__(self, o):
        v = self.v / o.v
        den = o.v.abs() - o.e
        e = torch.where(den > 0, (self.e + v.abs() * o.e) / den.clamp_min(1e-300), torch.full_like(v, math.inf))
        return _round(v, e, TINY)

    def __neg__(self):
        return _V(-self.v, self.e)

    def scale(self, c):
        """* 0.5f or * 2.f: exact."""
        return _V(self.v * c, self.e * abs(c))


def _round(v, e, tiny):
    return _V(v, e + U * (v.abs() + e) + tiny)


def _const(c, like):
    return _V(torch.full_like(like, c))


def _sqrt(a):
    """sqrtf(a) or sqrt_pos(a) (P.py:10-14: a > 0 ? sqrtf(a) : 0): the computed argument lies in [a - e, a + e], so
    the result lies in [sqrt(max(a - e, 0)), sqrt(max(a + e, 0))]; then one correctly rounded sqrt."""
    v = a.v.clamp_min(0).sqrt()
    hi = (a.v + a.e).clamp_min(0).sqrt()
    lo = (a.v - a.e).clamp_min(0).sqrt()
    return _round(v, torch.maximum(hi - v, v - lo), 0.0)


def _fmax(a, c):
    return _V(a.v.clamp_min(c), a.e)


def _func(v, lip_e, ulps):
    """A libdevice function of `ulps` ulp whose exact value at the exact argument is v, moved by at most lip_e by the
    argument's error: ulps * 2^-23 relative (= 2 ulps U) and ulps subnormal ulps absolute."""
    return _V(v, lip_e + 2 * ulps * U * (v.abs() + lip_e) + ulps * SUB)


def _sumsq(a, b, c):
    return a * a + b * b + c * c


def _sin_half_over_angle(half, ang):
    """sin_half_over_angle (pm_pose.cu, P.py:35-43): |ang| < 1e-6f ? 0.5f - (ang * ang) / 48.f : sinf(half) / ang, with
    ang = 2 half exactly at both call sites.  Both branches stand for f(h) = sin(h) / (2 h) (f(0) = 1/2).
    * Moving h by e_h moves f by at most L e_h, L = (h + e_h) / 6: f'(h) = (h cos h - sin h) / (2 h^2) and
      |h cos h - sin h| = |int_0^h t sin t dt| <= h^3 / 3.
    * sinf branch: sinf 2 ulp (4 U) and the division (U): 5 U of f at the computed h.
    * Taylor branch: q = fl(fl(ang^2) / 48) <= 2e-14 with 2 roundings, then 0.5f - q (one rounding, U / 2 <= U f):
      under 5 U of f as well, plus the truncation |0.5 - a^2/48 - f| <= a^4 / 3840, counted where the interval of ang
      reaches below 1e-6f (where the branch can be taken).
    So e_s = L e_h + 5 U (f + L e_h) (+ the truncation)."""
    h = half.v
    f = torch.where(h > 0, torch.sin(h) / (2 * h).clamp_min(1e-300), torch.full_like(h, 0.5))
    lip = (h + half.e) / 6 * half.e
    e = lip + 5 * U * (f + lip)
    taylor = (ang.v - ang.e) < EPS_BRANCH
    e = e + torch.where(taylor, (ang.v + ang.e) ** 4 / 3840, torch.zeros_like(e))
    return _V(f, e)


# ------------------------------------------------------------------------------------------------------------------
# rotation conversions (pm_pose.cu: rot6d_to_aa, aa_to_rot6d), -fmad=false
# ------------------------------------------------------------------------------------------------------------------


def rot6d_to_aa(d6):
    """Reference and bound of the device function rot6d_to_aa (pm_pose.cu, P.py:49-58 then 16-44), which both
    pose_compose_kernel and rot6d_to_aa_kernel run.  d6 (..., 6) fp32.  -fmad=false: one rounding per operation, in
    source order.  Stage by stage:

    * Gram-Schmidt: n1 = fmaxf(sqrtf(d0 d0 + d1 d1 + d2 d2), 1e-12f) (three products, two additions, the sqrt interval
      and its rounding; fmaxf is exact and 1-Lipschitz), b1 = d[0:3] / n1, dot = b1x d3 + b1y d4 + b1z d5,
      b2 = d[3:6] - dot b1, n2 = fmaxf(sqrtf(|b2|^2), 1e-12f), b2 /= n2.  Where the interval of n2 holds 0 (collinear
      or zero columns) the division's bound is infinite: the direction of b2 is the rounding noise's, and only a
      finite output is required there.
    * b3 = b1 x b2: two products and a subtraction per component.
    * The quaternion: w = 0.5f sqrt_pos(((1 + m00) + m11) + m22) and x, y, z with the signs of P.py:23-26, each sum
      left to right and its sqrt_pos by the interval rule.
    * The three sign decisions: sign_like(x, b3y - b2z), (y, b1z - b3x), (z, b2x - b1y).  A decision is taken from
      float64 where the difference lies farther from 0 than its bound; elsewhere both signs are candidates
      (`decided` False).  A sign flips only its own output component and no bound, so "the three outputs lie within
      bound of one of the <= 8 candidate combinations" is "each undecided output lies within bound of +-want":
      pick_signs applies it.
    * n = sqrtf(x x + y y + z z); half = atan2f(n, w): atan2 has gradient of norm 1 / r (r = |(n, w)|), so a
      perturbation of at most delta = e_n + e_w moves it by at most delta / (r - delta) (pi / 2 where r <= delta:
      n, w >= 0 keep half in [0, pi / 2]), then 3 ulp (6 U).
    * ang = 2.f half (exact), s = sin_half_over_angle(half, ang) (_sin_half_over_angle), aa_i = x_i / s.
    Returns (want (..., 3), bound (..., 3), decided (..., 3) bool), float64 on d6's device."""
    d = [_V(d6[..., c].double()) for c in range(6)]
    n1 = _fmax(_sqrt(_sumsq(d[0], d[1], d[2])), EPS_NORM)
    b1x, b1y, b1z = d[0] / n1, d[1] / n1, d[2] / n1
    dot = b1x * d[3] + b1y * d[4] + b1z * d[5]
    b2x, b2y, b2z = d[3] - dot * b1x, d[4] - dot * b1y, d[5] - dot * b1z
    n2 = _fmax(_sqrt(_sumsq(b2x, b2y, b2z)), EPS_NORM)
    b2x, b2y, b2z = b2x / n2, b2y / n2, b2z / n2
    b3x = b1y * b2z - b1z * b2y
    b3y = b1z * b2x - b1x * b2z
    b3z = b1x * b2y - b1y * b2x
    m00, m11, m22 = b1x, b2y, b3z
    one = _const(1.0, d6[..., 0].double())
    w = _sqrt(one + m00 + m11 + m22).scale(0.5)
    q = [_sqrt(one + m00 - m11 - m22).scale(0.5), _sqrt(one - m00 + m11 - m22).scale(0.5),
         _sqrt(one - m00 - m11 + m22).scale(0.5)]
    diffs = [b3y - b2z, b1z - b3x, b2x - b1y]
    decided = torch.stack([df.v.abs() > df.e for df in diffs], -1)
    q = [_V(torch.where(df.v < 0, -c.v, c.v), c.e) for c, df in zip(q, diffs)]
    n = _sqrt(_sumsq(*q))
    r = torch.hypot(n.v, w.v)
    delta = n.e + w.e
    e_half = torch.where(r > delta, delta / (r - delta).clamp_min(1e-300), torch.full_like(r, math.pi / 2))
    half = _func(torch.atan2(n.v, w.v), e_half.clamp_max(math.pi / 2 + 1e-6), 3)
    s = _sin_half_over_angle(half, half.scale(2.0))
    aa = [c / s for c in q]
    return (torch.stack([a.v for a in aa], -1), torch.stack([a.e for a in aa], -1) * SECOND, decided)


def pick_signs(got, want, decided):
    """want with each undecided component given the sign of the candidate nearer to got (see rot6d_to_aa)."""
    flip = (got.double() - want).abs() > (got.double() + want).abs()
    return torch.where(~decided & flip, -want, want)


def _aa_to_rot6d(a):
    """aa_to_rot6d (pm_pose.cu, P.py:63-104) on three _V components: the list of the six outputs."""
    ang = _sqrt(_sumsq(*a))
    half = ang.scale(0.5)
    s = _sin_half_over_angle(half, ang)
    # cosf: 1-Lipschitz (tighter: |sin| + e_h), 2 ulp
    r = _func(torch.cos(half.v), (torch.sin(half.v).abs() + half.e).clamp_max(1.0) * half.e, 2)
    i, j, k = a[0] * s, a[1] * s, a[2] * s
    two_s = _const(2.0, r.v) / (r * r + i * i + j * j + k * k)
    one = _const(1.0, r.v)
    return [one - two_s * (j * j + k * k), two_s * (i * j - k * r), two_s * (i * k + j * r),
            two_s * (i * j + k * r), one - two_s * (i * i + k * k), two_s * (j * k - i * r)]


def aa_to_rot6d(aa):
    """Reference and bound of the device function aa_to_rot6d (pm_pose.cu, P.py:63-104): pose_compose's motion4inf
    columns (fed the kernel's own axis-angle) and motion_rep's rot6d columns.  aa (..., 3) fp32.  -fmad=false, in
    source order: ang = sqrtf(a0 a0 + a1 a1 + a2 a2) (the sqrt interval), half = 0.5f ang (exact),
    s = sin_half_over_angle(half, ang), r = cosf(half) (|sin| <= 1 Lipschitz, 2 ulp), (i, j, k) = a s,
    two_s = 2.0f / (((r r + i i) + j j) + k k), then the six outputs, e.g. o0 = 1.f - two_s (j j + k k) and
    o1 = two_s (i j - k r), each product, sum and difference one rounding.  The exact values are the rotation
    matrix's first two rows (r^2 + i^2 + j^2 + k^2 = 1 in exact arithmetic).
    Returns (want (..., 6), bound (..., 6)) float64."""
    o = _aa_to_rot6d([_V(aa[..., c].double()) for c in range(3)])
    return torch.stack([x.v for x in o], -1), torch.stack([x.e for x in o], -1) * SECOND


# which part / slot of pose_compose feeds each SMPL-X joint, from the reference's joint lists (oracle/emage_oracle.py)
def joint_sources():
    """{joint: (part, column offset)} of pose_compose: part in ('upper', 'lower', 'hands', 'face')."""
    from oracle import emage_oracle as O
    src = {}
    for part, joints in (("upper", O.UPPER_JOINTS), ("lower", O.LOWER_JOINTS), ("hands", O.HANDS_JOINTS)):
        for slot, j in enumerate(joints):
            src[j] = (part, 6 * slot)
    src[22] = ("face", 0)                                          # the jaw: face[:6] (M.py:181)
    return src


def pose_compose(face, upper, hands, lower):
    """Reference and bound of ops.pose_compose (pose_compose_kernel, pm_pose.cu): the (bs, t, D) decoder outputs, each
    may be None.  Returns {"axis_angle": (want (bs, t, 165), bound, decided (bs, t, 165))} for the rotation of every
    joint with a present part (rot6d_to_aa) and an exact 0 for the others (eyes, absent parts).  The motion4inf and copy
    columns are checked by pose_compose_rest on the kernel's own axis-angle."""
    parts = dict(face=face, upper=upper, hands=hands, lower=lower)
    ref = next(p for p in parts.values() if p is not None)
    shp = ref.shape[:2]
    want = torch.zeros(*shp, 55, 3, dtype=torch.float64, device=ref.device)
    bound = torch.zeros_like(want)
    decided = torch.ones_like(want, dtype=torch.bool)
    for j, (part, off) in joint_sources().items():
        if parts[part] is not None:
            want[:, :, j], bound[:, :, j], decided[:, :, j] = rot6d_to_aa(parts[part][:, :, off:off + 6])
    flat = lambda x: x.reshape(*shp, 165)
    return flat(want), flat(bound), flat(decided)


def pose_compose_rest(face, lower, axis_angle):
    """The other outputs of pose_compose_kernel, from the kernel's own axis_angle (bs, t, 165): motion4inf
    (bs, t, 337) = aa_to_rot6d of each joint (reference and bound) then lower[54:61] (or 0) copied, and expression =
    face[6:] (or 0) copied.  Returns ((want, bound) of motion4inf, exact expression)."""
    bs, t = axis_angle.shape[:2]
    w6, b6 = aa_to_rot6d(axis_angle.reshape(bs, t, 55, 3))
    tail = (lower[:, :, 54:].double() if lower is not None
            else torch.zeros(bs, t, 7, dtype=torch.float64, device=axis_angle.device))
    want = torch.cat([w6.reshape(bs, t, 330), tail], -1)
    bound = torch.cat([b6.reshape(bs, t, 330), torch.zeros_like(tail)], -1)
    expr = face[:, :, 6:] if face is not None else torch.zeros(bs, t, 100, device=axis_angle.device)
    return (want, bound), expr


# ------------------------------------------------------------------------------------------------------------------
# DisCo content mix (pm_pose.cu: softmax2_mix_kernel), -fmad=false
# ------------------------------------------------------------------------------------------------------------------


def softmax2_mix(sel, c1, c2):
    """Reference and bound of ops.softmax2_mix(sel, c1, c2) (softmax2_mix_kernel, pm_pose.cu): sel (..., 2),
    c1, c2 (..., ch).  -fmad=false, in source order:
    * m = fmaxf(a, b) (exact); a - m and b - m: one is exactly 0, the other one rounding.
    * ea, eb = expf(.): exp moves by exp(t) expm1(e_t) for an argument error e_t, then 2 ulp.  A gap beyond ~104
      underflows expf to 0 or a subnormal: the 2 subnormal ulps of _func cover it, and the result is then the other
      operand's column up to the roundings below.
    * s = ea + eb, then ea / s, eb / s, the two products and the sum: one rounding each.
    Returns (want, bound) float64 of c1's shape."""
    a, b = _V(sel[..., 0:1].double()), _V(sel[..., 1:2].double())
    m = _V(torch.maximum(a.v, b.v))
    ta, tb = a - m, b - m

    def exp(t):
        v = torch.exp(t.v)
        return _func(v, v * torch.expm1(t.e), 2)

    ea, eb = exp(ta), exp(tb)
    s = ea + eb
    out = (ea / s) * _V(c1.double()) + (eb / s) * _V(c2.double())
    return out.v, out.e * SECOND


# ------------------------------------------------------------------------------------------------------------------
# motion representation (pm_pose.cu: motion_rep_kernel), -fmad=false
# ------------------------------------------------------------------------------------------------------------------


def motion_rep(poses, joints, dt, two_dt):
    """Reference and bound of ops.motion_rep(poses, joints, dt, two_dt, out) (motion_rep_kernel, pm_pose.cu): poses
    (batch, t, 165) (any view), joints (batch, t, 55, 3), dt and two_dt the fp32 values the kernel received.  Per
    (frame, joint) the 15 columns [position | velocity | rot6d | angular velocity]:
    * position: a copy of joints, exact (bound 0).
    * velocity: (joints[hi] - joints[lo]) / den, hi = min(tt + 1, t - 1), lo = max(tt - 1, 0), den = dt at both clip
      ends and two_dt inside: a subtraction and a division, one rounding each.
    * rot6d: aa_to_rot6d of the frame's pose.
    * angular velocity: the velocity formula on the poses.
    Returns (want, bound) float64 (batch, t, 825)."""
    batch, t = poses.shape[:2]
    dev = poses.device
    P = poses.double().reshape(batch, t, 55, 3)
    J = joints.double().reshape(batch, t, 55, 3)
    tt = torch.arange(t, device=dev)
    hi, lo = (tt + 1).clamp_max(t - 1), (tt - 1).clamp_min(0)
    ends = (tt == 0) | (tt == t - 1)
    den = torch.full((t,), F32(two_dt), dtype=torch.float64, device=dev)
    den[ends] = F32(dt)
    den = _V(den[None, :, None, None].expand(batch, t, 55, 3))
    vel = (_V(J[:, hi]) - _V(J[:, lo])) / den
    ang = (_V(P[:, hi]) - _V(P[:, lo])) / den
    r6, b6 = aa_to_rot6d(poses.reshape(batch, t, 55, 3))
    want = torch.cat([J, vel.v, r6, ang.v], -1).reshape(batch, t, 825)
    bound = torch.cat([torch.zeros_like(J), vel.e * SECOND, b6, ang.e * SECOND], -1).reshape(batch, t, 825)
    return want, bound


# ------------------------------------------------------------------------------------------------------------------
# SMPL-X forward kinematics and skinning (pm_body.cu), contraction allowed
# ------------------------------------------------------------------------------------------------------------------


def _frames(x, batch, t, ch):
    """(batch * t, ch) float64 of a (batch, t, ch) view, or None."""
    return None if x is None else x.double().reshape(batch * t, ch)


def _rodrigues(r):
    """Stage 2 of smplx_fk_kernel (smplx batch_rodrigues) on the three _V components of r = pose + pose_mean:
    e = r + 1e-8f, ang = sqrtf(ex ex + ey ey + ez ez), k = r / ang, sincosf(ang) (1-Lipschitz, 2 ulp each),
    omc = 1.f - c, then the nine entries, e.g. R0 = 1.f + omc (-kz kz - ky ky), R1 = -s kz + omc (kx ky): each product
    and sum one rounding (the separate form; a contracted fma only drops a product's rounding).  The list of 9."""
    eps = _const(EPS_RODRIGUES, r[0].v)
    ex, ey, ez = r[0] + eps, r[1] + eps, r[2] + eps
    ang = _sqrt(_sumsq(ex, ey, ez))
    kx, ky, kz = r[0] / ang, r[1] / ang, r[2] / ang
    s = _func(torch.sin(ang.v), ang.e, 2)
    c = _func(torch.cos(ang.v), ang.e, 2)
    one = _const(1.0, ang.v)
    omc = one - c
    return [one + omc * (-kz * kz - ky * ky), -s * kz + omc * (kx * ky), s * ky + omc * (kx * kz),
            s * kz + omc * (kx * ky), one + omc * (-kz * kz - kx * kx), -s * kx + omc * (ky * kz),
            -s * ky + omc * (kx * kz), s * kx + omc * (ky * kz), one + omc * (-ky * ky - kx * kx)]


def rest_joints(betas, expression, batch, t, j_template, j_dirs):
    """Stage 3 of smplx_fk_kernel: J = j_template + j_dirs^T [betas | expression] of every frame, as the fmaf chain
    `acc = fmaf(w, coef, acc)` over k in [k0, k1): k0 = 0 with betas, else 300; k1 = 400 with expression, else 300.
    An n-step fma chain errs by at most gamma(n) (|j_template| + sum |w coef|).
    Returns _V (batch * t, 165)."""
    rows = batch * t
    jt, jd = j_template.double(), j_dirs.double()
    coef = torch.zeros(rows, 400, dtype=torch.float64, device=jt.device)
    if betas is not None:
        coef[:, :300] = betas.double()[:, None].expand(batch, t, 300).reshape(rows, 300)
    if expression is not None:
        coef[:, 300:] = _frames(expression, batch, t, 100)
    k0, k1 = (0 if betas is not None else 300), (400 if expression is not None else 300)
    v = jt + coef[:, k0:k1] @ jd[k0:k1]
    e = gamma(k1 - k0) * (jt.abs() + coef[:, k0:k1].abs() @ jd[k0:k1].abs())
    return _V(v, e), coef


def smplx_fk(poses, betas, expression, joint_mask, tables, joints, rel):
    """Teacher-forced reference and bound of ops.smplx_fk (smplx_fk_kernel, pm_body.cu; contraction allowed) called
    with transl=None, so that `joints` (rows, 55, 3) is each joint's global translation G_t and rel (rows, 55, 12)
    holds its global rotation G_R in the entries with (m & 3) != 3.  Every joint's G_j is compared with
    G_parent [R_j | J_j - J_parent] formed in float64 from the KERNEL'S OWN G_parent, so each level is held to one
    level's error and an error that grows with depth cannot hide:
    * R_j: _rodrigues of r = (joint in mask ? pose : 0) + pose_mean (that addition one rounding).
    * J: rest_joints.
    * root: G_R = R (copied), G_t = J_root.  Other joints: G_R[row][c] = p0 R[c] + p1 R[3 + c] + p2 R[6 + c] with
      the exact parent rotation p, and G_t[row] = p0 t0 + p1 t1 + p2 t2 + gp_t[row] with t = J_j - J_parent (one
      rounding each): the errors of R and t through the exact p, plus the dot products' roundings.
    * rel's translation: G_t - (G_R[row] . J_j): the exact kernel G, J's error, four roundings.
    * feat (GEMM operand row): [coef | R_j - I of joints 1..54]: coef copied exactly; the diagonal's `R[m] - 1.f` one
      more rounding.
    Returns {"rot": (rows, 55, 9), "trans": (rows, 55, 3), "rel_t": (rows, 55, 3), "feat": (rows, 886)}, each
    (want, bound); fk_outputs gives the kernel's tensors in the same layout."""
    jt, jd, pmean, parents, _, _ = tables
    batch, t = poses.shape[:2]
    rows = batch * t
    dev = poses.device
    keep = torch.tensor([(int(joint_mask) >> j) & 1 for j in range(55)], dtype=torch.float64, device=dev)
    p = _frames(poses, batch, t, 165).reshape(rows, 55, 3) * keep[:, None]
    pm = pmean.double().reshape(55, 3)
    R = _rodrigues([_V(p[..., c]) + _V(pm[:, c].expand(rows, 55)) for c in range(3)])
    J, coef = rest_joints(betas, expression, batch, t, jt, jd)
    Jv, Je = J.v.reshape(rows, 55, 3), J.e.reshape(rows, 55, 3)
    GR = rel.double().reshape(rows, 55, 3, 4)[..., :3]
    Gt = joints.double().reshape(rows, 55, 3)
    par = [int(x) for x in parents.tolist()]
    pidx = torch.tensor([max(x, 0) for x in par], device=dev)
    is_root = torch.tensor([x < 0 for x in par], device=dev)
    PR, Pt = GR[:, pidx], Gt[:, pidx]                              # the kernel's parent transforms
    Jj = [_V(Jv[..., c], Je[..., c]) for c in range(3)]
    Jp = [_V(Jv[:, pidx, c], Je[:, pidx, c]) for c in range(3)]
    tv = [Jj[c] - Jp[c] for c in range(3)]
    rot, trans = [], []
    for row in range(3):
        P = [_V(PR[..., row, k]) for k in range(3)]
        for c in range(3):
            rot.append(P[0] * R[c] + P[1] * R[3 + c] + P[2] * R[6 + c])
        trans.append(P[0] * tv[0] + P[1] * tv[1] + P[2] * tv[2] + _V(Pt[..., row]))
    root = is_root[None, :]
    rot_v = torch.stack([torch.where(root, R[m].v, rot[m].v) for m in range(9)], -1)
    rot_e = torch.stack([torch.where(root, R[m].e, rot[m].e) for m in range(9)], -1)
    tr_v = torch.stack([torch.where(root, Jv[..., c], trans[c].v) for c in range(3)], -1)
    tr_e = torch.stack([torch.where(root, Je[..., c], trans[c].e) for c in range(3)], -1)
    rel_t = []
    for row in range(3):
        g = [_V(GR[..., row, k]) for k in range(3)]
        rel_t.append(_V(Gt[..., row]) - (g[0] * Jj[0] + g[1] * Jj[1] + g[2] * Jj[2]))
    one = _const(1.0, R[0].v)
    fe = [R[m] - one if m % 4 == 0 else R[m] for m in range(9)]
    feat_v = torch.cat([coef, torch.stack([x.v for x in fe], -1)[:, 1:].reshape(rows, 486)], 1)
    feat_e = torch.cat([torch.zeros_like(coef), torch.stack([x.e for x in fe], -1)[:, 1:].reshape(rows, 486)], 1)
    return {"rot": (rot_v, rot_e * SECOND), "trans": (tr_v, tr_e * SECOND),
            "rel_t": (torch.stack([x.v for x in rel_t], -1), torch.stack([x.e for x in rel_t], -1) * SECOND),
            "feat": (feat_v, feat_e * SECOND)}


def fk_outputs(joints, rel, feat):
    """The kernel's outputs in smplx_fk's layout."""
    rows = joints.shape[0]
    r = rel.reshape(rows, 55, 3, 4)
    return {"rot": r[..., :3].reshape(rows, 55, 9), "trans": joints.reshape(rows, 55, 3), "rel_t": r[..., 3],
            "feat": feat[:, :886]}


def transl_add(joints, transl):
    """Stage 5's `v += transl[...]`: the joints of a call with transl from those of the same call without it (one
    rounding).  joints (rows, 55, 3), transl (batch, t, 3) any view.  Returns (want, bound)."""
    rows = joints.shape[0]
    out = _V(joints.double().reshape(rows, 55, 3)) + _V(transl.double().reshape(rows, 1, 3).expand(rows, 55, 3))
    return out.v, out.e * SECOND


def smplx_skin(v_posed, n_verts, csr, rel, transl, t):
    """Reference and bound of ops.smplx_skin (smplx_skin_kernel, pm_body.cu; contraction allowed) given the v_posed
    rows (rows, >= 3 n_verts) it was called on and the rel (rows, 55, 12) it read.  Per vertex:
    * T = sum_e w_e A[col_e]: the fmaf chain over the vertex's CSR entries, n_v = row_ptr[v + 1] - row_ptr[v] steps
      from 0: gamma(n_v) sum_e |w_e A[col_e]| per entry.
    * out_c = T[c4] x + T[c4 + 1] y + T[c4 + 2] z + T[c4 + 3] + d_c (d = the frame's transl, or 0.f): three products
      and four additions, left to right, one rounding each, carried with T's errors by the running rules.
    Returns (want, bound) float64 (rows, 3 n_verts)."""
    row_ptr, col, val = (x.long() if x.dtype == torch.int32 else x for x in csr)
    rows = v_posed.shape[0]
    dev = v_posed.device
    row_ptr = row_ptr[:n_verts + 1]
    nnz = row_ptr[1:] - row_ptr[:-1]
    vert = torch.repeat_interleave(torch.arange(n_verts, device=dev), nnz)
    e0, e1 = int(row_ptr[0]), int(row_ptr[-1])
    W = torch.zeros(n_verts, 55, dtype=torch.float64, device=dev)
    W.index_put_((vert, col[e0:e1]), val[e0:e1].double(), accumulate=True)
    A = rel.double().reshape(rows, 55, 12)
    T = torch.einsum("vj,rjm->rvm", W, A)
    eT = torch.einsum("vj,rjm->rvm", W.abs(), A.abs()) * torch.tensor(
        [gamma(int(n)) for n in nnz.tolist()], dtype=torch.float64, device=dev)[None, :, None]
    x = v_posed[:, :3 * n_verts].double().reshape(rows, n_verts, 3)
    X = [_V(x[..., k]) for k in range(3)]
    if transl is not None:
        d = transl.double().reshape(rows, 3)[:, None, :].expand(rows, n_verts, 3)
    else:
        d = torch.zeros(rows, n_verts, 3, dtype=torch.float64, device=dev)
    out = []
    for c in range(3):
        Tc = [_V(T[..., 4 * c + k], eT[..., 4 * c + k]) for k in range(4)]
        out.append(Tc[0] * X[0] + Tc[1] * X[1] + Tc[2] * X[2] + Tc[3] + _V(d[..., c]))
    want = torch.stack([o.v for o in out], -1).reshape(rows, 3 * n_verts)
    bound = torch.stack([o.e for o in out], -1).reshape(rows, 3 * n_verts)
    return want, bound * SECOND

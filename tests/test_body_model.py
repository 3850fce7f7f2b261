"""SMPL-X body model without a GPU: invariants of the float64 restatement, the restatement against the golden made by
the reference's own code, the float32 floor behind the GPU gates, model-file validation, the npz writer's pelvis
placement and the marshalling of the new kernel calls."""
import ctypes
import os

import numpy as np
import pytest
import torch

from body_cases import JOINT_GATE, VERTEX_GATE, full_arrays, random_poses, random_tree, small_arrays
from oracle.smplx_oracle import SmplxRestatement, forward_poses, rodrigues
from pantomatrix_b200 import _lib, motion_io, ops
from pantomatrix_b200.body_model import MOTION_REP_JOINTS, SmplxBodyModel
from synthetic_models import SMPLX_PARENTS, smplx_arrays, smplx_hash, write_smplx_npz

F64 = torch.float64


def _model(seed, parents, zero_means=True, n_verts=220):
    a = smplx_arrays(n_verts, seed, parents)
    if zero_means:
        a["hands_meanl"], a["hands_meanr"] = np.zeros(45), np.zeros(45)
    return a, SmplxRestatement(a, F64)


def _trees():
    rng = np.random.default_rng(5)
    return [SMPLX_PARENTS] + [random_tree(rng) for _ in range(3)]


@pytest.mark.parametrize("tree", range(4))
def test_restatement_invariants(tree):
    parents = _trees()[tree]
    a, m = _model(tree, parents)
    rng = np.random.default_rng(tree)
    n = 6
    betas, expr = torch.from_numpy(rng.normal(0, 1, (n, 300))), torch.from_numpy(rng.normal(0, 1, (n, 100)))
    zero = torch.zeros(n, 165, dtype=F64)
    j0, v0 = forward_poses(m, zero, betas, expr)
    # zero pose with zero hand means: the rest joints J_regressor @ v_shaped; no pose corrective, no skinning motion
    v_shaped = m.v_template + torch.einsum("bl,mkl->bmk", torch.cat([betas, expr], 1), m.shapedirs)
    torch.testing.assert_close(j0, torch.einsum("bik,ji->bjk", v_shaped, m.J_regressor), rtol=0, atol=1e-12)
    torch.testing.assert_close(v0, v_shaped, rtol=0, atol=1e-12)
    # a root rotation alone moves every joint and vertex rigidly about J[0]
    root = zero.clone()
    root[:, :3] = torch.from_numpy(rng.normal(0, 1.0, (n, 3)))
    j1, v1 = forward_poses(m, root, betas, expr)
    R = rodrigues(root[:, :3])
    about = lambda x: torch.einsum("bij,bvj->bvi", R, x - j0[:, :1]) + j0[:, :1]
    torch.testing.assert_close(j1, about(j0), rtol=0, atol=1e-12)
    torch.testing.assert_close(v1, about(v0), rtol=0, atol=1e-12)
    # bone lengths are preserved under any pose (to 1e-7: the 1e-8 added before the norm leaves |k| = 1 - O(1e-8), so
    # R is orthogonal only to that order, as in smplx)
    poses = torch.from_numpy(random_poses(rng, n, 1.5))
    j2, _ = forward_poses(m, poses, betas, expr)
    bone = lambda j: (j[:, 1:] - j[:, list(parents[1:])]).norm(dim=-1)
    torch.testing.assert_close(bone(j2), bone(j0), rtol=0, atol=1e-7)


def test_one_hot_skinning_row_moves_rigidly_with_its_joint():
    a, _ = _model(1, SMPLX_PARENTS)
    a["posedirs"] = np.zeros_like(a["posedirs"])        # v_posed = v_shaped: only skinning moves the vertex
    for v in range(4):
        a["weights"][v] = 0.0
        a["weights"][v, 18] = 1.0
    m = SmplxRestatement(a, F64)
    poses = torch.from_numpy(random_poses(np.random.default_rng(2), 5, 1.0))
    j0, v0 = forward_poses(m, torch.zeros(5, 165, dtype=F64))
    j1, v1 = forward_poses(m, poses)
    pts = lambda j, v: torch.cat([j[:, 18:19], v[:, :4]], 1)
    dist = lambda p: torch.cdist(p, p)
    torch.testing.assert_close(dist(pts(j1, v1)), dist(pts(j0, v0)), rtol=0, atol=1e-7)   # R orthogonal to ~1e-8
    assert (v1[:, :4] - v0[:, :4]).abs().max() > 1e-2          # it did move


def test_rodrigues_of_zero_is_exact_identity():
    for dt in (torch.float32, F64):
        r = rodrigues(torch.zeros(4, 3, dtype=dt))
        assert torch.equal(r, torch.eye(3, dtype=dt).expand(4, 3, 3))


def test_restatement_matches_golden_of_reference_code(golden_dir):
    g = np.load(os.path.join(golden_dir, "case_body.npz"))
    assert str(g["model_sha256"]) == smplx_hash(small_arrays()), "synthetic SMPL-X model differs from the golden's"
    m = SmplxRestatement(small_arrays(), F64)
    poses = torch.from_numpy(g["poses"]).double().reshape(-1, 165)
    keep = torch.tensor([(MOTION_REP_JOINTS >> j) & 1 for j in range(55)], dtype=F64).repeat_interleave(3)
    j, _ = forward_poses(m, poses * keep, vertices=False)
    want = torch.from_numpy(g["rep_position"]).double().reshape(-1, 55, 3)
    assert (j - want).abs().max() < 1e-6                    # float32 rounding of the reference's arithmetic
    assert np.array_equal(g["rep_axis_angle"], g["poses"])


def test_float32_floor_and_gates():
    """float32 vs float64 restatement on the full-size model; the GPU gates must be at least 4x this gap."""
    a = full_arrays()
    m64, m32 = SmplxRestatement(a, F64), SmplxRestatement(a, torch.float32)
    rng = np.random.default_rng(11)
    n = 16
    ins = [torch.from_numpy(x).float() for x in (random_poses(rng, n), rng.normal(0, 1, (n, 300)),
                                                 rng.normal(0, 1, (n, 100)), rng.normal(0, 1, (n, 3)))]
    j32, v32 = forward_poses(m32, *ins)
    j64, v64 = forward_poses(m64, *[x.double() for x in ins])
    gap_j, gap_v = float((j32.double() - j64).abs().max()), float((v32.double() - v64).abs().max())
    print(f"float32 floor: joints {gap_j:.3g} m, vertices {gap_v:.3g} m")
    assert 0 < gap_j and 0 < gap_v
    assert JOINT_GATE >= 4 * gap_j and VERTEX_GATE >= 4 * gap_v, (gap_j, gap_v)


def _save(path, a):
    np.savez(path, **a)
    return str(path)


def test_loader_validation(tmp_path):
    a = small_arrays()
    ok = SmplxBodyModel.from_npz(_save(tmp_path / "ok.npz", a), "cpu")
    assert ok.n_verts == a["v_template"].shape[0] and ok.j_dirs.shape == (400, 165) and ok.blend.w.shape == (1, 3 * ok.n_verts, 886)
    assert int(ok.level_start[-1]) == 55 and ok.n_levels == 11
    want = np.einsum("jv,vc->jc", a["J_regressor"], a["v_template"]).reshape(-1)
    np.testing.assert_allclose(ok.j_template.numpy(), want, rtol=1e-6, atol=1e-7)
    row_ptr, col, val = ok.skin_csr
    assert int(row_ptr[-1]) == col.numel() == val.numel() and (row_ptr[1:] - row_ptr[:-1]).max() <= 4
    cases = {
        "missing key": ({k: v for k, v in a.items() if k != "posedirs"}, "posedirs"),
        "wrong shape": ({**a, "J_regressor": a["J_regressor"][:, :-1]}, "J_regressor"),
        "few shape components": ({**a, "shapedirs": a["shapedirs"][:, :, :300]}, "shape components"),
        "bad tree": ({**a, "kintree_table": np.stack([np.r_[-1, 2, np.zeros(53, np.int64)], np.arange(55)])}, "tree"),
    }
    for name, (arrays, msg) in cases.items():
        with pytest.raises(ValueError, match=msg):
            SmplxBodyModel.from_npz(_save(tmp_path / "bad.npz", arrays), "cpu")


def test_loader_accepts_sparse_j_regressor(tmp_path):
    import scipy.sparse
    a = dict(small_arrays())
    dense = SmplxBodyModel(a, "cpu")
    a["J_regressor"] = np.array(scipy.sparse.csc_matrix(a["J_regressor"]), dtype=object)
    np.savez(tmp_path / "sparse.npz", **a)
    sparse = SmplxBodyModel.from_npz(str(tmp_path / "sparse.npz"), "cpu")
    assert torch.equal(sparse.j_template, dense.j_template) and torch.equal(sparse.j_dirs, dense.j_dirs)


class _RestatementBodyModel:
    """The float32 restatement behind the body model's call convention (CPU)."""
    device = torch.device("cpu")

    def __init__(self, arrays):
        self.m = SmplxRestatement(arrays, torch.float32)

    def forward(self, poses, betas=None):
        j, _ = forward_poses(self.m, poses.reshape(-1, 165), betas=betas, vertices=False)
        return {"joints": j.reshape(*poses.shape[:2], 55, 3)}


def test_beat_format_save_places_the_pelvis_like_the_reference(tmp_path, golden_dir):
    g = np.load(os.path.join(golden_dir, "case_body.npz"))
    bm = _RestatementBodyModel(small_arrays())
    path = str(tmp_path / "out.npz")
    motion_io.beat_format_save(path, g["save_motion"], betas=g["betas"], trans=None, upsample=2, body_model=bm)
    out = np.load(path)
    assert out["trans"].dtype == g["save_trans"].dtype and np.array_equal(out["trans"], g["save_trans"])
    assert np.array_equal(out["betas"], g["betas"][0]) and out["poses"].shape == (24, 165)
    motion_io.beat_format_save(path, g["save_motion"], trans=None, upsample=2, body_model=bm)
    assert np.array_equal(np.load(path)["trans"], g["save_trans_zero_betas"])


def test_body_model_refuses_cpu_tensors_and_bad_inputs():
    m = SmplxBodyModel(small_arrays(), "cpu")
    with pytest.raises(_lib.PmError):
        m.forward(torch.zeros(1, 2, 165))
    with pytest.raises(_lib.PmError):
        m.motion_rep(torch.zeros(1, 2, 165))
    with pytest.raises(ValueError):
        m.forward(torch.zeros(2, 165))
    with pytest.raises(ValueError):
        m.forward(np.zeros((1, 2, 165), np.float32))


def test_ops_wrappers_marshal_valid_arguments(monkeypatch):
    """The body model's ops wrappers on CPU tensors with the library call replaced by a recorder (as in
    test_boundary.py): every argument converts to its declared ctypes type, in both plane formats."""
    calls = []

    def record(name, *args):
        sig = _lib.SIGNATURES[name]
        assert len(args) == len(sig), (name, len(args), len(sig))
        for i, (x, t) in enumerate(zip(args, sig)):
            if t is ctypes.c_void_p:
                assert x is None or isinstance(x, int), (name, i, type(x))
            elif t is ctypes.c_float:
                assert isinstance(x, float), (name, i, type(x))
            else:
                assert isinstance(x, int) and not isinstance(x, bool), (name, i, type(x))
                t(x)
        calls.append((name, args))

    monkeypatch.setattr(_lib, "call", record)
    monkeypatch.setattr(ops, "_chk", lambda t, dtype=torch.float32: t)
    monkeypatch.setattr(ops, "_stream", lambda: 0)
    monkeypatch.setattr(ops, "_PLANE_DTYPE", ops._PLANE_DTYPE)
    m = SmplxBodyModel(small_arrays(), "cpu")
    b, t, rows = 2, 5, 10
    wide = torch.zeros(b, 2 * t, 200)
    poses, expr, transl = wide[:, ::2, 7:172], torch.zeros(b, t, 100), torch.zeros(b, t, 3)
    for fmt, bit in (("bf16", 0), ("fp16", ops.FMT_F16)):
        ops.set_plane_format(fmt)
        calls.clear()
        joints = torch.empty(rows, 55, 3)
        rel = torch.empty(rows, 55, 12)
        planes = ops._new_planes(2, (1, rows), 886, "cpu")
        ops.smplx_fk(poses, torch.zeros(b, 300), expr, transl, MOTION_REP_JOINTS, m._tables, joints, rel, None, planes)
        ops.smplx_skin(torch.zeros(rows, 3 * m.n_verts + 2), m.n_verts, m.skin_csr, rel, transl, t)
        ops.motion_rep(poses, joints, 1 / 30, 2 / 30, torch.empty(b, t, 825))
        fk = dict(calls)["pm_smplx_fk_f32"]
        assert fk[1:3] == (poses.stride(0), poses.stride(1)) and fk[11] == MOTION_REP_JOINTS and fk[20] == 11
        assert fk[28] == 2 | bit and fk[23] is None

"""SMPL-X body model on the H100 against the float64 restatement (oracle/smplx_oracle.py) and against the golden made by
the reference's own motion-representation and writer code (tests/golden/case_body.npz).  Gates: tests/body_cases.py."""
import os
import subprocess
import sys
import wave

import numpy as np
import pytest
import torch

from body_cases import (JOINT_GATE, ROTATION_GATE, VELOCITY_GATE, VERTEX_GATE, full_arrays, masked, random_poses,
                        random_tree, small_arrays)
from helpers import check_tapgemm, use_precision
from oracle.smplx_oracle import SmplxRestatement, forward_poses
from simt_bounds import tapgemm_f32, within
from pantomatrix_b200 import _lib
from pantomatrix_b200.body_model import ALL_JOINTS, MOTION_REP_JOINTS, SmplxBodyModel
from synthetic_models import SMPLX_PARENTS, smplx_arrays

pytestmark = pytest.mark.gpu
DEV = "cuda"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _pair(arrays):
    return SmplxBodyModel(arrays, DEV), SmplxRestatement(arrays, torch.float64).to(DEV)


def _oracle(m64, poses, betas=None, expr=None, transl=None, mask=ALL_JOINTS, vertices=False, chunk=1200):
    """float64 joints (and vertices) of (B, T, ...) inputs, frame chunks to bound memory."""
    B, T = poses.shape[:2]
    flat = lambda x, c: None if x is None else x.double().reshape(-1, c)
    p = masked(flat(poses, 165), mask)
    b = None if betas is None else betas.double()[:, None].expand(B, T, 300).reshape(-1, 300)
    e, tr = flat(expr, 100), flat(transl, 3)
    js, vs = [], []
    for s in range(0, B * T, chunk):
        sl = slice(s, s + chunk)
        j, v = forward_poses(m64, p[sl], None if b is None else b[sl], None if e is None else e[sl],
                             None if tr is None else tr[sl], vertices=vertices)
        js.append(j)
        vs.append(v)
    j = torch.cat(js).view(B, T, 55, 3)
    return (j, torch.cat(vs).view(B, T, -1, 3)) if vertices else (j, None)


def _inputs(rng, B, T, strided):
    """float32 CUDA (poses, betas, expression, transl); strided=True gives views with clip / frame strides."""
    def put(x, c):
        x = torch.from_numpy(np.asarray(x, np.float32)).to(DEV).reshape(B, T, c)
        if not strided:
            return x
        wide = torch.zeros(B, 2 * T, c + 13, device=DEV)
        v = wide[:, ::2, 5:5 + c]
        v.copy_(x)
        return v
    poses = put(random_poses(rng, B * T), 165)
    betas = torch.from_numpy(rng.normal(0, 1, (B, 300)).astype(np.float32)).to(DEV)
    if strided:
        betas = torch.zeros(B, 320, device=DEV)[:, 10:310].copy_(betas)
    return poses, betas, put(rng.normal(0, 1, (B * T, 100)), 100), put(rng.normal(0, 1, (B * T, 3)), 3)


def test_fk_joints_against_float64():
    rng = np.random.default_rng(3)
    models = [("smplx", small_arrays())] + [(f"tree{i}", smplx_arrays(330, 10 + i, random_tree(rng))) for i in range(2)]
    worst = 0.0
    for name, arrays in models:
        bm, m64 = _pair(arrays)
        for (B, T) in ((1, 1), (1, 7), (32, 300)) if name == "smplx" else ((1, 7), (3, 40)):
            for strided in (False, True):
                poses, betas, expr, transl = _inputs(rng, B, T, strided)
                for use_b, use_e, use_t, mask in ((0, 0, 0, ALL_JOINTS), (1, 1, 1, ALL_JOINTS), (1, 0, 1, MOTION_REP_JOINTS),
                                                  (0, 1, 0, ALL_JOINTS)):
                    args = (betas if use_b else None, expr if use_e else None, transl if use_t else None)
                    joints, _, _ = bm._fk(poses, *args, mask, False)
                    want, _ = _oracle(m64, poses, *args, mask=mask)
                    err = float((joints.view(B, T, 55, 3).double() - want).abs().max())
                    worst = max(worst, err)
                    assert err <= JOINT_GATE, (name, B, T, strided, use_b, use_e, use_t, hex(mask), err)
    print(f"FK joints: max |err| {worst:.3g} m (gate {JOINT_GATE:g})")


def _fp32_gemm_bound_check(feat, lin, got):
    """fp32 SIMT blend GEMM: |err| <= (K + 2) 2^-24 (|A| |W| + |bias|) + 2^-24 |result|, every element
    (simt_bounds.tapgemm_f32)."""
    want, bound = tapgemm_f32(feat[:, :886].unsqueeze(0), lin.w, lin.b)
    assert within(got.unsqueeze(0), want, bound)


@pytest.mark.parametrize("precision", ["fp16x3", "bf16x6", "fp32"])
def test_vertices_full_model_against_float64(request, precision):
    use_precision(request, precision)
    bm, m64 = _pair(full_arrays())
    rng = np.random.default_rng(7)
    B, T = 32, 300
    poses, betas, expr, transl = _inputs(rng, B, T, strided=True)
    out = bm.forward(poses, betas, expr, transl, vertices=True)
    assert out["vertices"].shape == (B, T, bm.n_verts, 3)
    # the blend GEMM per element, on the operand the FK kernel wrote
    _, rel, operand = bm._fk(poses, betas, expr, transl, ALL_JOINTS, True)
    v_posed = bm._blend(operand, B * T)[:, :3 * bm.n_verts]
    if precision == "fp32":
        _fp32_gemm_bound_check(operand, bm.blend, v_posed)
    else:
        check_tapgemm(operand, bm.blend.packed(operand.nsplit), bm.blend.b, v_posed.unsqueeze(0), None, tag=precision,
                      rows_out=B * T)
    del v_posed, operand
    err_j = err_v = 0.0
    for c in range(0, B, 4):
        sl = slice(c, c + 4)
        wj, wv = _oracle(m64, poses[sl], betas[sl], expr[sl], transl[sl], vertices=True)
        err_j = max(err_j, float((out["joints"][sl].double() - wj).abs().max()))
        err_v = max(err_v, float((out["vertices"][sl].double() - wv).abs().max()))
        del wj, wv
    print(f"{precision}: joints {err_j:.3g} m, vertices {err_v:.3g} m over {B * T} frames")
    assert err_j <= JOINT_GATE and err_v <= VERTEX_GATE, (err_j, err_v)


def test_motion_rep_against_reference_golden(golden_dir):
    g = np.load(os.path.join(golden_dir, "case_body.npz"))
    bm = SmplxBodyModel(small_arrays(), DEV)
    poses = torch.from_numpy(g["poses"]).to(DEV)
    wide = torch.zeros(poses.shape[0], poses.shape[1], 170, device=DEV)
    for p in (poses, wide[:, :, 3:168].copy_(poses)):           # dense and strided
        rep = {k: v.cpu() for k, v in bm.motion_rep(p).items()}
        want = {k[4:]: torch.from_numpy(g[k]) for k in g.files if k.startswith("rep_")}
        assert torch.equal(rep["angular_velocity"], want["angular_velocity"])
        assert torch.equal(rep["axis_angle"], want["axis_angle"])
        assert (rep["rotation"] - want["rotation"]).abs().max() <= ROTATION_GATE
        assert (rep["position"] - want["position"]).abs().max() <= JOINT_GATE
        assert (rep["velocity"] - want["velocity"]).abs().max() <= VELOCITY_GATE
        v = rep["rep15d"].view(*rep["rep15d"].shape[:2], 55, 15)
        assert torch.equal(v[..., 12:15], want["angular_velocity"]) and rep["rep15d"].shape == want["rep15d"].shape
        assert (rep["rep15d"] - want["rep15d"]).abs().max() <= VELOCITY_GATE


def test_pipeline_outputs_in_place_and_cuda_graph_replay():
    from synthetic_models import build_product
    from oracle.weights import synth_audio
    from pantomatrix_b200.pipeline import CapturedPipeline
    model, vqm = build_product(seed=0, device=DEV)
    bs, n = 2, 70000
    pipe = CapturedPipeline(model, vqm, bs, n)
    _, pred = pipe(torch.from_numpy(synth_audio(bs, n, 99)).to(DEV))
    bm, m64 = _pair(full_arrays())
    aa, expr, trans = pred["motion_axis_angle"], pred["expression"], pred["trans"]
    betas = torch.from_numpy(np.random.default_rng(4).normal(0, 1, (bs, 300)).astype(np.float32)).to(DEV)
    ptrs = [x.data_ptr() for x in (aa, expr, trans)]
    eager = bm.forward(aa, betas, expr, trans, vertices=True)
    assert [x.data_ptr() for x in (aa, expr, trans)] == ptrs
    wj, wv = _oracle(m64, aa, betas, expr, trans, vertices=True)
    assert float((eager["joints"].double() - wj).abs().max()) <= JOINT_GATE
    assert float((eager["vertices"].double() - wv).abs().max()) <= VERTEX_GATE
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        captured = bm.forward(aa, betas, expr, trans, vertices=True)
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(captured["joints"], eager["joints"]) and torch.equal(captured["vertices"], eager["vertices"])


def test_edge_cases():
    bm = SmplxBodyModel(small_arrays(), DEV)
    with pytest.raises(ValueError):
        bm.forward(torch.zeros(0, 5, 165, device=DEV))
    with pytest.raises(ValueError):
        bm.motion_rep(torch.zeros(0, 5, 165, device=DEV))
    with pytest.raises(ValueError):
        bm.motion_rep(torch.zeros(2, 1, 165, device=DEV))
    with pytest.raises(ValueError):
        bm.forward(torch.zeros(1, 5, 165, device=DEV), betas=torch.zeros(2, 300, device=DEV))
    with pytest.raises(ValueError):
        bm.forward(torch.zeros(1, 5, 165, device=DEV, dtype=torch.float64))
    with pytest.raises(_lib.PmError):
        bm.forward(torch.zeros(1, 5, 165))
    with pytest.raises(_lib.PmError):
        bm.forward(torch.zeros(1, 5, 165, device=DEV), transl=torch.zeros(1, 5, 3))


def test_camn_demo_writes_the_reference_pelvis_translation(tmp_path, golden_dir):
    np.savez(tmp_path / "model.npz", **small_arrays())
    wavs = tmp_path / "wavs"
    wavs.mkdir()
    with wave.open(str(wavs / "a.wav"), "wb") as w:
        w.setnchannels(1), w.setsampwidth(2), w.setframerate(16000)
        t = np.arange(16000 * 2) / 16000
        w.writeframes((np.sin(2 * np.pi * 220 * t) * 8000).astype("<i2").tobytes())
    subprocess.run([sys.executable, os.path.join(ROOT, "examples", "camn_disco_demo.py"), "--model", "camn", "--synthetic",
                    "--audio_folder", str(wavs), "--save_folder", str(tmp_path / "out"), "--smplx",
                    str(tmp_path / "model.npz")], check=True, cwd=ROOT)
    trans = np.load(tmp_path / "out" / "a_output.npz")["trans"]
    want = np.load(os.path.join(golden_dir, "case_body.npz"))["save_trans_zero_betas"][0]
    np.testing.assert_allclose(trans, np.broadcast_to(want, trans.shape), rtol=0, atol=1e-6)

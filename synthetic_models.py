"""Benchmark / test support: the drop-in modules filled with the deterministic synthetic checkpoint.

There is no network, so the Hugging Face checkpoints the reference downloads are not available; every tensor of a
reference-layout state_dict is drawn from the name-keyed generator in oracle/weights.py (pure data generation - no
oracle arithmetic) and loaded through load_state_dict(strict=True), i.e. through the checkpoint boundary.
Used by bench.py, __graft_entry__.smoke(), tools/ and tests/; the product package never imports it."""
from __future__ import annotations

import hashlib

import numpy as np

from oracle.weights import EMAGE_CFG, LSTM_CFG, VQ_CFGS, load_synthetic

# The 55-joint SMPL-X tree (pelvis, legs, spine, neck / collars / head, arms, jaw, eyes, 15 left- then 15 right-hand
# joints): root to finger tip is 10 levels.
SMPLX_PARENTS = (-1, 0, 0, 0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 9, 9, 12, 13, 14, 16, 17, 18, 19, 15, 15, 15,
                 20, 25, 26, 20, 28, 29, 20, 31, 32, 20, 34, 35, 20, 37, 38,
                 21, 40, 41, 21, 43, 44, 21, 46, 47, 21, 49, 50, 21, 52, 53)
SMPLX_FULL_VERTS = 10475        # the real model's vertex count: GPU tests and the benchmark
SMPLX_SMALL_VERTS = 330         # CPU tests and tests/golden/case_body.npz


def smplx_arrays(n_verts=SMPLX_FULL_VERTS, seed=0, parents=SMPLX_PARENTS):
    """A synthetic SMPL-X model with the keys and shapes of SMPLX_NEUTRAL_2020.npz, drawn from numpy PCG64 (identical on
    every machine): bones of 5-40 cm, vertices scattered around their joint, J_regressor rows positive and summing to 1,
    at most 4 skinning weights per vertex summing to 1, blend directions ~1e-2 m per unit, hand means ~0.2 rad."""
    rng = np.random.Generator(np.random.PCG64(seed))
    nj = len(parents)
    joints = np.zeros((nj, 3))
    for j in range(1, nj):
        d = rng.standard_normal(3)
        joints[j] = joints[parents[j]] + d / np.linalg.norm(d) * rng.uniform(0.05, 0.40)
    owner = np.arange(n_verts) % nj
    v_template = joints[owner] + rng.normal(0.0, 0.03, (n_verts, 3))
    j_reg = np.zeros((nj, n_verts))
    j_reg[owner, np.arange(n_verts)] = rng.uniform(0.5, 1.5, n_verts)
    j_reg /= j_reg.sum(1, keepdims=True)
    weights = np.zeros((n_verts, nj))
    for v in range(n_verts):
        cand = [owner[v]] + ([parents[owner[v]]] if parents[owner[v]] >= 0 else [])
        cand += [int(c) for c in rng.choice(nj, 2, replace=False)]
        cand = list(dict.fromkeys(cand))[:4]
        weights[v, cand] = rng.dirichlet(np.ones(len(cand)))
    decay = 1.0 / (1.0 + np.arange(400) / 50.0)
    shapedirs = rng.standard_normal((n_verts, 3, 400)) * 1e-2 * decay
    posedirs = rng.standard_normal((n_verts, 3, 486)) * 1e-2
    kintree = np.stack([np.asarray(parents, dtype=np.int64), np.arange(nj, dtype=np.int64)])
    return {
        "v_template": v_template, "shapedirs": shapedirs.astype(np.float32), "posedirs": posedirs.astype(np.float32),
        "J_regressor": j_reg, "weights": weights, "kintree_table": kintree,
        "hands_meanl": rng.normal(0.0, 0.2, 45), "hands_meanr": rng.normal(0.0, 0.2, 45),
        "f": rng.integers(0, n_verts, (2 * n_verts, 3)).astype(np.int32),
    }


def write_smplx_npz(path, n_verts=SMPLX_FULL_VERTS, seed=0):
    """Write smplx_arrays(...) as an SMPLX_NEUTRAL_2020.npz-format file; returns the arrays."""
    arrays = smplx_arrays(n_verts, seed)
    np.savez(path, **arrays)
    return arrays


def smplx_hash(arrays) -> str:
    """sha256 over the arrays (names, dtypes, shapes, bytes): pins a golden to the model it was made with."""
    h = hashlib.sha256()
    for k in sorted(arrays):
        a = np.ascontiguousarray(arrays[k])
        h.update(f"{k}:{a.dtype.str}:{a.shape}".encode())
        h.update(a.tobytes())
    return h.hexdigest()


def build_product(seed=0, device="cuda"):
    """(EmageAudioModel, EmageVQModel) of pantomatrix_b200.emage_audio with synthetic weights."""
    from pantomatrix_b200.emage_audio import (EmageAudioConfig, EmageAudioModel, EmageVAEConv, EmageVAEConvConfig,
                                              EmageVQModel, EmageVQVAEConv, EmageVQVAEConvConfig)
    model = load_synthetic(EmageAudioModel(EmageAudioConfig(**EMAGE_CFG)), seed, "emage").to(device).eval()
    vq = {p: load_synthetic(EmageVQVAEConv(EmageVQVAEConvConfig(**VQ_CFGS[p])), seed, "vq_" + p).to(device).eval()
          for p in ("face", "upper", "hands", "lower")}
    glob = load_synthetic(EmageVAEConv(EmageVAEConvConfig(**VQ_CFGS["global"])), seed, "vq_global").to(device).eval()
    vqm = EmageVQModel(face_model=vq["face"], upper_model=vq["upper"], lower_model=vq["lower"],
                       hands_model=vq["hands"], global_model=glob).to(device).eval()
    return model, vqm


def build_lstm_product(kind, seed=0, device="cuda"):
    """CamnAudioModel ("camn") or DiscoAudioModel ("disco") of pantomatrix_b200.lstm_audio with synthetic weights."""
    from pantomatrix_b200.lstm_audio import CamnAudioConfig, CamnAudioModel, DiscoAudioConfig, DiscoAudioModel
    cls, ccls = (CamnAudioModel, CamnAudioConfig) if kind == "camn" else (DiscoAudioModel, DiscoAudioConfig)
    return load_synthetic(cls(ccls(**LSTM_CFG)), seed, kind).to(device).eval()

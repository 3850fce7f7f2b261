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


# Rest offsets (metres, y up) of the 22 body joints from their parents, a rough standing figure: the surface model's
# skeleton, so that its mesh is framed like a body by the render's camera.  Hand joints are laid out procedurally.
_BODY_OFFSETS = {1: (0.06, -0.09, 0.0), 2: (-0.06, -0.09, 0.0), 3: (0.0, 0.11, -0.02), 4: (0.04, -0.38, 0.0),
                 5: (-0.04, -0.38, 0.0), 6: (0.0, 0.13, 0.02), 7: (-0.01, -0.40, -0.04), 8: (0.01, -0.40, -0.04),
                 9: (0.0, 0.05, 0.0), 10: (0.02, -0.06, 0.12), 11: (-0.02, -0.06, 0.12), 12: (0.0, 0.21, -0.02),
                 13: (0.08, 0.12, -0.01), 14: (-0.08, 0.12, -0.01), 15: (0.0, 0.09, 0.05), 16: (0.11, 0.04, -0.01),
                 17: (-0.11, 0.04, -0.01), 18: (0.26, -0.01, -0.02), 19: (-0.26, -0.01, -0.02), 20: (0.25, 0.01, 0.0),
                 21: (-0.25, 0.01, 0.0), 22: (0.0, -0.01, 0.03), 23: (0.03, 0.06, 0.07), 24: (-0.03, 0.06, 0.07)}


def _surface_joints(parents):
    off = np.zeros((len(parents), 3))
    for j, o in _BODY_OFFSETS.items():
        off[j] = o
    for j in range(25, len(parents)):                 # 5 fingers x 3 joints per hand, fanned out from the wrist
        side = 1.0 if j < 40 else -1.0
        finger, knuckle = divmod((j - 25) % 15, 3)
        off[j] = (side * 0.03, 0.0, 0.035 - 0.02 * finger) if knuckle == 0 else (side * 0.025, 0.0, 0.0)
    joints = np.zeros_like(off)
    for j in range(1, len(parents)):
        joints[j] = joints[parents[j]] + off[j]
    return joints


def _capsule(a, b, radius, n):
    """A closed capsule around segment a -> b with at most n vertices (two poles and rings x segments) and its outward
    triangles.  Returns (vertices, faces, which end each vertex belongs to (0 at a, 1 at b), the equator ring at a)."""
    segs = max(range(6, 25), key=lambda s: (s * ((n - 2) // s), -abs(s - 12)))
    rings = (n - 2) // segs
    half = rings // 2                                  # rings [0, half) on the hemisphere at a, the rest at b
    z = b - a
    z = z / np.linalg.norm(z)
    x = np.cross(z, [1.0, 0.0, 0.0] if abs(z[0]) < 0.9 else [0.0, 1.0, 0.0])
    x /= np.linalg.norm(x)
    y = np.cross(z, x)
    phi = np.arange(segs) * 2 * np.pi / segs
    circle = np.cos(phi)[:, None] * x + np.sin(phi)[:, None] * y
    verts, end = [a - z * radius], [0.0]
    for r in range(rings):
        at_b = r >= half
        polar = np.pi / 2 * ((r + 1) / half if not at_b else 1 + (r - half) / (rings - half))
        verts += list((b if at_b else a) - z * radius * np.cos(polar) + radius * np.sin(polar) * circle)
        end += [float(at_b)] * segs
    verts.append(b + z * radius)
    end.append(1.0)
    top = len(verts) - 1
    ring = lambda r, s: 1 + r * segs + s % segs
    faces = []
    for s in range(segs):
        faces += [(0, ring(0, s + 1), ring(0, s)), (top, ring(rings - 1, s), ring(rings - 1, s + 1))]
        for r in range(rings - 1):
            faces += [(ring(r, s), ring(r + 1, s + 1), ring(r + 1, s)), (ring(r, s), ring(r, s + 1), ring(r + 1, s + 1))]
    return np.array(verts), np.array(faces), np.array(end), [ring(half - 1, s) for s in range(segs)]


def smplx_surface_arrays(n_verts=SMPLX_FULL_VERTS, seed=0, parents=SMPLX_PARENTS):
    """A synthetic SMPL-X model with a real surface: the keys and shapes of smplx_arrays, but v_template is a closed
    capsule around each of the 55 bones of a standing figure (joint j's capsule runs from j to its first child, or on
    past j for a leaf), the vertices split evenly across the capsules (any remainder sits unreferenced at the joint), f
    their outward-wound triangulation, J_regressor the mean of the capsule's equator ring at its joint, and each vertex
    skinned to its capsule's joint, blended 30 % with the parent on the half at the joint.  The other arrays are drawn
    as in smplx_arrays.  Closed meshes with body-like triangle sizes, for the render's tests and benchmark."""
    rng = np.random.Generator(np.random.PCG64(seed))
    nj = len(parents)
    if n_verts < 16 * nj:
        raise ValueError(f"smplx_surface_arrays needs at least {16 * nj} vertices")
    joints = _surface_joints(parents)
    children = {j: [c for c in range(nj) if parents[c] == j] for j in range(nj)}
    v_template = np.zeros((n_verts, 3))
    j_reg = np.zeros((nj, n_verts))
    weights = np.zeros((n_verts, nj))
    faces, start = [], 0
    for j in range(nj):
        n = n_verts // nj + (j < n_verts % nj)
        a = joints[j]
        if j == 15:                                    # the head: a ball above the neck rather than a tube to the jaw
            b, radius = a + (0.0, 0.14, 0.01), 0.09
        else:
            if children[j]:
                b = joints[children[j][0]]
            else:
                b = a + 0.5 * (a - joints[parents[j]])
            radius = 0.12 if j == 0 else float(np.clip(0.3 * np.linalg.norm(b - a), 0.008, 0.09))
        v, f, end, equator = _capsule(a, b, radius, n)
        v_template[start:start + n] = a
        v_template[start:start + len(v)] = v
        faces.append(f + start)
        j_reg[j, start + np.array(equator)] = 1.0 / len(equator)
        weights[start:start + n, j] = 1.0
        near = start + np.nonzero(end == 0.0)[0]
        if parents[j] >= 0:
            weights[near, j], weights[near, parents[j]] = 0.7, 0.3
        start += n
    decay = 1.0 / (1.0 + np.arange(400) / 50.0)
    shapedirs = rng.standard_normal((n_verts, 3, 400)) * 1e-2 * decay
    posedirs = rng.standard_normal((n_verts, 3, 486)) * 1e-2
    kintree = np.stack([np.asarray(parents, dtype=np.int64), np.arange(nj, dtype=np.int64)])
    return {
        "v_template": v_template, "shapedirs": shapedirs.astype(np.float32), "posedirs": posedirs.astype(np.float32),
        "J_regressor": j_reg, "weights": weights, "kintree_table": kintree,
        "hands_meanl": rng.normal(0.0, 0.2, 45), "hands_meanr": rng.normal(0.0, 0.2, 45),
        "f": np.concatenate(faces).astype(np.int32),
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

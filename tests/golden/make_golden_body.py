"""Generate tests/golden/case_body.npz: the reference's own motion-representation and npz-writer code run over the small
synthetic SMPL-X model.

    python tests/golden/make_golden_body.py [REFERENCE_ROOT]

The unmodified emage_utils.motion_rep_transfer and emage_utils.motion_io are imported with two stub modules: `smplx`,
whose create() returns the float32 restatement of oracle/smplx_oracle.py over synthetic_models.smplx_arrays(
SMPLX_SMALL_VERTS), and `wget`, whose download() raises (the model file is put where the reference looks for it, in a
temporary working directory, so its download branch is never taken).  This pins what the reference composes around the
body model (which joints are zeroed, the ignored betas, the difference formulas, the rot6d route, the rep15d layout, the
pelvis formula and the upsampling) without any reference source entering this repository.

Stored: the inputs (poses, betas), the six get_motion_rep_tensor outputs (2 clips x 34 frames, device="cpu"), the trans
written by beat_format_save(trans=None, upsample=2) with non-zero betas (`save_trans`) and with betas=None
(`save_trans_zero_betas`, what the CaMN / DisCo demo writes), and the sha256 of the model arrays.
"""
import os
import sys
import tempfile
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

from oracle import smplx_oracle  # noqa: E402
from synthetic_models import SMPLX_SMALL_VERTS, smplx_hash, write_smplx_npz  # noqa: E402

CLIPS, FRAMES, SAVE_FRAMES = 2, 34, 12


def poses_case(rng):
    """Seeded axis-angle poses (clips, frames, 165) with a zero joint, a tiny rotation and angles near pi."""
    p = rng.normal(0.0, 0.4, (CLIPS, FRAMES, 55, 3))
    p[:, :, 5] = 0.0
    p[:, :, 7] = rng.normal(0.0, 1e-7, (CLIPS, FRAMES, 3))
    axis = rng.normal(size=(CLIPS, FRAMES, 3))
    p[:, :, 16] = axis / np.linalg.norm(axis, axis=-1, keepdims=True) * (np.pi - 1e-3)
    return p.reshape(CLIPS, FRAMES, 165).astype(np.float32)


def main(ref_root="/root/reference"):
    rng = np.random.default_rng(20261016)
    poses = poses_case(rng)
    betas = rng.normal(0.0, 1.0, (SAVE_FRAMES, 300)).astype(np.float32)
    motion = rng.normal(0.0, 0.3, (SAVE_FRAMES, 165)).astype(np.float32)
    out = {"poses": poses, "betas": betas, "save_motion": motion}
    cwd = os.getcwd()
    with tempfile.TemporaryDirectory() as tmp:
        model_dir = os.path.join(tmp, "emage_evaltools", "smplx_models", "smplx")
        os.makedirs(model_dir)
        arrays = write_smplx_npz(os.path.join(model_dir, "SMPLX_NEUTRAL_2020.npz"), SMPLX_SMALL_VERTS)
        out["model_sha256"] = np.array(smplx_hash(arrays))
        stub = types.ModuleType("smplx")
        stub.create = lambda *a, **kw: smplx_oracle.create(*a, dtype=torch.float32, **kw)
        wget = types.ModuleType("wget")

        def no_download(*a, **kw):
            raise RuntimeError("wget.download called: the synthetic model file was not found")

        wget.download = no_download
        sys.modules["smplx"], sys.modules["wget"] = stub, wget
        sys.path.insert(0, ref_root)
        os.chdir(tmp)
        try:
            from emage_utils import motion_io, motion_rep_transfer
            rep = motion_rep_transfer.get_motion_rep_tensor(torch.from_numpy(poses), pose_fps=30, device="cpu")
            for k, v in rep.items():
                out["rep_" + k] = v.numpy()
            motion_io.beat_format_save(os.path.join(tmp, "a.npz"), motion, betas=betas, trans=None, upsample=2)
            out["save_trans"] = np.load(os.path.join(tmp, "a.npz"))["trans"]
            motion_io.beat_format_save(os.path.join(tmp, "b.npz"), motion, trans=None, upsample=2)
            out["save_trans_zero_betas"] = np.load(os.path.join(tmp, "b.npz"))["trans"]
        finally:
            os.chdir(cwd)
    np.savez(os.path.join(HERE, "case_body.npz"), **out)


if __name__ == "__main__":
    main(*sys.argv[1:])

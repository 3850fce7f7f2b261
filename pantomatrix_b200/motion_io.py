"""Output writer of the EMAGE path: the step right after the hot path (SURVEY.md section 8f-3).

Behavioural mirror of the parts of /root/reference/emage_utils/motion_io.py the demo needs
(`beat_format_save` :103-163, `beat_format_load` :165-179, `time_upsample_numpy` :69-101, joint-mask
select / recover :22-67), written against numpy only.  When `trans` is None the reference builds the SMPL-X body
model to derive a default translation; here the caller passes the model (`body_model=`, pantomatrix_b200.body_model),
and without one `trans=None` raises with an explanation (the EMAGE demo always passes the translation it generated,
test_emage_audio.py:53-55).
"""
from __future__ import annotations

import numpy as np

NPZ_MODEL, NPZ_GENDER, NPZ_FPS = "smplx2020", "neutral", 30


def time_upsample_numpy(data: np.ndarray, k: int) -> np.ndarray:
    """(..., t, c) -> (..., k*t, c): piecewise-linear resampling on k*t points spread evenly over [0, t-1]
    (so first and last frames are kept and the spacing is (t-1)/(k*t-1), as in the reference)."""
    if k == 1:
        return data.copy()
    t = data.shape[-2]
    pos = np.linspace(0, t - 1, k * t)
    lo = np.clip(np.floor(pos).astype(np.int64), 0, max(t - 2, 0))
    frac = (pos - lo).reshape((-1, 1))
    a = np.take(data, lo, axis=-2)
    b = np.take(data, np.minimum(lo + 1, t - 1), axis=-2)
    return a + (b - a) * frac


def recover_from_mask(selected: np.ndarray, mask) -> np.ndarray:
    """(..., n_selected*c) joint features -> (..., n_joints*c) with zeros at unselected joints."""
    mask = np.asarray(mask, dtype=bool)
    n_sel = int(mask.sum())
    c = selected.shape[-1] // n_sel
    out = np.zeros(selected.shape[:-1] + (mask.size, c), dtype=selected.dtype)
    out[..., mask, :] = selected.reshape(selected.shape[:-1] + (n_sel, c))
    return out.reshape(selected.shape[:-1] + (mask.size * c,))


def select_with_mask(motion: np.ndarray, mask) -> np.ndarray:
    mask = np.asarray(mask, dtype=bool)
    c = motion.shape[-1] // mask.size
    picked = motion.reshape(motion.shape[:-1] + (mask.size, c))[..., mask, :]
    return picked.reshape(motion.shape[:-1] + (int(mask.sum()) * c,))


def pelvis_translation(body_model, betas0) -> np.ndarray:
    """(3,) float32 translation the reference writer derives when none is given (motion_io.py:116-143): minus the
    midpoint of joints 10 and 11 (the feet) of the rest pose for betas0 (300,).  body_model: a
    body_model.SmplxBodyModel (or anything with its forward() and device)."""
    import torch
    dev = body_model.device
    b = torch.from_numpy(np.asarray(betas0)[None]).float().to(dev)
    joints = body_model.forward(torch.zeros(1, 1, 165, device=dev), betas=b)["joints"].reshape(-1, 55, 3)[:1].cpu()
    return (-((joints[:, 10, :] + joints[:, 11, :]) / 2)).numpy()[0]


def beat_format_save(save_path, motion_data, mask=None, betas=None, expressions=None, trans=None, upsample=None,
                     body_model=None):
    """Write a BEAT-format npz: betas (300,), poses (T,165), expressions (T,100), trans (T,3), model, gender,
    mocap_frame_rate - same keys, shapes and constants as the reference writer.  trans=None places the pelvis as the
    reference does (pelvis_translation of betas[0], repeated over the frames), which needs the SMPL-X `body_model`."""
    motion_data = np.asarray(motion_data)
    n = motion_data.shape[0]
    if betas is None:
        betas = np.zeros((n, 300), dtype=motion_data.dtype)
    if expressions is None:
        expressions = np.zeros((n, 100), dtype=motion_data.dtype)
    if trans is None:
        if body_model is None:
            raise NotImplementedError(
                "beat_format_save(trans=None) needs the SMPL-X body model to place the pelvis: pass "
                "body_model=body_model.SmplxBodyModel.from_npz('SMPLX_NEUTRAL_2020.npz'), or the translation produced "
                "by EmageVQModel.decode(get_global_motion=True)")
        trans = np.repeat(pelvis_translation(body_model, betas[0])[None], n, axis=0)
    if mask is not None:
        motion_data = recover_from_mask(motion_data, mask)
    if upsample is not None and upsample > 1:
        motion_data, betas = time_upsample_numpy(motion_data, upsample), time_upsample_numpy(betas, upsample)
        expressions, trans = time_upsample_numpy(expressions, upsample), time_upsample_numpy(np.asarray(trans), upsample)
    np.savez(save_path, betas=betas[0], poses=motion_data, expressions=expressions, trans=trans,
             model=NPZ_MODEL, gender=NPZ_GENDER, mocap_frame_rate=NPZ_FPS)


def beat_format_load(load_path, mask=None):
    data = np.load(load_path, allow_pickle=True)
    poses = data["poses"]
    if mask is not None:
        poses = select_with_mask(poses, mask)
    return {"poses": poses, "betas": data["betas"], "expressions": data["expressions"], "trans": data["trans"]}

"""Generate tests/golden/case_render_layouts.npz: the reference's body-only and prediction-beside-ground-truth render
compositions (emage_utils/fast_render.py render_one_sequence_no_gt and render_one_sequence) run over the small synthetic
SMPL-X model, with every scene they would draw recorded.

    python tests/golden/make_golden_render_layouts.py [REFERENCE_ROOT]

The unmodified emage_utils.fast_render and emage_utils.motion_io are imported with the stub modules of
make_golden_render.py (`smplx` is the float32 restatement of oracle/smplx_oracle.py, pyrender / trimesh / imageio /
matplotlib are recorders, .cuda() is the identity); the silent-video writers run the reference's distribute_frames /
render_frames_and_enqueue / write_images_from_queue (and their _no_gt forms) without the process pool, and
add_audio_to_video does nothing.  Two cases, keys prefixed body_ and pair_:
  body  15 fps poses (37 frames) written by the reference's beat_format_save(..., upsample=2) with trans=None, so the
        writer places the pelvis with the model, then render_one_sequence_no_gt on that npz;
  pair  render_one_sequence(pred, gt) with different betas, expressions and translations on each side and the ground
        truth longer than the prediction.
Recorded per case: the npz contents the renderer read, the vertices of each drawn scene in frame order ((n, views, V,
3), left to right), the frame count, the viewport and the shape of each written image.
"""
import os
import queue
import sys
import tempfile

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)

from make_golden_render import _stubs  # noqa: E402
from synthetic_models import SMPLX_SMALL_VERTS, smplx_hash, write_smplx_npz  # noqa: E402

BODY_FRAMES = 37            # 15 fps -> 74 frames at 30 fps -> 60 drawn
PRED_FRAMES, GT_FRAMES = 40, 52


def _silent_writer(fast_render, scenes_per_image, record):
    """generate_silent_videos(_no_gt) without the process pool and the video encoder: records the frame count."""
    def write(frames, *args):
        *verts, faces, output_dir = args
        record["frames"] = frames
        if scenes_per_image == 1:
            ids, pairs = fast_render.distribute_frames_no_gt(frames, *verts)
            enqueue, drain = fast_render.render_frames_and_enqueue_no_gt, fast_render.write_images_from_queue_no_gt
        else:
            ids, pairs = fast_render.distribute_frames(frames, *verts)
            enqueue, drain = fast_render.render_frames_and_enqueue, fast_render.write_images_from_queue
        q = queue.Queue()
        for i in range(len(ids)):
            enqueue(ids[i], pairs[i], faces, fast_render.args["render_video_width"],
                    fast_render.args["render_video_height"], q)
        q.put(None)
        drain(q, output_dir, fast_render.args["render_tmp_img_filetype"])
        out = os.path.join(output_dir, "silence_video.mp4")
        open(out, "w").close()
        return out
    return write


def _collect(scenes, images, views, frames):
    """Scene vertices (frames, views, V, 3) in frame order, the viewport and the image shape."""
    assert len(scenes) == views * frames and len(images) == frames
    verts = [np.asarray(scene.added[0][0].args[0].kw["vertices"], np.float32) for scene, _ in scenes]
    assert all(vp == scenes[0][1] for _, vp in scenes) and all(im[1] == images[0][1] for im in images)
    order = np.argsort([int(name.split("_")[1].split(".")[0]) for name, _ in images], kind="stable")
    return np.stack(verts).reshape(frames, views, -1, 3)[order], np.array(scenes[0][1]), np.array(images[0][1])


def main(ref_root="/root/reference"):
    rng = np.random.default_rng(20261018)
    scenes, images = [], []
    sys.modules.update(_stubs(scenes, images))
    sys.path.insert(0, ref_root)
    cuda_t, cuda_m = torch.Tensor.cuda, torch.nn.Module.cuda
    torch.Tensor.cuda = lambda self, *a, **kw: self
    torch.nn.Module.cuda = lambda self, *a, **kw: self
    cwd = os.getcwd()
    out = {}
    try:
        from emage_utils import fast_render, motion_io
        fast_render.add_audio_to_video = lambda *a, **kw: None
        with tempfile.TemporaryDirectory() as tmp:
            os.chdir(tmp)
            # beat_format_save(trans=None) loads ./emage_evaltools/smplx_models/, the renderer model_folder
            model_dir = os.path.join(tmp, "emage_evaltools", "smplx_models")
            os.makedirs(os.path.join(model_dir, "smplx"))
            arrays = write_smplx_npz(os.path.join(model_dir, "smplx", "SMPLX_NEUTRAL_2020.npz"), SMPLX_SMALL_VERTS)
            out["model_sha256"] = np.array(smplx_hash(arrays))

            # body only: CaMN / DisCo output as the reference test scripts write and render it
            poses15 = rng.normal(0.0, 0.3, (BODY_FRAMES, 165)).astype(np.float32)
            npz = os.path.join(tmp, "body.npz")
            motion_io.beat_format_save(npz, poses15, upsample=2)
            rec = {}
            fast_render.generate_silent_videos_no_gt = _silent_writer(fast_render, 1, rec)
            fast_render.render_one_sequence_no_gt(npz, os.path.join(tmp, "out_body"), "audio.wav", model_folder=model_dir)
            saved = np.load(npz)
            verts, viewport, shape = _collect(scenes, images, 1, rec["frames"])
            out.update(body_poses15=poses15, body_poses=saved["poses"], body_expressions=saved["expressions"],
                       body_trans=saved["trans"], body_betas=saved["betas"], body_vertices=verts,
                       body_frames=np.array(rec["frames"]), body_viewport=viewport, body_image_shape=shape)
            scenes.clear()
            images.clear()

            # prediction beside a longer ground truth, each with its own betas, expressions and translation
            sides = {}
            for tag, t in (("pred", PRED_FRAMES), ("gt", GT_FRAMES)):
                sides[tag] = {"poses": rng.normal(0.0, 0.3, (t, 165)).astype(np.float32),
                              "expressions": rng.normal(0.0, 0.5, (t, 100)).astype(np.float32),
                              "trans": (rng.normal(0.0, 0.05, (t, 3)) + (0.0, 1.0, 0.0)).astype(np.float32),
                              "betas": rng.normal(0.0, 1.0, 300).astype(np.float32)}
                np.savez(os.path.join(tmp, f"{tag}.npz"), **sides[tag])
            rec = {}
            fast_render.generate_silent_videos = _silent_writer(fast_render, 2, rec)
            fast_render.render_one_sequence(os.path.join(tmp, "pred.npz"), os.path.join(tmp, "gt.npz"),
                                            os.path.join(tmp, "out_pair"), "audio.wav", model_folder=model_dir)
            verts, viewport, shape = _collect(scenes, images, 2, rec["frames"])
            for tag, d in sides.items():
                out.update({f"pair_{tag}_{k}": v for k, v in d.items()})
            out.update(pair_vertices=verts, pair_frames=np.array(rec["frames"]), pair_viewport=viewport,
                       pair_image_shape=shape)
    finally:
        os.chdir(cwd)
        torch.Tensor.cuda, torch.nn.Module.cuda = cuda_t, cuda_m
    np.savez(os.path.join(HERE, "case_render_layouts.npz"), **out)


if __name__ == "__main__":
    main(*sys.argv[1:])

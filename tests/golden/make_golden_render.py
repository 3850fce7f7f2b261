"""Generate tests/golden/case_render.npz: the reference's own render composition (emage_utils/fast_render.py
render_one_sequence_with_face) run over the small synthetic SMPL-X model, with every scene it would draw recorded.

    python tests/golden/make_golden_render.py [REFERENCE_ROOT]

The unmodified emage_utils.fast_render is imported with stub modules for what is not installed: `smplx` (create() returns
the float32 restatement of oracle/smplx_oracle.py over synthetic_models.smplx_arrays(SMPLX_SMALL_VERTS)), `pyrender`,
`trimesh`, `imageio` and `matplotlib` (recorders), and with .cuda() made the identity.  generate_silent_videos runs the
reference's distribute_frames / render_frames_and_enqueue / write_images_from_queue without the process pool, and
add_audio_to_video does nothing.  Recorded per drawn frame, in left-to-right order: the vertex arrays, faces, camera and
light poses, xmag / ymag, light intensity and colour, mesh colour and the viewport; plus the frame count and the shape
of the merged image.  This pins the x7 / -10 face view, the jaw-only pose, the frame-0 translation, the view order and
the whole-second truncation without any reference source entering this repository.
"""
import os
import queue
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

FRAMES = 2 * 30 + 7


class _Rec:
    """Records its constructor arguments; any method call is accepted and recorded."""

    def __init__(self, *a, **kw):
        self.args, self.kw, self.added = a, kw, []

    def add(self, obj, pose=None):
        self.added.append((obj, pose))


def _stubs(scenes, images):
    pyrender = types.ModuleType("pyrender")

    class Mesh(_Rec):
        @staticmethod
        def from_trimesh(tm, smooth=False):
            return Mesh(tm, smooth=smooth)

    class OffscreenRenderer(_Rec):
        def render(self, scene):
            w, h = self.args
            scenes.append((scene, (w, h)))
            return np.zeros((h, w, 3), np.uint8), np.zeros((h, w), np.float32)

        def delete(self):
            pass

    pyrender.Mesh, pyrender.OffscreenRenderer = Mesh, OffscreenRenderer
    for name in ("Scene", "OrthographicCamera", "DirectionalLight"):
        setattr(pyrender, name, type(name, (_Rec,), {}))
    trimesh = types.ModuleType("trimesh")
    trimesh.Trimesh = type("Trimesh", (_Rec,), {})
    imageio = types.ModuleType("imageio")
    imageio.imwrite = lambda fn, img: images.append((os.path.basename(fn), img.shape))
    mpl = types.ModuleType("matplotlib")
    mpl.use = lambda *a, **kw: None
    mpl.pyplot = types.ModuleType("matplotlib.pyplot")
    smplx = types.ModuleType("smplx")
    smplx.create = lambda *a, **kw: smplx_oracle.create(*a, dtype=torch.float32, **kw)
    return {"pyrender": pyrender, "trimesh": trimesh, "imageio": imageio, "matplotlib": mpl,
            "matplotlib.pyplot": mpl.pyplot, "smplx": smplx}


def main(ref_root="/root/reference"):
    rng = np.random.default_rng(20261017)
    data = {"poses": rng.normal(0.0, 0.3, (FRAMES, 165)).astype(np.float32),
            "expressions": rng.normal(0.0, 0.5, (FRAMES, 100)).astype(np.float32),
            "trans": (rng.normal(0.0, 0.05, (FRAMES, 3)) + (0.0, 1.0, 0.0)).astype(np.float32),
            "betas": rng.normal(0.0, 1.0, 300).astype(np.float32)}
    scenes, images, silent = [], [], {}
    sys.modules.update(_stubs(scenes, images))
    sys.path.insert(0, ref_root)
    cuda_t, cuda_m = torch.Tensor.cuda, torch.nn.Module.cuda
    torch.Tensor.cuda = lambda self, *a, **kw: self
    torch.nn.Module.cuda = lambda self, *a, **kw: self
    try:
        from emage_utils import fast_render
        with tempfile.TemporaryDirectory() as tmp:
            model_dir = os.path.join(tmp, "smplx")
            os.makedirs(model_dir)
            arrays = write_smplx_npz(os.path.join(model_dir, "SMPLX_NEUTRAL_2020.npz"), SMPLX_SMALL_VERTS)
            npz = os.path.join(tmp, "res.npz")
            np.savez(npz, **data)

            def generate_silent_videos(frames, vertices_all, vertices1_all, faces, output_dir):
                silent["frames"] = frames
                ids, verts = fast_render.distribute_frames(frames, vertices_all, vertices1_all)
                q = queue.Queue()
                for i in range(len(ids)):
                    fast_render.render_frames_and_enqueue(ids[i], verts[i], faces, fast_render.args["render_video_width"],
                                                          fast_render.args["render_video_height"], q)
                q.put(None)
                fast_render.write_images_from_queue(q, output_dir, fast_render.args["render_tmp_img_filetype"])
                out = os.path.join(output_dir, "silence_video.mp4")
                open(out, "w").close()
                return out

            fast_render.generate_silent_videos = generate_silent_videos
            fast_render.add_audio_to_video = lambda *a, **kw: None
            fast_render.render_one_sequence_with_face(npz, os.path.join(tmp, "out"), "audio.wav", model_folder=tmp)
    finally:
        torch.Tensor.cuda, torch.nn.Module.cuda = cuda_t, cuda_m
    # scenes and images arrive in the order of distribute_frames' lists (two scenes per image, left then right): sort
    # them by the frame id written into each image's file name
    n = silent["frames"]
    assert len(scenes) == 2 * n and len(images) == n
    verts, faces, cams, lights = [], None, [], []
    for i in range(2 * n):
        scene, viewport = scenes[i]
        (mesh, _), (cam, cam_pose), (light, light_pose) = scene.added
        tm = mesh.args[0]
        verts.append(np.asarray(tm.kw["vertices"], np.float32))
        faces = np.asarray(tm.kw["faces"])
        cams.append(cam_pose)
        lights.append(light_pose)
    frame_ids = [int(images[i][0].split("_")[1].split(".")[0]) for i in range(n)]
    perm = np.argsort(frame_ids, kind="stable")
    v = np.stack(verts).reshape(n, 2, -1, 3)[perm]
    out = dict(data, vertices=v, faces=faces, camera_pose=np.stack(cams)[0], light_pose=np.stack(lights)[0],
               camera_poses_equal=np.array(all(np.array_equal(c, cams[0]) for c in cams)
                                           and all(np.array_equal(li, lights[0]) for li in lights)),
               xmag=np.array(cam.kw["xmag"]), ymag=np.array(cam.kw["ymag"]), light_intensity=np.array(light.kw["intensity"]),
               light_color=np.array(light.kw["color"]), mesh_color=np.array(tm.kw["vertex_colors"]),
               smooth=np.array(mesh.kw["smooth"]), viewport=np.array(viewport), frames=np.array(n),
               merged_shape=np.array(images[0][1]), model_sha256=np.array(smplx_hash(arrays)))
    np.savez(os.path.join(HERE, "case_render.npz"), **out)


if __name__ == "__main__":
    main(*sys.argv[1:])

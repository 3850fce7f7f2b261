#!/usr/bin/env python
"""Audio folder -> BEAT-format npz with CaMN or DisCo on the H100 path (reference test_camn_audio.py / test_disco_audio.py).

    python examples/camn_disco_demo.py --model camn --checkpoint /path/to/camn_audio --audio_folder ./wavs
    python examples/camn_disco_demo.py --model disco --synthetic --audio_folder ./wavs
    python examples/camn_disco_demo.py ... --smplx SMPLX_NEUTRAL_2020.npz --render   # + <name>_frames/frame_%05d.png
    python examples/camn_disco_demo.py ... --smplx SMPLX_NEUTRAL_2020.npz --video    # + <name>_output.mp4
    python examples/camn_disco_demo.py ... --smplx SMPLX_NEUTRAL_2020.npz --video --with-audio   # the mp4 with sound

These models emit the upper body + hands only and no translation; like the reference demos the npz writer places the
pelvis with the SMPL-X body model: pass the model file with --smplx SMPLX_NEUTRAL_2020.npz (the translation the
reference writer derives), or --trans-zero to write zeros instead.
`--render` (needs --smplx) draws the reference demos' SMPL-X body view (fast_render.py render_one_sequence_no_gt: one
480 x 720 view, whole seconds at 30 fps) of the motion upsampled to 30 fps as the npz stores it, on the GPU, with the
translation the npz receives, and writes the frames as PNG files next to each npz, encoded on the GPU
(pantomatrix_b200.png).  `--video` (needs --smplx) encodes the same frames as H.264 on the GPU (pantomatrix_b200.video)
and writes <npz base>.mp4 (30 fps) beside each npz, silent unless `--with-audio` is given: that reads the WAV at its
own rate and channel count and writes it into the file as a FLAC track encoded on the GPU (pantomatrix_b200.flac),
trimmed to the video's length."""
import argparse
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from models.camn_audio import CamnAudioModel  # noqa: E402
from models.disco_audio import DiscoAudioModel  # noqa: E402
from pantomatrix_b200.audio_io import load_audio, read_track  # noqa: E402
from pantomatrix_b200.motion_io import beat_format_save, pelvis_translation  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--model", choices=["camn", "disco"], default="camn")
    ap.add_argument("--audio_folder", default="./examples/audio")
    ap.add_argument("--save_folder", default="./examples/motion")
    ap.add_argument("--checkpoint", default=None)
    ap.add_argument("--synthetic", action="store_true")
    ap.add_argument("--trans-zero", action="store_true")
    ap.add_argument("--smplx", default=None, metavar="PATH", help="SMPL-X model file (SMPLX_NEUTRAL_2020.npz)")
    ap.add_argument("--render", action="store_true")
    ap.add_argument("--video", action="store_true", help="write <npz base>.mp4 (needs --smplx)")
    ap.add_argument("--with-audio", action="store_true", help="put the WAV's sound in the --video file")
    ap.add_argument("--gop", type=int, default=1,
                    help="--video keyframe interval: an IDR frame every GOP frames, P frames between (1: all IDR)")
    ap.add_argument("--search", type=int, default=0,
                    help="--video motion search range in pixels, 0..32, for the P frames (0: zero motion)")
    ap.add_argument("--intra4x4", action="store_true",
                    help="--video: also code intra macroblocks as Intra 4x4 (nine prediction modes per 4x4 block)")
    args = ap.parse_args()
    if not args.trans_zero and args.smplx is None:
        ap.error("the npz needs a pelvis translation: pass --smplx SMPLX_NEUTRAL_2020.npz, or --trans-zero to write zeros")
    if args.render and args.smplx is None:
        ap.error("--render needs --smplx SMPLX_NEUTRAL_2020.npz")
    if args.video and args.smplx is None:
        ap.error("--video needs --smplx SMPLX_NEUTRAL_2020.npz")
    if args.with_audio and not args.video:
        ap.error("--with-audio needs --video")
    if args.gop < 1:
        ap.error("--gop must be at least 1")
    if not 0 <= args.search <= 32:
        ap.error("--search must be in 0..32")
    device = torch.device("cuda")
    body_model = renderer = None
    if args.smplx is not None:
        from pantomatrix_b200.body_model import SmplxBodyModel
        smplx_model = SmplxBodyModel.from_npz(args.smplx, device)
        body_model = None if args.trans_zero else smplx_model
        if args.render or args.video:
            from pantomatrix_b200.render import MeshRenderer
            renderer = MeshRenderer(smplx_model)
    if args.synthetic:
        sys.path.insert(0, os.path.join(ROOT, "tests"))
        from synthetic_models import build_lstm_product
        model = build_lstm_product(args.model, device=device)
    else:
        cls = CamnAudioModel if args.model == "camn" else DiscoAudioModel
        model = cls.from_pretrained(args.checkpoint).to(device).eval()
    os.makedirs(args.save_folder, exist_ok=True)
    sr, fps, seed_frames = model.cfg.audio_sr, model.cfg.pose_fps, model.cfg.seed_frames
    frames, t0 = 0, time.time()
    for name in sorted(f for f in os.listdir(args.audio_folder) if f.endswith(".wav")):
        audio = torch.from_numpy(load_audio(os.path.join(args.audio_folder, name), sr=sr)).unsqueeze(0).to(device)
        aa = model(audio, torch.zeros(1, 1, dtype=torch.long, device=device), seed_frames=seed_frames)["motion_axis_angle"]
        t = aa.shape[1]
        trans = None if body_model is not None else np.zeros((t, 3), dtype=np.float32)
        npz = os.path.join(args.save_folder, os.path.splitext(name)[0] + "_output.npz")
        beat_format_save(npz, aa.cpu().numpy().reshape(t, -1), upsample=30 // fps, trans=trans, body_model=body_model)
        if renderer is not None:
            # the npz's translation: the writer's pelvis placement (betas zero), or zeros under --trans-zero
            pelvis = np.zeros(3, np.float32) if trans is not None else pelvis_translation(body_model, np.zeros(300, np.float32))
            tr = torch.as_tensor(pelvis, device=device).expand(1, t, 3)
            drawn = renderer.render_body(aa.reshape(1, t, -1), tr, upsample=30 // fps)[0]
            if args.render:
                from pantomatrix_b200 import png
                png.write_frames(drawn, os.path.splitext(npz)[0] + "_frames")
            if args.video:
                from pantomatrix_b200 import video
                video.write_mp4(drawn, os.path.splitext(npz)[0] + ".mp4", fps=30,
                                audio=read_track(os.path.join(args.audio_folder, name), device)
                                if args.with_audio else None, gop=args.gop,
                                search=args.search, intra4x4=args.intra4x4)
        frames += t
    print(f"generate total {frames / fps:.2f} seconds motion in {time.time() - t0:.2f} seconds, saved in {args.save_folder}")


if __name__ == "__main__":
    main()

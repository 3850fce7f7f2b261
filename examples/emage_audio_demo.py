#!/usr/bin/env python
"""Audio folder -> BEAT-format motion npz files: the reference demo (test_emage_audio.py:71-105) on the H100 path.

    python examples/emage_audio_demo.py --checkpoint /path/to/emage_audio --audio_folder ./wavs --save_folder ./out
    python examples/emage_audio_demo.py --synthetic --audio_folder ./wavs            # seeded random weights (no network)
    python examples/emage_audio_demo.py ... --smplx SMPLX_NEUTRAL_2020.npz --render   # + <name>_frames/frame_%05d.png
    python examples/emage_audio_demo.py ... --smplx SMPLX_NEUTRAL_2020.npz --video    # + <name>_output.mp4
    python examples/emage_audio_demo.py ... --smplx SMPLX_NEUTRAL_2020.npz --video --with-audio   # the mp4 with sound

`--render` draws the reference demo's two-view SMPL-X frames (fast_render.py render_one_sequence_with_face: face
close-up left, body right, whole seconds at 30 fps) on the GPU and writes them as PNG files next to each npz,
encoded on the GPU (pantomatrix_b200.png).  `--video` (needs --smplx) encodes the same frames as H.264 on the GPU
(pantomatrix_b200.video) and writes <npz base>.mp4 (30 fps) beside each npz, silent unless `--with-audio` is given:
that reads the WAV at its own rate and channel count and writes it into the file as a FLAC track encoded on the GPU
(pantomatrix_b200.flac), trimmed to the video's length.
`--checkpoint` is a local copy of the Hugging Face repo layout the reference downloads (config.json +
model.safetensors at the top level, VQ models under emage_vq/{face,upper,lower,hands,global}).
"""
import argparse
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from models.emage_audio import EmageAudioModel, EmageVAEConv, EmageVQModel, EmageVQVAEConv  # noqa: E402  (GPU drop-in)
from pantomatrix_b200.audio_io import load_audio, read_track  # noqa: E402
from pantomatrix_b200.motion_io import beat_format_save  # noqa: E402
from pantomatrix_b200.pipeline import generate  # noqa: E402


def load_models(args, device):
    if args.synthetic:
        sys.path.insert(0, os.path.join(ROOT, "tests"))
        from synthetic_models import build_product
        return build_product(seed=0, device=device)
    ck = args.checkpoint
    vq = {p: EmageVQVAEConv.from_pretrained(ck, subfolder=f"emage_vq/{p}").to(device) for p in ("face", "upper", "lower", "hands")}
    glob = EmageVAEConv.from_pretrained(ck, subfolder="emage_vq/global").to(device)
    motion_vq = EmageVQModel(face_model=vq["face"], upper_model=vq["upper"], lower_model=vq["lower"],
                             hands_model=vq["hands"], global_model=glob).to(device).eval()
    return EmageAudioModel.from_pretrained(ck).to(device).eval(), motion_vq


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--audio_folder", default="./examples/audio")
    ap.add_argument("--save_folder", default="./examples/motion")
    ap.add_argument("--checkpoint", default=None)
    ap.add_argument("--synthetic", action="store_true")
    ap.add_argument("--smplx", default=None, help="SMPLX_NEUTRAL_2020.npz (needed by --render and --video)")
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
    if not args.synthetic and not args.checkpoint:
        ap.error("give --checkpoint DIR or --synthetic")
    if args.render and not args.smplx:
        ap.error("--render needs --smplx SMPLX_NEUTRAL_2020.npz")
    if args.video and not args.smplx:
        ap.error("--video needs --smplx SMPLX_NEUTRAL_2020.npz")
    if args.with_audio and not args.video:
        ap.error("--with-audio needs --video")
    if args.gop < 1:
        ap.error("--gop must be at least 1")
    if not 0 <= args.search <= 32:
        ap.error("--search must be in 0..32")
    os.makedirs(args.save_folder, exist_ok=True)
    device = torch.device("cuda")                      # no CPU fallback by design
    model, motion_vq = load_models(args, device)
    renderer = None
    if args.render or args.video:
        from pantomatrix_b200.body_model import SmplxBodyModel
        from pantomatrix_b200.render import MeshRenderer
        renderer = MeshRenderer(SmplxBodyModel.from_npz(args.smplx, device))
    sr, fps = model.cfg.audio_sr, model.cfg.pose_fps
    files = sorted(f for f in os.listdir(args.audio_folder) if f.endswith(".wav"))
    frames, t0 = 0, time.time()
    for name in files:
        audio = torch.from_numpy(load_audio(os.path.join(args.audio_folder, name), sr=sr)).unsqueeze(0)
        _, pred = generate(model, motion_vq, audio.to(device))
        t = pred["motion_axis_angle"].shape[1]
        npz = os.path.join(args.save_folder, os.path.splitext(name)[0] + "_output.npz")
        beat_format_save(npz, pred["motion_axis_angle"].cpu().numpy().reshape(t, -1), upsample=30 // fps,
                         expressions=pred["expression"].cpu().numpy().reshape(t, -1),
                         trans=pred["trans"].cpu().numpy().reshape(t, -1))
        if renderer is not None:
            drawn = renderer.render_sequence(pred["motion_axis_angle"], pred["expression"], pred["trans"])[0]
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
    print(f"generate total {frames / fps:.2f} seconds motion in {time.time() - t0:.2f} seconds")


if __name__ == "__main__":
    main()
